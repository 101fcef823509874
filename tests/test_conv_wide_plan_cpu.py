"""Host-side routing of the forward launches onto the wide kernel (no GPU needed): rave_conv1d_tc_wide_stages equals
the rule restated here at the shapes of the v2 training step's forward launches and at the edge cases (Cout not a
multiple of 192, Cout = 1536, short k, input widths that are not a multiple of 32)."""
import pytest


def restated(B, Cin, Cout, Lout, K):
    """Cout a multiple of 192, BLOCK_K = 64 (Cin % 64 == 0) or 32 (Cin % 32 == 0), at least 12 k-blocks of BLOCK_K
    input channels per tile; the ring keeps 4 stages (BLOCK_K = 64) or 8 (BLOCK_K = 32) next to the 48 KB output slot."""
    bk = 64 if Cin % 64 == 0 else 32 if Cin % 32 == 0 else 0
    if not bk or Cout % 192 or K * -(-Cin // bk) < 12:
        return 0
    return 4 if bk == 64 else 8


# (B, Cin, Cout, Lout, K) -> whether the wide kernel takes it
SHAPES = [
    # MSD layers 2-4 at the three scales (K 15, stride 4)
    ((64, 96, 192, 4096, 15), True), ((64, 96, 192, 1024, 15), True), ((64, 192, 384, 1024, 15), True),
    ((64, 192, 384, 256, 15), True), ((64, 384, 768, 256, 15), True), ((64, 384, 768, 64, 15), True),
    # MPD layers 2-4 (K 5, stride 4), periods 2 and 11
    ((128, 96, 192, 512, 5), True), ((704, 96, 192, 94, 5), True), ((128, 192, 384, 128, 5), True),
    ((704, 192, 384, 24, 5), True), ((128, 384, 768, 32, 5), True), ((704, 384, 768, 6, 5), True),
    # encoder convs of 1536 / 768 / 384 output channels
    ((32, 1536, 1536, 32, 3), True), ((32, 768, 1536, 64, 3), True), ((32, 384, 768, 64, 8), True),
    ((32, 192, 384, 256, 8), True),
    # short k: the first layers (64 im2col channels, K 1), 9 k-blocks, a 1536-wide output of 6 k-blocks
    ((64, 64, 384, 4096, 1), False), ((32, 192, 384, 1024, 3), False), ((32, 128, 1536, 32, 3), False),
    # widths that are not a multiple of 192, inputs that are not a multiple of 32
    ((32, 96, 96, 4096, 15), False), ((32, 768, 1024, 64, 15), False), ((32, 768, 128, 64, 3), False),
    ((16, 48, 192, 4096, 15), False), ((16, 16, 384, 4096, 15), False),
]


@pytest.fixture(scope="module")
def lib():
    from rave_b200 import _lib
    return _lib.load()


@pytest.mark.parametrize("shape,wide", SHAPES, ids=["-".join(map(str, s)) for s, _ in SHAPES])
def test_wide_stages_match_the_restated_rule(lib, shape, wide):
    got = lib.rave_conv1d_tc_wide_stages(*shape)
    assert got == restated(*shape)
    assert (got > 0) == wide


def test_the_discriminator_layers_keep_their_other_queries(lib):
    """The launches the wide kernel takes still report what conv_tc_kernel and the ping-pong kernel would run."""
    v = lib.rave_conv1d_tc_plan(64, 192, 384, 1024, 15)
    assert (v & 0xFFF, (v >> 12) & 0xFFF) == (128, 64)
    assert lib.rave_conv1d_tc_pp_fwd_stages(64, 192, 384, 1024, 15) == 5

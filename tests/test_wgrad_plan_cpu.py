"""Host-side plan of the weight-gradient launches (no GPU needed): rave_conv1d_tc_wgrad_splits equals the split-K
formula restated here, and rave_conv1d_tc_wgrad_plan reports the tile the launch runs and its ring depth, at the shapes
of the v2 training step and at the edge cases (one split, the 32-split cap, ragged channel counts, fewer CTAs than
SMs)."""
import math

import pytest

# (B, Cm, Lp, Cn, K) of the v2 step's weight-gradient launches (scripts/profile_layers.py) and the edge cases
SHAPES = [
    (64, 192, 4096, 384, 4), (128, 192, 2048, 96, 5), (704, 192, 373, 96, 5), (64, 384, 1024, 768, 4),
    (64, 768, 256, 1536, 4), (704, 384, 94, 192, 5), (448, 768, 37, 384, 5), (32, 32, 4096, 96, 7),
    (32, 96, 4096, 96, 1), (32, 96, 4096, 96, 3), (32, 192, 1024, 192, 3), (32, 384, 256, 384, 3),
    (32, 1536, 32, 768, 4), (32, 1536, 32, 128, 3), (128, 384, 2048, 64, 1), (448, 16, 37, 768, 1),
    (64, 16, 64, 768, 1), (32, 768, 64, 768, 1),
    (1, 64, 64, 64, 1),            # one chunk: one split
    (32, 96, 4096, 96, 1),         # 32-split cap
    (4, 40, 700, 24, 3), (8, 200, 300, 136, 2),    # ragged channel counts (multiples of 8, not of 32)
    (2, 64, 128, 64, 1),           # fewer CTAs than SMs
]


def old_splits(B, Cm, Lp, Cn, K):
    """The split-K formula of the weight-gradient launch, restated: 64-row chunks of BB batches x BL rows, 128-row
    tiles of Cm, 64- or 128-column tiles of Cn, enough slices for about one wave (two below 66 tiles), at most 32, at
    least 8 chunks per slice."""
    bl = 64
    while bl > Lp and bl > 8:
        bl //= 2
    n_chunks = math.ceil(Lp / bl) * math.ceil(B / (64 // bl))
    bn = 64 if Cn <= 64 else 128
    tiles = K * math.ceil(Cm / 128) * math.ceil(Cn / bn)
    s = math.ceil((132 if tiles >= 66 else 264) / tiles)
    s = min(s, 32, n_chunks // 8, n_chunks)
    return max(s, 1)


@pytest.fixture(scope="module")
def lib():
    from rave_b200 import _lib
    return _lib.load()


@pytest.mark.parametrize("shape", SHAPES)
def test_splits_match_the_restated_formula(lib, shape):
    assert lib.rave_conv1d_tc_wgrad_splits(*shape) == old_splits(*shape)


@pytest.mark.parametrize("shape", SHAPES)
def test_plan_reports_the_launched_tile(lib, shape):
    B, Cm, Lp, Cn, K = shape
    v = lib.rave_conv1d_tc_wgrad_plan(*shape)
    bn, bm, stages = v & 0xff, (v >> 8) & 0xff, v >> 16
    assert bn == (64 if Cn <= 64 else 128)      # the wgrad_tc_kernel<64 / 128> instance the launch names
    assert bm == 128
    # (2 P slabs + BLOCK_N / 64 Q slabs) of 8 KB per stage in a 200 KB ring, at most 6 stages
    assert stages == min(6, 200 * 1024 // ((2 + bn // 64) * 8192))


def test_edge_cases_are_covered(lib):
    splits = [lib.rave_conv1d_tc_wgrad_splits(*s) for s in SHAPES]
    assert 1 in splits and 32 in splits
    ctas = []
    for (B, Cm, Lp, Cn, K), s in zip(SHAPES, splits):
        v = lib.rave_conv1d_tc_wgrad_plan(B, Cm, Lp, Cn, K)
        ctas.append(K * s * math.ceil(Cm / ((v >> 8) & 0xff)) * math.ceil(Cn / (v & 0xff)))
    assert min(ctas) < 132

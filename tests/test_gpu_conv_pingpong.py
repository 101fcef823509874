"""GPU: the ping-pong input-gradient kernel (two MMA warpgroups on alternate tiles, epilogue from the accumulator
registers, LeakyReLU' mask / feature-matching partner rows / gradient skip loaded by TMA into shared memory).

It runs every conv launch with a LeakyReLU' mask (dact_src) whose only output is bf16.  Each launch is checked three
ways on the same bf16 operands: against the emulator (tests/tc_emulator.py), bit for bit against the same launch with
the fp32 stream also requested (which runs conv_tc_kernel: same MMA order, same fp32 epilogue sequence), and bit for bit
against a second launch of itself.  Output rows the launch does not own -- other phases, the pitch slack past Lout --
must keep the value they were pre-filled with.  Every case asserts the BLOCK_N / BLOCK_K instance it runs
(rave_conv1d_tc_plan) and that the ping-pong kernel takes it (rave_conv1d_tc_pp_stages); one test reads the kernel
names off the profiler.  Output widths 96 / 192 (BLOCK_N = 96) and 384 / 768 (BLOCK_N = 128), 96 and 192 input
channels (BLOCK_K = 32 and 64), K = 1 and 2, a ragged last time tile, short rows with several batches per tile and a
part-empty last batch group, and the phase rows of a transposed conv."""
import pytest
import torch

from tests import tc_emulator as E
from tests.conftest import rel_l2

pytestmark = pytest.mark.gpu

FILL = 7.0


def _instance(B, Cin, Cout, Lout, K, fm, res_bf16):
    """(BLOCK_N, BLOCK_K, ping-pong ring stages; 0 = the launch runs conv_tc_kernel)"""
    from rave_b200 import _lib
    lib = _lib.load()
    plan = lib.rave_conv1d_tc_plan(B, Cin, Cout, Lout, K)
    return plan & 0xFFF, (plan >> 12) & 0xFFF, lib.rave_conv1d_tc_pp_stages(B, Cin, Cout, Lout, K, int(fm != 0),
                                                                           int(res_bf16))


def _run(B, Cin, Cout, L, K=1, pad=(0, 0), *, res_bf16=False, fm=0, phases=None, slack=0, seed=0, bn=None):
    from rave_b200 import ops
    g = torch.Generator().manual_seed(seed)
    Lout = L + pad[0] + pad[1] - (K - 1)
    BN, BK, stages = _instance(B, Cin, Cout, Lout, K, fm, res_bf16)
    assert BK == (64 if Cin % 64 == 0 else 32) and (bn is None or BN == bn), (BN, BK)
    # conv_tc_kernel runs BLOCK_N = 96 at BLOCK_K = 64 (the ping-pong instance spills), and mask + partner rows + skip
    # at BLOCK_N = 128, BLOCK_K = 64 (the operand slots leave the ring one stage)
    fallback = BK == 64 and (BN == 96 or (BN == 128 and fm != 0 and res_bf16))
    assert (stages == 0) == fallback, (BN, BK, stages)
    assert stages == 0 or stages >= 2
    ors, oro = phases if phases else (1, 0)
    rows = Lout * ors + slack
    x = torch.randn(B, L, Cin, generator=g).bfloat16()
    wt = (torch.randn(K, Cout, Cin, generator=g) / (Cin * K) ** 0.5).bfloat16()
    full = torch.nn.functional.leaky_relu(torch.randn(2 * B if fm < 0 else B, rows, Cout, generator=g), 0.2).bfloat16()
    skip = torch.randn(B, rows, Cout, generator=g).bfloat16() if res_bf16 else None
    fm_d = torch.tensor([0.37, -0.21]) if fm else None
    kw = dict(stride=1, dil=1, pad=pad, act=0, slope=0.2, want_f32=False, want_act=False, Lout=Lout, Lin=L,
              out_rows=rows, out_row_stride=ors, out_row_offset=oro)

    def args(dev):
        mv = lambda v: v.to(dev) if v is not None else None
        f = mv(full)
        return dict(res_bf16=mv(skip), dact_src=f[B:] if fm < 0 else f, fm_partner=f[:B] if fm < 0 else None,
                    fm_d=mv(fm_d))

    ref = torch.full((B, rows, Cout), FILL, dtype=torch.bfloat16)
    E.conv1d_tc(x, wt, out_f32=None, out_act=ref, **args("cpu"), **kw)

    xc, wc, a = x.cuda(), wt.cuda(), args("cuda")

    def launch(with_f32=False):
        oa = torch.full((B, rows, Cout), FILL, dtype=torch.bfloat16, device="cuda")
        o32 = torch.full((B, rows, Cout), FILL, device="cuda") if with_f32 else None
        ops.conv1d_tc(xc, wc, out_f32=o32, out_act=oa, **a, **kw)
        return oa

    out, again, single = launch(), launch(), launch(with_f32=True)
    torch.cuda.synchronize()
    out, again, single = out.cpu(), again.cpu(), single.cpu()
    idx = torch.arange(Lout) * ors + oro
    other = torch.ones(rows, dtype=torch.bool)
    other[idx] = False
    assert rel_l2(out[:, idx].float(), ref[:, idx].float()) < 5e-3
    assert bool((out[:, other].float() == FILL).all()), "rows outside the launch's output rows were written"
    assert torch.equal(out.view(torch.int16), again.view(torch.int16)), "two launches of the same inputs differ"
    assert torch.equal(out[:, idx].view(torch.int16), single[:, idx].view(torch.int16)), \
        "differs from the single-warpgroup kernel"


# the input-gradient epilogues the engine issues: mask only, mask + gradient skip, fused feature-matching term of a
# [real; fake] batch (fm = 1) or of the fake half against the real rows stored before it (fm = -1), and all three
EPI = {
    "dact": dict(),
    "dact_res_bf16": dict(res_bf16=True),
    "fm_pos": dict(fm=1),
    "fm_neg": dict(fm=-1),
    "fm_pos_res_bf16": dict(fm=1, res_bf16=True),
}


BN = {96: 96, 192: 96, 384: 128, 768: 128}    # BLOCK_N of these widths once the launch has >= 132 M tiles


@pytest.mark.parametrize("cin,K", [(96, 1), (96, 2), (192, 2)])
@pytest.mark.parametrize("epi", list(EPI))
@pytest.mark.parametrize("cout", [96, 192, 384, 768])
def test_ragged_time_tile(cout, epi, cin, K):
    """Lout = 4500 is not a multiple of BL = 128 (4 x 36 = 144 M tiles), and the pitch has slack rows past Lout; 96 input
    channels run BLOCK_K = 32 (3 k-blocks per tap), 192 run BLOCK_K = 64."""
    _run(4, cin, cout, 4500 + K - 1, K=K, slack=5, seed=cout + K + cin, bn=BN[cout], **EPI[epi])


@pytest.mark.parametrize("epi", list(EPI))
@pytest.mark.parametrize("cout", [96, 192, 384, 768])
def test_short_rows_ragged_batch(cout, epi):
    """L = 20 -> BL = 32, four batches per tile; B = 530 leaves the last of 133 batch groups half empty, and the
    [real; fake] boundary at batch 265 falls inside a batch group."""
    _run(530, 96, cout, 21, K=2, seed=cout + 1, bn=BN[cout], **EPI[epi])


@pytest.mark.parametrize("oro", [1, 3])
@pytest.mark.parametrize("epi", ["dact", "dact_res_bf16", "fm_pos", "fm_pos_res_bf16"])
@pytest.mark.parametrize("cout", [192, 384])
def test_phase_rows(cout, epi, oro):
    """Phase oro of a stride-4 transposed conv: output row = l * 4 + oro; the other phases keep their contents."""
    _run(24, 96, cout, 300, K=3, pad=(1, 1), phases=(4, oro), slack=2, seed=cout + oro, bn=BN[cout], **EPI[epi])


@pytest.mark.parametrize("epi", ["dact", "fm_pos"])
def test_many_tiles_per_cta(epi):
    """2048 tiles of 128 x 96 over at most 132 CTAs: about 8 tiles per warpgroup, so the ring, the operand slots and the
    ordering barriers go through several phases."""
    _run(16, 96, 96, 16384, K=1, seed=11, bn=96, **EPI[epi])


def test_kernel_names():
    """The profiler sees conv_tc_pp_kernel run the input-gradient launch, and conv_tc_kernel run the same launch with
    the fp32 stream requested and the mask + partner rows + skip launch at BLOCK_N = 128, BLOCK_K = 64."""
    from torch.profiler import ProfilerActivity, profile
    from rave_b200 import ops

    def launch(B, Cin, Cout, L, fm, res_bf16, f32):
        x = torch.randn(B, L, Cin, device="cuda").bfloat16()
        wt = torch.randn(1, Cout, Cin, device="cuda").bfloat16()
        dact = torch.randn(B, L, Cout, device="cuda").bfloat16()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ops.conv1d_tc(x, wt, act=0, want_f32=False, want_act=True, Lout=L, dact_src=dact,
                          res_bf16=torch.randn(B, L, Cout, device="cuda").bfloat16() if res_bf16 else None,
                          fm_d=torch.tensor([0.37, -0.21], device="cuda") if fm else None,
                          out_f32=torch.empty(B, L, Cout, device="cuda") if f32 else None)
            torch.cuda.synchronize()
        return [e.name for e in prof.events() if "conv_tc" in e.name]

    pp = launch(4, 96, 96, 4500, True, True, False)
    assert any("conv_tc_pp_kernel<96, 32, true, true>" in n for n in pp) and not any("conv_tc_kernel" in n for n in pp), pp
    single = launch(4, 96, 96, 4500, True, True, True)
    assert any("conv_tc_kernel" in n for n in single) and not any("conv_tc_pp_kernel" in n for n in single), single
    full = launch(4, 192, 384, 4500, True, True, False)
    assert any("conv_tc_kernel<128, 64" in n for n in full) and not any("pp_kernel" in n for n in full), full

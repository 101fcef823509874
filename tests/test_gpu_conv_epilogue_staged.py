"""GPU: the conv epilogue that stages its bf16 output tile in shared memory and writes it with TMA tensor stores.

Every operand combination the engine issues, at the output widths it uses (Cout = 16, 48, 96, 192, 768), on tile
geometries whose edges the tensor-store clipping has to get right: time steps past Lout in the last tile, batches past B
in the last batch group of a short-sequence tile (BL < 128: several batches per tile), and the phase rows of a transposed
conv (out_row_stride > 1 with an offset).  Each launch is compared against the emulator (tests/tc_emulator.py) on the
same bf16 operands, and every output row the launch does not own -- other phases, the pitch slack past Lout -- must keep
the value it was pre-filled with."""
import pytest
import torch

from tests import tc_emulator as E
from tests.conftest import rel_l2

pytestmark = pytest.mark.gpu

FILL = 7.0          # pre-filled output value that rows outside [0, Lout) x phase must keep


def _plan(B, Cin, Cout, Lout, K):
    from rave_b200 import _lib
    return _lib.load().rave_conv1d_tc_plan(B, Cin, Cout, Lout, K)


def _run(B, Cin, Cout, L, K=1, pad=(0, 0), *, bias=True, res=False, res_bf16=False, dact=False, res_act=False, fm=0,
         want_f32=False, act=1, phases=None, slack=0, seed=0):
    from rave_b200 import ops
    g = torch.Generator().manual_seed(seed)
    Lout = L + pad[0] + pad[1] - (K - 1)
    ors, oro = phases if phases else (1, 0)
    rows = Lout * ors + slack
    x = torch.randn(B, L, Cin, generator=g).bfloat16()
    wt = (torch.randn(K, Cout, Cin, generator=g) / (Cin * K) ** 0.5).bfloat16()
    lrelu = lambda *s: torch.nn.functional.leaky_relu(torch.randn(*s, generator=g), 0.2).bfloat16()
    t = dict(bias=torch.randn(Cout, generator=g) if bias else None,
             res_cl=torch.randn(B, rows, Cout, generator=g) if res else None,
             res_bf16=torch.randn(B, rows, Cout, generator=g).bfloat16() if res_bf16 else None,
             res_act=lrelu(B, rows, Cout) if res_act else None)
    full = lrelu(2 * B if fm < 0 else B, rows, Cout) if (dact or fm) else None
    fm_d = torch.tensor([0.37, -0.21]) if fm else None
    kw = dict(stride=1, dil=1, pad=pad, act=act, slope=0.2, want_f32=False, want_act=False, Lout=Lout, Lin=L,
              out_rows=rows, out_row_stride=ors, out_row_offset=oro)

    def outs(dev):
        o32 = torch.full((B, rows, Cout), FILL, device=dev) if want_f32 else None
        oa = torch.full((B, rows, Cout), FILL, dtype=torch.bfloat16, device=dev)
        return o32, oa

    def args(dev):
        mv = lambda v: v.to(dev) if v is not None else None
        a = {k: mv(v) for k, v in t.items()}
        f = mv(full)
        a.update(dact_src=(f[B:] if fm < 0 else f) if f is not None else None, fm_partner=f[:B] if fm < 0 else None,
                 fm_d=mv(fm_d))
        return a

    r32, ra = outs("cpu")
    E.conv1d_tc(x, wt, out_f32=r32, out_act=ra, **args("cpu"), **kw)
    o32, oa = outs("cuda")
    ops.conv1d_tc(x.cuda(), wt.cuda(), out_f32=o32, out_act=oa, **args("cuda"), **kw)
    torch.cuda.synchronize()
    idx = torch.arange(Lout) * ors + oro
    other = torch.ones(rows, dtype=torch.bool)
    other[idx] = False
    assert rel_l2(oa[:, idx].float(), ra[:, idx].float()) < 5e-3          # bf16 rounding of the stored operand
    assert bool((oa[:, other].float() == FILL).all()), "rows outside the launch's output rows were written"
    if want_f32:
        assert rel_l2(o32[:, idx], r32[:, idx]) < 2e-5
        assert bool((o32[:, other] == FILL).all())


# operand combinations of the engine's launches: forward (bias -> LeakyReLU operand, optionally with the fp32 stream or
# a residual), the unit's second conv (skip recovered from its own operand), dgrads (LeakyReLU' mask, gradient skip,
# fused feature-matching term of a [real; fake] batch or of the fake half against its partner rows)
EPI = {
    "bias_act": dict(),
    "bias_f32_act": dict(want_f32=True),
    "res_f32_act": dict(res=True, want_f32=True),
    "res_act": dict(bias=False, res_act=True, act=0),
    "dact": dict(bias=False, dact=True, act=0),
    "dact_res_bf16": dict(bias=False, dact=True, res_bf16=True, act=0),
    "fm_pos": dict(bias=False, fm=1, act=0),
    "fm_neg": dict(bias=False, fm=-1, act=0),
}


@pytest.mark.parametrize("epi", list(EPI))
@pytest.mark.parametrize("cout", [16, 48, 96, 192, 768])
def test_ragged_time_tile(cout, epi):
    """Lout = 1000 is not a multiple of BL = 128, and the pitch has slack rows past Lout."""
    B = 4 if EPI[epi].get("fm", 0) > 0 else 3
    _run(B, 16, cout, 1000, slack=5, seed=cout, **EPI[epi])


@pytest.mark.parametrize("epi", list(EPI))
@pytest.mark.parametrize("cout", [16, 48, 96, 192, 768])
def test_short_rows_ragged_batch(cout, epi):
    """L = 20 -> BL = 32, four batches per tile; B = 10 (6 with the [real; fake] halves) leaves the last batch group
    part empty, and Lout = 20 leaves 12 time steps of every batch slot of a tile past Lout."""
    B = 6 if EPI[epi].get("fm", 0) > 0 else 10
    _run(B, 64, cout, 20, seed=cout + 1, **EPI[epi])


@pytest.mark.parametrize("oro", [1, 3])
@pytest.mark.parametrize("epi", ["bias_act", "bias_f32_act", "dact", "fm_pos"])
@pytest.mark.parametrize("cout", [48, 192])
def test_phase_rows(cout, epi, oro):
    """Phase oro of a stride-4 transposed conv: output row = l * 4 + oro; the other phases keep their contents."""
    B = 4 if EPI[epi].get("fm", 0) > 0 else 3
    _run(B, 32, cout, 300, K=3, pad=(1, 1), phases=(4, oro), slack=2, seed=cout + oro, **EPI[epi])


@pytest.mark.parametrize("cout", [16, 48, 96, 192, 768])
def test_short_k_plans_staged_output(cout):
    """One k-block per tile (first layers): the plan stages the bf16 output through shared memory."""
    v = _plan(64, 64, cout, 4096, 1)
    assert v & 0xFFF and (v >> 25) & 1

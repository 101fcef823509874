"""CPU: the launch checker (tests/launch_checker.py) passes a correct result and flags each planted defect.  The
"kernel" is the fp32 evaluation of tests/tc_emulator.py and the reference its float64 evaluation; the GPU twin
(tests/test_gpu_launch_replay.py) plants the same defects in the output of a real launch."""
import math

import pytest
import torch

from tests import launch_checker as lc
from tests import tc_emulator as emu


def conv_args(device, B=3, Cin=128, Cout=32, K=3, Lin=300, seed=0):
    """One phase (offset 1 of 2) of a phase-fused style launch: out rows 2 l + 1, a ragged last 128-row tile (Lin = 300),
    two 64-channel k-blocks per tap, bias, and slack rows past 2 Lout in the caller's zero-initialised output."""
    g = torch.Generator().manual_seed(seed)
    xa = torch.randn(B, Lin, Cin, generator=g).to(torch.bfloat16)
    wt = (torch.randn(K, Cout, Cin, generator=g) / math.sqrt(K * Cin)).to(torch.bfloat16)
    bias = 0.1 * torch.randn(Cout, generator=g)
    out_rows = 2 * Lin + 8
    out_f32 = torch.zeros(B, out_rows, Cout)
    a = dict(xa_cl=xa, wt=wt, bias=bias, res_cl=None, stride=1, dil=1, pad=(1, 1), act=0, slope=0.2, want_f32=False,
             want_act=False, out_f32=out_f32, out_act=None, out_rows=out_rows, out_row_stride=2, out_row_offset=1,
             Lout=Lin, res_bf16=None, dact_src=None, Lin=Lin, res_act=None, res_slope=0.2, fm_d=None, fm_partner=None,
             x3=False, act_cs=0)
    return {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in a.items()}


def wgrad_args(device, B=4, L=512, Cm=192, Cn=96, K=3, seed=1):
    g = torch.Generator().manual_seed(seed)
    P = torch.randn(B, L, Cm, generator=g).to(torch.bfloat16)
    Q = torch.randn(B, L, Cn, generator=g).to(torch.bfloat16)
    a = dict(P_cl=P, Q_cl=Q, K=K, stride=1, dil=2, pad_l=2, Lp=None, Lq=None, dbias=None)
    return {k: (v.to(device) if torch.is_tensor(v) else v) for k, v in a.items()}


def fm_args(device, Bh=2, Cin=64, Cout=32, K=3, L=200, seed=2):
    """The fake half of a fused feature-matching dgrad: out_act is the second half of the gradient buffer gx (its real
    half stays zero), fm_partner the real rows stored right before dact_src in one allocation."""
    g = torch.Generator().manual_seed(seed)
    xa = torch.randn(Bh, L, Cin, generator=g).to(torch.bfloat16).to(device)
    wt = (torch.randn(K, Cout, Cin, generator=g) / math.sqrt(K * Cin)).to(torch.bfloat16).to(device)
    dact = torch.randn(2 * Bh, L, Cout, generator=g).to(torch.bfloat16).to(device)
    gx = torch.zeros(2 * Bh, L, Cout, dtype=torch.bfloat16, device=device)
    return dict(xa_cl=xa, wt=wt, bias=None, res_cl=None, stride=1, dil=1, pad=(1, 1), act=0, slope=0.2, want_f32=False,
                want_act=False, out_f32=None, out_act=gx[Bh:], out_rows=0, out_row_stride=0, out_row_offset=0, Lout=L,
                res_bf16=None, dact_src=dact[Bh:], Lin=L, res_act=None, res_slope=0.2,
                fm_d=torch.tensor([0.25, -0.125], device=device), fm_partner=dact[:Bh], x3=False, act_cs=0)


def conv_bound(args):
    """The checker's elementwise bound of conv_args' launch (bias only: one epilogue term)."""
    n = args["wt"].shape[0] * args["xa_cl"].shape[2]
    with emu.compute(torch.float64):
        S, _ = emu.conv1d_tc(args["xa_cl"].abs(), args["wt"].abs(), None, None, 1, 1, args["pad"], want_f32=True,
                             Lout=args["Lout"], Lin=args["Lin"])
    return (n * 17 / 16 + 1) * lc.U23 * S + 2 * lc.U23 * args["bias"].double().abs()


def _rows(a):
    return emu.out_row_index(a["Lout"], a["out_row_stride"], a["out_row_offset"], a["xa_cl"].device)


def drop_kblock(a, out):
    """Tile (0, 0) loses the contribution of tap 1's second 64-channel k-block."""
    w = a["wt"].clone()
    w[1, :, 64:128] = 0
    with emu.compute(torch.float32):
        part, _ = emu.conv1d_tc(a["xa_cl"][:1], w, a["bias"], None, 1, 1, a["pad"], want_f32=True, Lout=a["Lout"],
                                Lin=a["Lin"])
    out[0][0, _rows(a)[:128], :16] = part[0, :128, :16].to(out[0].device)


def shift_phase(a, out):
    """The phase's rows land one position late."""
    idx = _rows(a)
    out[0][:, idx[1:]] = out[0][:, idx[:-1]].clone()


def unwritten_last_tile(a, out):
    """The last (ragged) 128-position tile of the last batch is never stored."""
    idx = _rows(a)
    out[0][-1, idx[(a["Lout"] // 128) * 128:]] = float("nan")


def slack_write(a, out):
    out[0][0, -1, 3] = 1.0


def bump_element(a, out):
    idx = _rows(a)
    b = conv_bound(a)
    out[0][1, idx[77], 5] += 4 * float(b[1, 77, 5])


def perturb_tile(a, out):
    """Tile (0, 0) moved by half the elementwise bound with random signs: inside the bound, caught per tile."""
    idx = _rows(a)[:128]
    b = conv_bound(a)[0, :128, :16]
    sign = (torch.randint(0, 2, b.shape, generator=torch.Generator().manual_seed(5)).double() * 2 - 1).to(b.device)
    out[0][0, idx, :16] += (0.5 * b * sign).to(out[0].device, out[0].dtype)


def write_real_half(a, out):
    """A store into the real half of the gradient buffer, outside the out_act view."""
    t = out[1]
    full = torch.empty(0, dtype=t.dtype, device=t.device).set_(t.untyped_storage(), 0, (t.untyped_storage().nbytes() // 2,),
                                                                (1,))
    full[5] = 1.0


def write_partner_rows(a, out):
    """A store into the partner (real) rows of dact_src, an input the launch only reads."""
    a["fm_partner"][0, 0, 0] += 1


def drop_split(a, dwt):
    """The slice carrying the most weight is lost (zero partial tile)."""
    s = int(dwt.double().reshape(dwt.shape[0], -1).norm(dim=1).argmax())
    dwt[s] = 0


# name -> (mutation, the check that must flag it)
CONV_MUTATIONS = {"kblock_dropped": (drop_kblock, "bound"), "phase_rows_shifted": (shift_phase, "bound"),
                  "last_partial_tile_unwritten": (unwritten_last_tile, "coverage"),
                  "slack_row_written": (slack_write, "outside"), "element_off_by_4x_bound": (bump_element, "bound"),
                  "tile_within_bound_perturbed": (perturb_tile, "tile")}
FM_MUTATIONS = {"real_half_written": (write_real_half, "outside"),
                "partner_rows_written": (write_partner_rows, "input")}
WGRAD_MUTATIONS = {"wgrad_split_dropped": (drop_split, "tile")}   # one of 32 splits can stay under the bound


def emulated_conv(**a):
    with emu.compute(torch.float32):
        return emu.conv1d_tc(**a)


def emulated_wgrad(**a):
    with emu.compute(torch.float32):
        return emu.conv1d_tc_wgrad(**a)


def run_case(fn, name, args, mutate):
    ck = lc.LaunchChecker("checker self-test", max_failures=1000)
    ck.checked_call(name, fn, args, mutate)
    return ck


def flagged_by(ck, kind, mutation):
    """The mutation was flagged, by the named check (tile_within_bound_perturbed: by the tile check alone)."""
    kinds = {f.split(":", 1)[0] for f in ck.failures}
    assert kind in kinds, f"{mutation} was not flagged by the {kind} check (flagged by: {sorted(kinds)})"
    if mutation == "tile_within_bound_perturbed":
        assert kinds == {"tile"}, kinds
    return f"{mutation}: flagged -- {[f for f in ck.failures if f.startswith(kind)][0][:200]}"


def test_clean_conv_and_wgrad_pass():
    for fn, name, args in ((emulated_conv, "conv1d_tc", conv_args("cpu")), (emulated_conv, "conv1d_tc", fm_args("cpu")),
                           (emulated_wgrad, "conv1d_tc_wgrad", wgrad_args("cpu"))):
        ck = run_case(fn, name, args, None)
        assert not ck.failures, ck.failures
        st = ck.records[-1][2]
        print(f"{name}: worst bound ratio {st.ratio:.3g}, worst tile {st.tile:.3g} of its limit")


@pytest.mark.parametrize("mutation", sorted(CONV_MUTATIONS) + sorted(FM_MUTATIONS) + sorted(WGRAD_MUTATIONS))
def test_planted_defect_is_flagged(mutation):
    if mutation in CONV_MUTATIONS:
        (fn, kind), ck_args = CONV_MUTATIONS[mutation], (emulated_conv, "conv1d_tc", conv_args("cpu"))
    elif mutation in FM_MUTATIONS:
        (fn, kind), ck_args = FM_MUTATIONS[mutation], (emulated_conv, "conv1d_tc", fm_args("cpu"))
    else:
        (fn, kind), ck_args = WGRAD_MUTATIONS[mutation], (emulated_wgrad, "conv1d_tc_wgrad", wgrad_args("cpu"))
    print(flagged_by(run_case(*ck_args, fn), kind, mutation))


def test_emulator_default_is_fp32():
    """Outside compute(...) the emulator keeps its fp32 semantics (tests/test_engine_cpu.py relies on them)."""
    a = conv_args("cpu")
    out, _ = emu.conv1d_tc(a["xa_cl"], a["wt"], a["bias"], None, 1, 1, a["pad"], want_f32=True, Lout=a["Lout"])
    assert out.dtype == torch.float32
    with emu.compute(torch.float64):
        out64, _ = emu.conv1d_tc(a["xa_cl"], a["wt"], a["bias"], None, 1, 1, a["pad"], want_f32=True, Lout=a["Lout"])
    assert out64.dtype == torch.float64 and emu.COMPUTE_DTYPE == torch.float32
    assert (out.double() - out64).abs().max() < 1e-4


def test_first_layer_cin_emulation_is_adjoint():
    """im2col_cin / gather_cin are adjoint: <im2col(x), P> == <x, gather(P)>."""
    g = torch.Generator().manual_seed(2)
    Bs, cin, T, K, stride, pad_l, period = 2, 2, 90, 5, 3, 2, 3
    Lin = -(-T // period)
    Lout = (Lin + 2 * pad_l - K) // stride + 1
    x = torch.randn(Bs, cin, T, generator=g, dtype=torch.float64)
    with emu.compute(torch.float64):
        saved = emu.OPERAND_DTYPE
        emu.OPERAND_DTYPE = torch.float64
        try:
            X = emu.im2col_cin(x, Lin, Lout, Lout + 3, K, stride, pad_l, period)
            P = torch.randn(X.shape, generator=g, dtype=torch.float64)
            P[:, Lout:] = 0
            dx = emu.gather_cin(P, (Bs, cin, T), Lin, Lout, K, stride, pad_l, period)
        finally:
            emu.OPERAND_DTYPE = saved
    assert X.shape[-1] == 16
    assert abs(float((X * P).sum() - (x * dx).sum())) < 1e-9

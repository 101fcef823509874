"""Algorithmic work of the library's launches: FLOPs and bytes per C-ABI call from its integer arguments (the
formulas of DESIGN.md section 5: every tensor a launch must read or write, once; weights once).

Used by bench.py (`roofline`, `step_roofline`) together with `_lib.PROFILE`, which logs
(entry point, integer arguments, pointer-presence string, milliseconds) for every call."""
from typing import Optional, Tuple


def conv_fwd_cost(ints, ptrs, x3: bool = False) -> Tuple[float, float]:
    """rave_conv1d_tc_fwd(xa, wt, bias, res, res_bf16, dact_src, res_act, [res_slope], out_f32, out_act, B, Cin, Lin,
    in_pitch, Cout, Lout, K, stride, dil, pad_l, ...).  ptrs: one char per pointer argument ('P' = non-null)."""
    Bc, Cin, Lin, pitch, Cout, Lout, K = ints[:7]
    mult = 3.0 if x3 else 1.0
    asz = 4.0 if x3 else 2.0                     # bytes per operand element ([hi | lo] pairs in the split mode)
    fl = 2.0 * Bc * Lout * Cout * Cin * K * mult
    by = asz * Bc * Lin * Cin + asz * K * Cout * Cin
    if x3:      # xa wt bias res res_act out_f32 out_act
        names = ("xa", "wt", "bias", "res", "res_act", "out_f32", "out_act")
    else:       # xa wt bias res res_bf16 dact res_act out_f32 out_act
        names = ("xa", "wt", "bias", "res", "res_bf16", "dact", "res_act", "out_f32", "out_act")
    have = {n: (i < len(ptrs) and ptrs[i] == "P") for i, n in enumerate(names)}
    rows = Bc * Lout * Cout
    if have.get("out_f32"):
        by += 4.0 * rows
    if have.get("out_act"):
        by += asz * rows
    if have.get("res"):
        by += 4.0 * rows
    if have.get("res_bf16"):
        by += 2.0 * rows
    if have.get("dact"):
        by += 2.0 * rows
    if have.get("res_act"):
        by += asz * rows
    # fused feature-matching gradient: the partner rows of the other batch half (last pointer before the stream)
    if not x3 and len(ptrs) >= 11 and ptrs[9] == "P":
        by += 2.0 * rows
    return fl, by


def wgrad_cost(ints) -> Tuple[float, float]:
    Bc, Cm, Lp, pp, Cn, Lq, qp, K = ints[:8]
    return 2.0 * Bc * Lp * Cm * Cn * K, 2.0 * Bc * (Lp * Cm + Lq * Cn) + 4.0 * K * Cm * Cn


def launch_cost(name: str, ints, ptrs) -> Optional[Tuple[float, float]]:
    """(flops, bytes) of one call, or None for entry points without a formula here (small elementwise kernels)."""
    if name == "rave_conv1d_tc_fwd":
        return conv_fwd_cost(ints, ptrs)
    if name == "rave_conv1d_tc_fwd_x3":
        return conv_fwd_cost(ints, ptrs, x3=True)
    if name == "rave_conv1d_tc_wgrad":
        return wgrad_cost(ints)
    if name in ("rave_pqmf_analysis_fwd", "rave_pqmf_analysis_fast"):
        B, T = ints[0], ints[1]
        return 2.0 * B * T * 66, 8.0 * B * T          # factorised form: 66 MACs per sample; x in + 16 bands out
    if name in ("rave_pqmf_synthesis_fwd", "rave_pqmf_synthesis_fast"):
        B, L = ints[0], ints[1]
        return 2.0 * B * 16 * L * 66, 8.0 * B * 16 * L
    return None


def roofline_seconds(flops: float, byts: float, peak_flops: float, peak_bw: float) -> float:
    return max(flops / peak_flops, byts / peak_bw)

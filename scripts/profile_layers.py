"""Per-launch picture of the benchmarked training step (v2, B = 32 x 65536, bf16 engine): every distinct tensor-core
conv / weight-gradient launch of one G-step and one D-step, re-timed alone over rotating buffers larger than L2.

    python scripts/profile_layers.py [--batch 32] [--json OUT.json]

One eager G-step and one eager D-step run with `_lib.PROFILE` set, which only serves to collect the launch shapes and
their call counts (its milliseconds also hold the host-side tensor-map encode, so they are not used as kernel times).
Each shape is then captured into a CUDA graph and replayed (scripts/_timing.graph_time_us).  Per shape the table gives
the microseconds per launch, the per-step total (3 G-steps : 1 D-step, as bench.py times them), the algorithmic GFLOP
and MB of rave_b200/roofline.py, which of the two bounds the launch and the fraction of that data-sheet roofline
reached.  The whole-step CUDA graph is timed as well, so the share of the step the listed launches hold can be read
off directly.  The card name and power limit are printed with the numbers."""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

L2_BYTES = 50 * 2 ** 20


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:      # the numbers are still printed; the card line says why it is missing
        return f"unknown ({type(e).__name__})"


def n_sets(set_bytes):
    """Buffer sets to rotate so that consecutive launches never find their operands in L2."""
    return max(2, min(16, math.ceil(2 * L2_BYTES / max(set_bytes, 1))))


def fwd_runner(torch, ops, ints, ptrs):
    """fn(i) issuing the rave_conv1d_tc_fwd launch of a PROFILE record on buffer set i (same operands present).
    The decoding of the record (integer and pointer order of rave_conv1d_tc_fwd, see ops.conv1d_tc) is the same as in
    bench.dominant_launch_roofline: the two change together when that argument list does."""
    Bc, Cin, Lin, pitch, Cout, Lout, K, stride, dil, pad_l, act, out_rows, ors, oro, fm_bh = ints[:15]
    have = [c == "P" for c in ptrs]
    rows = out_rows if out_rows else Lout
    fm = have[9]
    fm_half = fm and fm_bh < 0            # fake half only: the partner rows are stored right before it
    g = torch.Generator(device="cuda").manual_seed(0)
    mk = lambda *s: torch.randn(*s, device="cuda", generator=g).bfloat16()
    set_bytes = 2 * Bc * pitch * Cin + Bc * rows * Cout * (4 * (have[3] + have[7]) + 2 * (have[4] + have[5] + have[6] + have[8]))
    nb = n_sets(set_bytes)
    wt = (torch.randn(K, Cout, Cin, device="cuda", generator=g) * 0.02).bfloat16()
    bias = torch.randn(Cout, device="cuda") if have[2] else None
    bufs = []
    for _ in range(nb):
        b = dict(x=mk(Bc, pitch, Cin))
        if Lin < pitch:
            b["x"][:, Lin:] = 0
        b["res"] = torch.randn(Bc, rows, Cout, device="cuda") if have[3] else None
        b["res_bf16"] = mk(Bc, rows, Cout) if have[4] else None
        b["dact"] = mk(2 * Bc if fm_half else Bc, rows, Cout) if have[5] else None
        b["res_act"] = mk(Bc, rows, Cout) if have[6] else None
        b["o32"] = torch.empty(Bc, rows, Cout, device="cuda") if have[7] else None
        b["oa"] = torch.empty(Bc, rows, Cout, device="cuda", dtype=torch.bfloat16) if have[8] else None
        bufs.append(b)
    fm_d = torch.tensor([1e-3, 2e-3], device="cuda") if fm else None

    def run(i):
        b = bufs[i % nb]
        d = b["dact"][Bc:] if (b["dact"] is not None and fm_half) else b["dact"]
        ops.conv1d_tc(b["x"], wt, bias, b["res"], stride, dil, (pad_l, 0), act, 0.2, want_f32=False, want_act=False,
                      out_f32=b["o32"], out_act=b["oa"], out_rows=out_rows, out_row_stride=ors, out_row_offset=oro,
                      Lout=Lout, Lin=Lin, res_bf16=b["res_bf16"], dact_src=d, res_act=b["res_act"], fm_d=fm_d,
                      fm_partner=b["dact"][:Bc] if fm_half else None)
    return run, nb


def wgrad_runner(torch, ops, ints, ptrs):
    Bc, Cm, Lp, pp, Cn, Lq, qp, K, stride, dil, pad_l = ints[:11]
    g = torch.Generator(device="cuda").manual_seed(0)
    nb = n_sets(2 * Bc * (pp * Cm + qp * Cn))
    bufs = []
    for _ in range(nb):
        P = torch.randn(Bc, pp, Cm, device="cuda", generator=g).bfloat16()
        Q = torch.randn(Bc, qp, Cn, device="cuda", generator=g).bfloat16()
        Q[:, Lq:] = 0
        bufs.append((P, Q))
    db = torch.zeros(Cm, device="cuda") if ptrs[3] == "P" else None

    def run(i):
        P, Q = bufs[i % nb]
        ops.conv1d_tc_wgrad(P, Q, K, stride, dil, pad_l, Lp=Lp, Lq=Lq, dbias=db)
    return run, nb


def instance(lib, name, ints, ptrs):
    """Kernel of a launch; conv launches the ping-pong kernel takes are marked ` pp` and its ring stages, those the wide
    kernel (128 x 192 tiles) takes `wide<192,BLOCK_K> s` and its ring stages, weight-gradient launches carry their tile
    (rows of Cm x columns of Cn), split-K slices, CTAs and waves of 132 SMs."""
    if name == "rave_conv1d_tc_fwd":
        B, Cin, Cout, Lout, K, act = ints[0], ints[1], ints[4], ints[5], ints[6], ints[10]
        v = lib.rave_conv1d_tc_plan(B, Cin, Cout, Lout, K)
        bias, res, res_bf16, dact, res_act, o32, oa, fm = [c == "P" for c in ptrs[2:10]]   # order of fwd_runner
        stages = 0
        if oa and not (res or res_act or o32):
            if dact and not bias and act == 0:
                stages = lib.rave_conv1d_tc_pp_stages(B, Cin, Cout, Lout, K, int(fm), int(res_bf16))
            elif not (dact or res_bf16 or fm):
                wide = lib.rave_conv1d_tc_wide_stages(B, Cin, Cout, Lout, K)
                if wide:
                    return f"wide<192,{64 if Cin % 64 == 0 else 32}> s{wide}"
                stages = lib.rave_conv1d_tc_pp_fwd_stages(B, Cin, Cout, Lout, K)
        return f"conv<{v & 0xfff},{(v >> 12) & 0xfff}>" + (f" pp{stages}" if stages else "")
    if name == "rave_conv1d_tc_wgrad":
        Bc, Cm, Lp, pp, Cn = ints[:5]
        K = ints[7]
        s = lib.rave_conv1d_tc_wgrad_splits(Bc, Cm, Lp, Cn, K)
        v = lib.rave_conv1d_tc_wgrad_plan(Bc, Cm, Lp, Cn, K)
        bn, bm = v & 0xff, (v >> 8) & 0xff
        items = K * s * math.ceil(Cm / bm) * math.ceil(Cn / bn)
        return f"wgrad<{bn}> {bm}x{bn} x{s} {items}/{math.ceil(items / 132)}w"
    return name


def step_graph_ms(torch, model, x, steps=8):
    from rave_b200.graphs import GraphedTrainer
    tr = GraphedTrainer(model, x)
    for i in range(4):
        tr.step(x, i)
        model.on_train_batch_end()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        tr.step(x, i)
        model.on_train_batch_end()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--json", default=None, help="also write the table as JSON here")
    args = ap.parse_args()

    import torch
    import bench
    import rave_b200
    from rave_b200 import _lib, configs, ops
    from _timing import graph_time_us

    rave_b200.set_precision("bf16")
    pk = bench.peaks()
    peak_f, peak_b = pk["bf16_tflops"] * 1e12, pk["hbm_gbs"] * 1e9
    torch.manual_seed(0)
    model = configs.build_rave("v2", sampling_rate=bench.SR).cuda().train()
    model.warmed_up = True
    x = bench.synthetic_batch(args.batch).cuda()
    step_ms = step_graph_ms(torch, model, x)          # captured first, as bench.py does
    prof = bench.profile_step(torch, model, x, pk)
    lib = _lib.load()

    rows = {}
    for tag in ("G", "D"):
        for (name, ints, ptrs), (cnt, _ms, _r, cost) in prof[tag]["shapes"].items():
            r = rows.setdefault((name, ints, ptrs), dict(G=0, D=0, cost=cost))
            r[tag] += cnt
    table = []
    for (name, ints, ptrs), r in rows.items():
        if name == "rave_conv1d_tc_fwd":
            run, nb = fwd_runner(torch, ops, ints, ptrs)
        elif name == "rave_conv1d_tc_wgrad":
            run, nb = wgrad_runner(torch, ops, ints, ptrs)
        else:
            print(f"# not re-timed: {name} {ints}", flush=True)
            continue
        us = graph_time_us(run, n=nb * max(1, math.ceil(12 / nb)), replays=5)
        fl, by = r["cost"]
        t_tc, t_hbm = fl / peak_f, by / peak_b
        per_step = (3 * r["G"] + r["D"]) / 4
        table.append(dict(entry=name, instance=instance(lib, name, ints, ptrs), ints=list(ints), ptrs=ptrs, G=r["G"], D=r["D"],
                          us=us, us_per_step=per_step * us, gflop=fl / 1e9, mb=by / 1e6,
                          bound="tensor" if t_tc >= t_hbm else "hbm", frac=max(t_tc, t_hbm) * 1e6 / us))
    table.sort(key=lambda e: -e["us_per_step"])
    total = sum(e["us_per_step"] for e in table) / 1e3
    print(f"card: {card()}  (peaks: {pk['source']}: {pk['bf16_tflops']:.0f} TFLOP/s bf16, {pk['hbm_gbs']:.0f} GB/s)")
    print(f"whole-step graph: {step_ms:.2f} ms / step (3 G : 1 D); listed conv + wgrad launches: {total:.2f} ms / step "
          f"= {100 * total / step_ms:.1f} %")
    print(f"{'instance':22s} {'G':>3s} {'D':>3s} {'us':>8s} {'us/step':>9s} {'GFLOP':>7s} {'MB':>8s} {'bound':>6s} "
          f"{'frac':>5s}  shape")
    for e in table:
        print(f"{e['instance']:22s} {e['G']:3d} {e['D']:3d} {e['us']:8.1f} {e['us_per_step']:9.1f} {e['gflop']:7.1f} "
              f"{e['mb']:8.1f} {e['bound']:>6s} {e['frac']:5.2f}  {e['entry']} {tuple(e['ints'][:11])} {e['ptrs']}",
              flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card(), step_ms=step_ms, listed_ms=total, peaks=pk, launches=table), f, indent=1)


if __name__ == "__main__":
    main()

"""Unit shapes and generator of the v2_nopqmf configuration (rave/configs/v2_nopqmf.gin) at the bench shape B = 32 x
65536 samples.

    python scripts/time_nopqmf.py [--batch 32] [--json OUT.json]

1. Every Residual(DilatedUnit) shape of the configuration (encoder C = 64 .. 512 over the 16-band PQMF rows, generator
   C = 512 .. 64 up to the audio rate), training form (a1 kept for the backward): the fused kernel
   (rave_dilated_unit_tc_fwd, one launch) against the two per-layer launches the engine runs with engine.FUSE_UNITS off,
   alternated in one process, each captured once into a CUDA graph and replayed (scripts/_timing.py).
   Algorithmic work: GFLOP = 2 B L C^2 (3 + 1); GB fused = bf16 operand in + a1 out + operand out (+ 8 C^2 weights),
   two launches = that + a1 read back + the skip operand read again.  The bound is the larger of GFLOP over 989 TFLOP/s
   (bf16 dense) and GB over 3.35 TB/s; "roofline" is the bound's time over the measured time.
2. The generator's bf16 forward + backward (the whole capacity-64 raw-waveform generator, one engine chain), timed with
   CUDA events.
The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

PEAK, BW = 989e12, 3.35e12
T = 65536


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:          # noqa: BLE001  (the numbers are still printed)
        return f"unknown ({e})"


def unit_shapes():
    """(where, C, L, dilations) of every unit: encoder over T / 16 PQMF rows, ratios [4, 4, 4, 2]; generator ratios
    [8, 8, 8, 4] reversed, from the latent rate T / 2048 up (v2_nopqmf.gin:15-20, 45-64)."""
    dils = [[1, 3, 9], [1, 3, 9], [1, 3, 9], [1, 3]]
    out = []
    C, L = 64, T // 16
    for r, d in zip([4, 4, 4, 2], dils):
        out.append(("enc", C, L, d))
        C, L = C * 2, L // r
    C, L = 64 * 16, T // 2048
    for r, d in zip([4, 8, 8, 8], dils[::-1]):
        C, L = C // 2, L * r
        out.append(("gen", C, L, d))
    return out


def algo(B, C, L, fused):
    flop = 2.0 * B * L * C * C * 4
    act = 2.0 * B * L * C
    gb = (3 * act + 8 * C * C) if fused else (5 * act + 8 * C * C)
    return flop / 1e9, gb / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    from _timing import graph_time_us
    import rave_b200
    from rave_b200 import configs, ops
    assert torch.cuda.is_available(), "time_nopqmf.py measures on the GPU"
    B = args.batch
    dev = card()
    print("card:", dev)
    torch.manual_seed(0)
    rows = []
    for where, C, L, dils in unit_shapes():
        for dil in dils:
            sets = []
            for _ in range(2):
                xa = (torch.randn(B, L, C, device="cuda") * 0.5).to(torch.bfloat16)
                sets.append((xa, torch.empty_like(xa), torch.empty_like(xa), torch.empty(B, L, C, device="cuda",
                                                                                         dtype=torch.bfloat16)))
            w3t = (torch.randn(3, C, C, device="cuda") / (3 * C) ** 0.5).to(torch.bfloat16)
            w1t = (torch.randn(1, C, C, device="cuda") / C ** 0.5).to(torch.bfloat16)

            def two(i):
                xa, a1, out, _ = sets[i % 2]
                ops.conv1d_tc(xa, w3t, None, None, 1, dil, (dil, dil), ops.ACT_LEAKY, 0.2, want_f32=False,
                              want_act=False, out_act=a1, Lout=L, Lin=L)
                ops.conv1d_tc(a1, w1t, None, None, 1, 1, (0, 0), ops.ACT_LEAKY, 0.2, want_f32=False, want_act=False,
                              out_act=out, Lout=L, Lin=L, res_act=xa, res_slope=0.2)

            def fused(i):
                xa, a1, out, _ = sets[i % 2]
                a1_, _, _ = ops.dilated_unit_tc(xa, w3t, w1t, dil, dil, 0.2, 0.2, ops.ACT_LEAKY, 0.2, want_a1=True,
                                                out_act=out)
            has_fused = ops.dilated_unit_tc_supported(C, L)
            t2, tf = [], []
            for _ in range(3):                      # alternate the two forms
                t2.append(graph_time_us(two, n=10, replays=5))
                if has_fused:
                    tf.append(graph_time_us(fused, n=10, replays=5))
            r = dict(where=where, C=C, L=L, dil=dil, two_us=min(t2), fused_us=min(tf) if tf else None)
            for arm, fz in (("two", False), ("fused", True)):
                gf, gb = algo(B, C, L, fz)
                t = r[f"{arm}_us"]
                bound = max(gf * 1e9 / PEAK, gb * 1e9 / BW) * 1e6
                r[f"{arm}_gflop"], r[f"{arm}_gb"] = gf, gb
                r[f"{arm}_bound"] = "flop" if gf * 1e9 / PEAK > gb * 1e9 / BW else "hbm"
                r[f"{arm}_roofline"] = (bound / t) if t else None
            rows.append(r)
            f = f"{r['fused_us']:9.1f}" if r["fused_us"] else "      n/a"
            fr = f"{r['fused_roofline']:.2f}" if r["fused_us"] else " n/a"
            print(f"{where} C={C:4d} L={L:6d} dil={dil}: two-launch {r['two_us']:9.1f} us ({r['two_gb']:.3f} GB, "
                  f"{r['two_gflop']:.1f} GFLOP, {r['two_bound']}-bound, roofline {r['two_roofline']:.2f}) | fused {f} us "
                  f"({r['fused_gb']:.3f} GB, {r['fused_bound']}-bound, roofline {fr})", flush=True)
            del sets
    # ---- the generator's bf16 forward + backward
    rave_b200.set_precision("bf16")
    try:
        _, _, dec = configs.make_autoencoder("v2_nopqmf")
        dec.cuda().train()
        assert dec.net._tc_plan() is not None
        z = torch.randn(B, 128, T // 2048, device="cuda", requires_grad=True)
        gen = {}
        for fuse in (True, False, True, False):
            from rave_b200 import engine
            engine.FUSE_UNITS = fuse
            for _ in range(2):
                dec(z).square().mean().backward()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                dec(z).square().mean().backward()
            e1.record()
            torch.cuda.synchronize()
            gen.setdefault(fuse, []).append(e0.elapsed_time(e1) / 5)
        engine.FUSE_UNITS = True
    finally:
        rave_b200.set_precision("fp32")
    print(f"generator bf16 fwd+bwd B={B}x{T}: fused units {min(gen[True]):.2f} ms, two launches "
          f"{min(gen[False]):.2f} ms  (runs {gen})")
    res = dict(card=dev, batch=B, units=rows, generator_ms={"fused": gen[True], "two_launch": gen[False]})
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""Sampling from the latent prior (prior_v1.gin on a full-size v2 RAVE) on the device.

    python scripts/time_prior_sample.py [--latent-size 16] [--frames 1024] [--dense-frames 128] [--json OUT.json]

1. Prior.sample (cached, one library call): time per generated frame for B = 1 and B = 8 at --frames frames.
2. Prior.generate (the reference's dense loop on the stacked one-hot, O(T^2)): time per frame at --dense-frames frames.
3. Prior.decode_classes (classes -> latent in one kernel, then the RAVE decoder in bf16) of the B = 8 sample.
4. The weight bytes one frame reads, from the parameter shapes, and the time they take at the data sheet's 3.35 TB/s
   (a floor for the per-frame time; 78 MB does not fit the 50 MB L2).
The card name and power limit are read in the same run.  Times are host clocks around work that ends in a device
synchronise, after one warm-up call of the same shape."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:          # noqa: BLE001  (the numbers are still printed)
        return f"unknown ({e})"


def timed(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--latent-size", type=int, default=16)
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--dense-frames", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    import rave_b200
    from rave_b200 import configs

    if not torch.cuda.is_available():
        raise SystemExit("time_prior_sample.py needs a CUDA device")
    D = a.latent_size
    res = dict(card=card(), latent_size=D, frames=a.frames, dense_frames=a.dense_frames)
    print("card:", res["card"])
    torch.manual_seed(0)
    prior = configs.build_prior(configs.build_rave("v2"), latent_size=D).cuda()
    R = prior.quantized_normal.resolution
    last = prior.residuals[-1].rconv           # its output is unused, so the sampler never reads it
    n_param = sum(p.numel() for p in prior._trained_parameters()) - last.weight.numel() - last.bias.numel()
    res["weight_params"] = n_param
    res["weight_bytes_per_frame"] = 4 * n_param
    res["hbm_floor_us_per_frame"] = 4 * n_param / HBM_BYTES_PER_S * 1e6
    print(f"weights per frame: {n_param} fp32 parameters = {4 * n_param / 1e6:.1f} MB, "
          f"{res['hbm_floor_us_per_frame']:.1f} us at 3.35 TB/s")

    cls8 = None
    for B in (1, 8):
        prefix = torch.randint(0, R, (B, 1, D), dtype=torch.int32, device="cuda")
        u = torch.rand(B, a.frames, D, device="cuda")
        out = {}

        def run():
            out["cls"] = prior.sample(prefix, a.frames, uniform=u)
        s = timed(run, a.reps)
        per = s / (a.frames - 1) * 1e6
        res[f"sample_B{B}_us_per_frame"] = per
        print(f"sample B={B}: {s * 1e3:.2f} ms for {a.frames} frames = {per:.1f} us/frame")
        if B == 8:
            cls8 = out["cls"]

    for B in (1, 8):
        x0 = torch.randint(0, R, (B, D, a.dense_frames), device="cuda")
        one_hot = prior.quantized_normal.to_stack_one_hot(x0)
        s = timed(lambda: prior.generate(one_hot.clone()), 1)
        per = s / (a.dense_frames - 1) * 1e6
        res[f"generate_B{B}_us_per_frame"] = per
        print(f"dense generate B={B}: {s * 1e3:.1f} ms for {a.dense_frames} frames = {per:.1f} us/frame")

    rave_b200.set_precision("bf16")
    try:
        s = timed(lambda: prior.decode_classes(cls8), a.reps)
    finally:
        rave_b200.set_precision("fp32")
    res["decode_classes_B8_ms"] = s * 1e3
    print(f"decode_classes B=8, {a.frames} frames (bf16 decoder): {s * 1e3:.2f} ms")
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

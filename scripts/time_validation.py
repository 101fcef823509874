"""The validation pass on the device: v2 at 48 kHz, batches of 8 x 131072 samples (scripts/train.py's defaults).

    python scripts/time_validation.py [--batch 8] [--samples 131072] [--batches 200] [--json OUT.json]

1. ms per RAVE.validation_step (encode, reparametrise, decode, fused full-band spectral distance), in bf16 and fp32.
2. us per rave_latent_moments call on one batch's posterior means ([8, 128, 64], the mean half read in place).
3. The epoch-end latent analysis (core.latent_analysis) over 200 such batches at D = 128, and the same analysis done the
   reference's way on the same means (torch.cat -> .cpu() -> sklearn PCA(128).fit, rave/model.py:464-479).
The card name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from time_prior import card  # noqa: E402


def events_ms(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--samples", type=int, default=131072)
    ap.add_argument("--batches", type=int, default=200)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import numpy as np
    import torch
    import rave_b200
    from rave_b200 import configs, core, ops

    if not torch.cuda.is_available():
        raise SystemExit("time_validation.py measures the device: no CUDA device found")
    res = {"card": card(), "batch": a.batch, "samples": a.samples}
    torch.manual_seed(0)
    m = configs.build_rave("v2", sampling_rate=48000).cuda().eval()
    x = (0.5 * torch.randn(a.batch, 1, a.samples, device="cuda")).clamp(-1, 1)
    for precision in ("bf16", "fp32"):
        rave_b200.set_precision(precision)
        try:
            for i in range(3):
                m.validation_step(x, i)
            res[f"validation_step_ms_{precision}"] = events_ms(lambda: m.validation_step(x, 0), 20)
        finally:
            rave_b200.set_precision("fp32")
        print(f"validation_step ({precision}): {res[f'validation_step_ms_{precision}']:.2f} ms")

    D = m.latent_size
    _, mean = m.validation_step(x, 0)
    state = torch.zeros(1 + D + D * D, dtype=torch.float64, device="cuda")
    for _ in range(10):
        ops.latent_moments(mean, D, state)
    res["latent_moments_us"] = 1e3 * events_ms(lambda: ops.latent_moments(mean, D, state), 200)
    print(f"rave_latent_moments [{tuple(mean.shape)}]: {res['latent_moments_us']:.1f} us per call")

    g = torch.Generator(device="cuda").manual_seed(1)
    L = mean.shape[-1]
    scales = torch.logspace(-3, 0, D, device="cuda")[None, :, None]
    zs = [torch.randn(a.batch, 2 * D, L, device="cuda", generator=g) for _ in range(a.batches)]
    means = [(z[:, :D] * scales) for z in zs]
    core.latent_analysis(means[:2], D)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    core.latent_analysis(means, D)
    torch.cuda.synchronize()
    res["epoch_end_analysis_ms"] = 1e3 * (time.perf_counter() - t0)
    print(f"latent_analysis over {a.batches} batches (D = {D}): {res['epoch_end_analysis_ms']:.2f} ms")
    try:
        from sklearn.decomposition import PCA
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        z = torch.cat(means, 0).permute(0, 2, 1).reshape(-1, D)
        z = z - z.mean(0)
        PCA(D).fit(z.cpu().numpy())
        res["reference_analysis_ms"] = 1e3 * (time.perf_counter() - t0)
        print(f"reference way (cat -> cpu -> sklearn PCA): {res['reference_analysis_ms']:.2f} ms")
    except ImportError:
        res["reference_analysis_ms"] = "not measured (scikit-learn not installed)"
        print("reference way: not measured (scikit-learn not installed)")
    print("card:", res["card"])
    line = json.dumps(res)
    print(line)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

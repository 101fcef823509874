"""The exported model's `prior(temp)` (prior_v1.gin on a full-size v2 RAVE) on the device.

    python scripts/time_prior_export.py [--latent-size 16] [--reps 20] [--json OUT.json]

For B = 1 and B = 8 and T in {1, 2, 8, 64} frames per call:
  * ExportedRAVE.prior: the kept frame graph, one prologue launch and T replays per call;
  * Prior.sample(prefix, T + 1) of the same frames: the sampler captures and instantiates its frame graph in every call.
The two are alternated call by call, each call timed alone by a host clock around work that ends in a device
synchronise, after warm-up calls of the same shape; the medians are reported.  The real-time margin is one latent frame
of audio, 2048 / 48000 s = 42.7 ms, over the prior's time per frame.  The card name and power limit are read in the
same run."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from time_prior_sample import card  # noqa: E402

FRAME_S = 2048 / 48000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--latent-size", type=int, default=16)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    from rave_b200 import configs
    from rave_b200.export import ExportedRAVE

    if not torch.cuda.is_available():
        raise SystemExit("time_prior_export.py needs a CUDA device")
    D = a.latent_size
    res = dict(card=card(), latent_size=D, reps=a.reps, rows=[])
    print("card:", res["card"])
    torch.manual_seed(0)
    model = configs.build_rave("v2").cuda()
    prior = configs.build_prior(model, latent_size=D).cuda()
    ex = ExportedRAVE(model, prior=prior)
    R = prior.quantized_normal.resolution

    def host_time(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for B in (1, 8):
        ex.reset_prior()
        for T in (1, 2, 8, 64):
            temp = torch.zeros(B, 1, T, device="cuda")
            u, d = torch.rand(B, T, D, device="cuda"), torch.rand(B, T, D, device="cuda")
            prefix = torch.randint(0, R, (B, 1, D), dtype=torch.int32, device="cuda")
            us = torch.rand(B, T + 1, D, device="cuda")
            run_export = lambda: ex.prior(temp, u, d)                      # noqa: E731
            run_sample = lambda: prior.sample(prefix, T + 1, uniform=us)   # noqa: E731
            for _ in range(3):
                run_export()
                run_sample()
            te, ts = [], []
            for _ in range(a.reps):
                te.append(host_time(run_export))
                ts.append(host_time(run_sample))
            e_us, s_us = statistics.median(te) * 1e6, statistics.median(ts) * 1e6
            row = dict(B=B, T=T, prior_us_per_call=e_us, prior_us_per_frame=e_us / T, sample_us_per_call=s_us,
                       sample_us_per_frame=s_us / T, realtime_margin=FRAME_S / (e_us / T * 1e-6))
            res["rows"].append(row)
            print(f"B={B} T={T:3d}: prior {e_us:9.1f} us/call {e_us / T:8.1f} us/frame | sample(T+1) {s_us:9.1f} "
                  f"us/call {s_us / T:8.1f} us/frame | real-time margin x{row['realtime_margin']:.0f}")
    print(f"captures of the kept frame graph: {ex._prior_state.captures}")
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

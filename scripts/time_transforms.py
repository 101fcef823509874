"""The training-batch transforms on the device against the reference's per-example numpy / scipy pipeline on the host.

    python scripts/time_transforms.py [--json OUT.json]

Per shape: us per whole-batch call (rave_augment alone, with explicit draws; and the full call with the device draws),
timed with CUDA events over a CUDA graph of 20 calls replayed 10 times after a warm-up, and the achieved GB/s of the
bytes the algorithm needs (the cropped window read once, the output written once; normalise reads the window a second
time) against 3.35 TB/s.  Then ms per example of the reference's pipeline (crop, allpass, dequantise, optional
normalise) on this host's CPU, over the same examples.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from time_prior import card  # noqa: E402

SR = 44100
# (name, B, C, L, n_signal, int16, normalize)
SHAPES = [
    ("int16 [32,1,262144] -> [32,1,131072]", 32, 1, 262144, 131072, True, False),
    ("int16 [32,1,131072] -> [32,1,65536]", 32, 1, 131072, 65536, True, False),
    ("int16 stereo [16,2,262144] -> [16,2,131072]", 16, 2, 262144, 131072, True, False),
    ("int16 stereo [16,2,262144] -> [16,2,131072], normalise", 16, 2, 262144, 131072, True, True),
]


def graph_us(fn, n=20, replays=10):
    import torch
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            fn()
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(replays):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (n * replays)


def cpu_ms_per_example(raw_np, n_signal, normalize, examples):
    import numpy as np
    from oracle import transforms_oracle as TO
    rng = np.random.default_rng(0)
    t0 = time.perf_counter()
    for i in range(examples):
        x = raw_np[i]
        L = x.shape[-1]
        d = (rng.integers(0, L - n_signal + 1), 1.0, 2 * np.pi * 300 / SR, 1.0)
        TO.transform_example(x, n_signal, d, np.random.rand(x.shape[0], n_signal), normalize)
    return (time.perf_counter() - t0) * 1e3 / examples


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    ap.add_argument("--cpu-examples", type=int, default=8)
    args = ap.parse_args()
    import torch
    from rave_b200 import ops
    from rave_b200 import transforms as T
    assert torch.cuda.is_available(), "time_transforms.py measures on a GPU"
    info = card()
    print(json.dumps(info))
    rows = []
    for name, B, C, L, N, int16, normalize in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(0)
        raw = torch.randint(-20000, 20000, (B, C, L), dtype=torch.int16, device="cuda", generator=g)
        t = T.get_transforms(SR, N, normalize=normalize, augmentations=[T.RandomMute(0.1)], n_channels=C)
        out = torch.empty(B, C, N, device="cuda")
        draws = T.sample_draws(B, L, N, SR, device="cuda")
        key = torch.tensor([1, 2], dtype=torch.int64, device="cuda")
        kernel_us = graph_us(lambda: ops.augment(raw, draws, key, out, None, normalize, False))
        call_us = graph_us(lambda: t(raw, out=out))
        nbytes = B * C * N * (2 * (2 if normalize else 1) + 4)
        gbs = nbytes / kernel_us / 1e3
        cpu = cpu_ms_per_example(raw[:args.cpu_examples].cpu().numpy(), N, normalize, args.cpu_examples)
        row = {"shape": name, "kernel_us": round(kernel_us, 1), "call_us": round(call_us, 1),
               "bytes": nbytes, "GB_per_s": round(gbs, 1), "of_3350_GB_per_s": round(gbs / 3350, 3),
               "host_cpu_ms_per_example": round(cpu, 3), "host_cpu_ms_per_batch": round(cpu * B, 1)}
        rows.append(row)
        print(json.dumps(row))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()

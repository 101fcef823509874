"""Mono against stereo (n_channels = 2) training at the bench shape B = 32 x 65536 samples per channel.

    python scripts/time_stereo.py [--batch 32] [--cycles 3] [--rounds 3] [--json OUT.json]

1. The phase-2 step cycle -- one D-step and three G-steps (update_discriminator_every = 4) -- of v2 and v3, bf16, on
   whole-step CUDA graphs (GraphedTrainer), timed with CUDA events.  For each configuration the mono and the stereo model
   are built side by side and timed in alternation (`rounds` times, `cycles` cycles each); the minimum and the spread
   are printed.
2. The multichannel first-layer operand kernels alone, graph-timed (scripts/_timing.py), at cin = 1 and cin = 2 for the
   MSD (K = 15, stride 4, pools 1 / 4) and MPD (K = 5, stride 4, periods 2 / 11) first layers of a [real; fake] batch of
   2B rows: rave_im2col_cin (rave_im2col_c1 at cin = 1) and rave_gather_cin (rave_gather_c1).
3. The one copy stereo adds to the MRD: interleaving the B*C spectrograms [(b c), t, f, 2] into the channel-last
   [b, t, f, (c p)] input of the first conv, per FFT size.
The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

T = 65536


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:          # noqa: BLE001  (the numbers are still printed)
        return f"unknown ({e})"


def step_cycles(config, B, cycles, rounds):
    """{n_channels: [ms per 4-step cycle, one entry per round]} for the mono and stereo model of `config`."""
    import torch
    import rave_b200
    from rave_b200 import configs
    from rave_b200.graphs import GraphedTrainer
    rave_b200.set_precision("bf16")
    runs = {}
    try:
        trainers = {}
        for nc in (1, 2):
            torch.manual_seed(0)
            m = configs.build_rave(config, n_channels=nc).cuda().train()
            m.warmed_up = True
            g = torch.Generator(device="cuda").manual_seed(1234 + nc)
            x = (0.5 * torch.randn(B, nc, T, device="cuda", generator=g)).clamp(-1, 1)
            tr = GraphedTrainer(m, x)
            for i in range(4):
                tr.step(x, i)
            trainers[nc] = (m, tr, x)
        torch.cuda.synchronize()
        for _ in range(rounds):
            for nc, (m, tr, x) in trainers.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(4 * cycles):
                    tr.step(x, i)          # update_discriminator_every = 4 (v2.gin:86, v3 includes it)
                e1.record()
                torch.cuda.synchronize()
                runs.setdefault(nc, []).append(e0.elapsed_time(e1) / cycles)
        del trainers
    finally:
        rave_b200.set_precision("fp32")
        torch.cuda.empty_cache()
    return runs


def kernels(B):
    import torch
    from rave_b200 import ops
    from _timing import graph_time_us
    Bs = 2 * B
    rows = []
    for name, K, stride, pad, period, pool in [("msd0", 15, 4, 7, 1, 1), ("msd2", 15, 4, 7, 1, 4),
                                               ("mpd2", 5, 4, 2, 2, 1), ("mpd11", 5, 4, 2, 11, 1)]:
        Lin = (T + period - 1) // period if period > 1 else T // pool
        Lout = (Lin + 2 * pad - K) // stride + 1
        pitch = (Lout + 3) // 4 * 4
        for cin in (1, 2):
            W = ops.cin_width(cin, K)
            src = [torch.randn(Bs, cin, T, device="cuda") for _ in range(3)]
            P = [torch.randn(Bs * period, pitch, W, device="cuda") for _ in range(3)]
            if cin == 1:
                s1 = [s[:, 0].contiguous() for s in src]
                im = lambda i: ops.im2col_c1(s1[i % 3], Lin, Lout, pitch, K, stride, pad, period, pool)
                ga = lambda i: ops.gather_c1(P[i % 3], (Bs, T), Lin, Lout, K, stride, pad, period, pool)
            else:
                im = lambda i: ops.im2col_cin(src[i % 3], Lin, Lout, pitch, K, stride, pad, period, pool)
                ga = lambda i: ops.gather_cin(P[i % 3], (Bs, cin, T), Lin, Lout, K, stride, pad, period, pool)
            t_im = min(graph_time_us(im, n=9) for _ in range(3))
            t_ga = min(graph_time_us(ga, n=9) for _ in range(3))
            mb_im = (Bs * cin * T * 4 + Bs * period * pitch * W * 2) / 1e6
            mb_ga = (Bs * period * pitch * W * 4 + Bs * cin * T * 4 * 2) / 1e6
            r = dict(shape=name, cin=cin, W=W, im2col_us=t_im, im2col_gbs=mb_im / t_im * 1e3, gather_us=t_ga,
                     gather_gbs=mb_ga / t_ga * 1e3)
            rows.append(r)
            print(f"{name:6s} cin={cin} W={W}: im2col {t_im:7.1f} us ({r['im2col_gbs']:5.0f} GB/s)  gather {t_ga:7.1f} us "
                  f"({r['gather_gbs']:5.0f} GB/s)", flush=True)
            del src, P
    return rows


def mrd_interleave(B):
    import torch
    from _timing import graph_time_us
    Bs, C = 2 * B, 2
    out = {}
    for n_fft in (2048, 1024, 512):
        t = T // (n_fft // 4) + 1
        f = n_fft // 2 + 1
        zs = [torch.randn(Bs * C, t, f, 2, device="cuda") for _ in range(3)]
        fn = lambda i: zs[i % 3].unflatten(0, (Bs, C)).permute(0, 2, 3, 1, 4).reshape(Bs, t, f, 2 * C)
        us = min(graph_time_us(fn, n=9) for _ in range(3))
        mb = 2 * Bs * C * t * f * 2 * 4 / 1e6
        out[n_fft] = us
        print(f"MRD {n_fft}: stereo spectrogram interleave {us:7.1f} us ({mb / us * 1e3:5.0f} GB/s over {mb:.0f} MB)",
              flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--cycles", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_stereo.py measures on a CUDA device")
    dev = f"{torch.cuda.get_device_name()} | {card()}"
    print("card:", dev, flush=True)
    res = dict(card=dev, batch=args.batch, steps={})
    for config in ("v2", "v3"):
        runs = step_cycles(config, args.batch, args.cycles, args.rounds)
        res["steps"][config] = runs
        for nc, ts in runs.items():
            print(f"{config} n_channels={nc}: {min(ts):8.2f} ms per cycle (1 D + 3 G), {min(ts) / 4:7.2f} ms per step "
                  f"(rounds {[round(t, 2) for t in ts]})", flush=True)
    res["kernels"] = kernels(args.batch)
    res["mrd_interleave_us"] = mrd_interleave(args.batch)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

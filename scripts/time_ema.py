"""Cost of the weight average (`EMA`, csrc/ema.cu) on the flagship training step.

    python scripts/time_ema.py [--batch 32] [--steps 40] [--rounds 2] [--json OUT.json]

1. The graphed v2 bf16 phase-2 step (B x 65536, one G-step and one D-step graph) with and without `ema=`: the two
   trainers are built in turn on the same model, `--rounds` times, alternating, and each times `--steps` steps with
   CUDA events after 8 warm-up steps.
2. The update launch alone: CUDA events around a CUDA graph of 20 launches replayed 10 times; the swap likewise.  The
   bytes it must move (read p and ema, write ema: 12 bytes per parameter) over that time, against 3.35 TB/s.
3. The reference's eager per-tensor loop (scripts/train.py:87-95) over the same parameters on the same device.
The card name and power limit are read in the same run."""
import argparse
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from time_prior import card  # noqa: E402

HBM_TBS = 3.35


def events_ms(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--samples", type=int, default=65536)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()

    import torch
    import rave_b200
    from rave_b200 import configs
    from rave_b200.ema import EMA
    from rave_b200.graphs import GraphedTrainer

    rave_b200.set_precision("bf16")
    torch.manual_seed(0)
    model = configs.build_rave("v2", sampling_rate=48000).cuda().train()
    model.warmed_up = True
    n_params = sum(p.numel() for p in model.parameters())
    g = torch.Generator(device="cpu").manual_seed(1234)
    x = (0.5 * torch.randn(a.batch, 1, a.samples, generator=g)).clamp(-1, 1).cuda()
    ema = EMA(.999)

    steps = {"without": [], "with": []}
    launches = {}
    for _ in range(a.rounds):
        for kind in ("without", "with"):
            tr = GraphedTrainer(model, x, ema=ema if kind == "with" else None)
            launches[kind] = {("D" if k else "G"): v for k, v in tr.launches.items()}
            for i in range(8):
                tr.step(x, i)
            steps[kind].append(events_ms(lambda i: tr.step(x, i), a.steps))
            del tr
            gc.collect()
            torch.cuda.empty_cache()

    update_us = graph_us(ema._launch_update)
    swap_us = graph_us(ema._launch_swap)
    gbytes = 12 * n_params / 1e9

    weights = {n: p.data.clone() for n, p in model.named_parameters()}

    def reference_loop(_):
        for n, p in model.named_parameters():
            weights[n] = weights[n] * ema.factor + p.data * (1 - ema.factor)

    reference_loop(0)
    ref_ms = [events_ms(reference_loop, 20) for _ in range(2)]

    res = {
        "card": card(), "batch": [a.batch, 1, a.samples], "parameters": n_params,
        "tensors": len(list(model.parameters())), "rounds": a.rounds, "steps_per_window": a.steps,
        "step_ms_without_ema": steps["without"], "step_ms_with_ema": steps["with"],
        "library_launches_per_graph": launches,
        "update_us": update_us, "update_GBps": gbytes / (update_us * 1e-6),
        "update_share_of_hbm_peak": gbytes / (update_us * 1e-6) / (HBM_TBS * 1e3),
        "swap_us": swap_us, "reference_eager_loop_ms": ref_ms,
    }
    print(json.dumps(res))
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

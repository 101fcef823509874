"""Eval-mode forwards of a full-size v3 RAVE (`RAVE.forward`: PQMF, encoder, reparametrisation, decoder) with its AdaIN
layers in three style states, on the device.

    python scripts/time_style.py [--json OUT.json] [--min-seconds 1.0]

For B in {1, 8} and T in {2^16, 2^20} samples, in the identity state (nothing learned), the learn state (learn_target:
every call updates the statistics) and the transfer state (target and source learned, statistics frozen):
  fp32    the module-by-module fp32 parity kernels -- what an eval v3 forward ran in bf16 mode before the engine took
          eval-mode AdaIN chains;
  eager   the wgmma engine in bf16, launched from Python;
  graph   the same launches replayed from one CUDA graph captured per shape (the style state changes between replays
          through update_adain, in place).
Times are host clocks around work that ends in a device synchronise, after a warm-up call of the same shape, repeated
until --min-seconds have passed.  Then one torch.profiler pass per shape (engine, eager, transfer state) gives the share
of the kernel time spent in the two AdaIN kernels.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.time_prior_sample import card  # noqa: E402


def timed(fn, min_seconds):
    import torch
    fn()
    torch.cuda.synchronize()
    n, t0 = 0, time.perf_counter()
    while True:
        fn()
        n += 1
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if dt >= min_seconds and n >= 3:
            return dt / n * 1e3


def set_state(model, state):
    """identity: nothing learned; learn: learning the target; transfer: target and source learned (one call each on
    audio of two loudnesses), then frozen."""
    import torch
    model.update_adain(reset_target=True, reset_source=True)
    if state == "learn":
        model.update_adain(learn_target=True)
    elif state == "transfer":
        x = model.__dict__["_style_x"]
        with torch.no_grad():
            model.update_adain(learn_target=True)
            model(x)
            model.update_adain(learn_source=True)
            model(0.3 * x)
        model.update_adain()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None)
    ap.add_argument("--min-seconds", type=float, default=1.0)
    args = ap.parse_args()
    import torch
    import rave_b200
    from rave_b200 import configs

    assert torch.cuda.is_available(), "time_style.py measures on the GPU"
    torch.manual_seed(0)
    model = configs.build_rave("v3").cuda().eval()
    dev_name = card()
    print(f"device: {dev_name}")
    rows = []
    for T in (1 << 16, 1 << 20):
        for B in (1, 8):
            gen = torch.Generator(device="cuda").manual_seed(B * 31 + T)
            x = (0.5 * torch.randn(B, 1, T, generator=gen, device="cuda")).clamp(-1, 1)
            model.__dict__["_style_x"] = x
            res = {"B": B, "T": T}
            graph = static_y = None
            for state in ("identity", "learn", "transfer"):
                for mode in ("fp32", "eager", "graph"):
                    rave_b200.set_precision("fp32" if mode == "fp32" else "bf16")
                    set_state(model, state)
                    with torch.no_grad():
                        if mode == "graph":
                            if graph is None:
                                s = torch.cuda.Stream()
                                s.wait_stream(torch.cuda.current_stream())
                                with torch.cuda.stream(s):
                                    model(x)
                                torch.cuda.current_stream().wait_stream(s)
                                set_state(model, state)
                                graph = torch.cuda.CUDAGraph()
                                with torch.cuda.graph(graph):
                                    static_y = model(x)
                                set_state(model, state)
                            ms = timed(graph.replay, args.min_seconds)
                        else:
                            ms = timed(lambda: model(x), args.min_seconds)
                    res[f"{state}_{mode}_ms"] = ms
                    print(f"B={B} T=2^{T.bit_length() - 1} {state:9s} {mode:6s} {ms:9.3f} ms", flush=True)
            # AdaIN share of the kernel time: engine, eager, transfer state, one profiled call after a warm-up
            rave_b200.set_precision("bf16")
            set_state(model, "transfer")
            with torch.no_grad():
                model(x)
                torch.cuda.synchronize()
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    model(x)
                    torch.cuda.synchronize()
            tot = ada = 0.0
            for ev in prof.key_averages():          # CUDA activities only: kernels, memsets, copies
                tot += ev.device_time_total
                if "adain" in ev.key:
                    ada += ev.device_time_total
            res["adain_kernel_us"] = ada
            res["kernel_us"] = tot
            res["adain_share"] = ada / tot if tot else float("nan")
            print(f"B={B} T=2^{T.bit_length() - 1} AdaIN kernels {ada:.1f} us of {tot:.1f} us kernel time "
                  f"({100 * res['adain_share']:.2f} %)", flush=True)
            rows.append(res)
            del graph, static_y
            torch.cuda.empty_cache()
    rave_b200.set_precision("fp32")
    hdr = f"{'B':>2} {'T':>5} | " + " | ".join(f"{s:^26s}" for s in ("identity", "learn", "transfer")) + " | AdaIN"
    print(hdr)
    print(f"{'':>8} | " + " | ".join(f"{'fp32':>8} {'eager':>8} {'graph':>8}" for _ in range(3)) + " | share")
    for r in rows:
        cells = " | ".join(f"{r[f'{s}_fp32_ms']:8.2f} {r[f'{s}_eager_ms']:8.2f} {r[f'{s}_graph_ms']:8.2f}"
                           for s in ("identity", "learn", "transfer"))
        print(f"{r['B']:>2} 2^{r['T'].bit_length() - 1:<3} | {cells} | {100 * r['adain_share']:.2f} %")
    print("(milliseconds per RAVE.forward)")
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"device": dev_name, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()

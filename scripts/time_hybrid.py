"""Parts and step of the hybrid configuration (rave/configs/hybrid.gin on top of v2.gin) at the bench shape
B = 32 x 65536 samples, 48 kHz.

    python scripts/time_hybrid.py [--batch 32] [--steps 8] [--json OUT.json]

1. The mel front end (centred framing, cuFFT rfft, rave_mel_log1p_fwd) on [B, 1, 65536], CUDA events over 20 calls.
2. The two-layer GRU head (128 -> 128, T = 32 latent steps) forward and forward + backward: this project's kernels
   (ops.gru: GEMM + one persistent rave_gru_fwd / rave_gru_bwd launch per layer) next to cuDNN's nn.GRU as the stock
   arm, same shapes, fp32.
3. The bf16 phase-2 training step of v2 + hybrid against v2, the two models alternated in one process (eager steps,
   CUDA events, D-step every 4th as bench.py).
The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T = 65536


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:          # noqa: BLE001  (the numbers are still printed)
        return f"unknown ({e})"


def events_ms(fn, n):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    import rave_b200
    from rave_b200 import blocks, configs
    if not torch.cuda.is_available():
        raise SystemExit("time_hybrid.py needs a CUDA device")
    B = args.batch
    res = dict(card=card(), batch=B, T=T)
    print("card:", res["card"])

    mel = configs.mel_spectrogram(48000).cuda()
    x = (0.5 * torch.randn(B, 1, T, device="cuda")).clamp(-1, 1)
    res["mel_front_end_ms"] = events_ms(lambda: mel.encode_log1p(x), 20)
    print(f"mel front end [B={B}, 1, {T}]: {res['mel_front_end_ms']:.3f} ms")

    Lz = T // 2048
    torch.manual_seed(0)
    ours = blocks.GRU(128, 2).cuda()
    stock = torch.nn.GRU(128, 128, 2, batch_first=True).cuda()
    stock.load_state_dict(ours.gru.state_dict())
    z = torch.randn(B, 128, Lz, device="cuda", requires_grad=True)
    zt = z.detach().transpose(1, 2).contiguous().requires_grad_(True)

    def fb_ours():
        ours(z).sum().backward()

    def fb_stock():
        stock(zt)[0].sum().backward()
    with torch.no_grad():
        res["gru_fwd_ms"] = events_ms(lambda: ours(z), 20)
        res["gru_fwd_cudnn_ms"] = events_ms(lambda: stock(zt), 20)
    res["gru_fwd_bwd_ms"] = events_ms(fb_ours, 20)
    res["gru_fwd_bwd_cudnn_ms"] = events_ms(fb_stock, 20)
    print(f"GRU 2 x 128, B={B}, T={Lz}: forward {res['gru_fwd_ms']:.3f} ms (cuDNN {res['gru_fwd_cudnn_ms']:.3f}), "
          f"forward + backward {res['gru_fwd_bwd_ms']:.3f} ms (cuDNN {res['gru_fwd_bwd_cudnn_ms']:.3f})")

    rave_b200.set_precision("bf16")
    models = {}
    for name in ("v2", "v2_hybrid"):
        m = configs.build_rave(name, sampling_rate=48000).cuda().train()
        m.warmed_up = True
        m.optimizers()
        models[name] = m
    xb = (0.5 * torch.randn(B, 1, T, device="cuda")).clamp(-1, 1)
    step = {n: [] for n in models}
    for r in range(args.rounds):
        for name, m in models.items():
            i0 = [0]

            def one():
                m.training_step(xb, i0[0])
                i0[0] += 1
            step[name].append(events_ms(one, args.steps))
    res["step_ms"] = step
    for name, v in step.items():
        print(f"bf16 phase-2 step {name}: " + ", ".join(f"{t:.2f}" for t in v) + " ms")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

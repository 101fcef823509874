"""The latent regularisers of `--config v2 --config wasserstein` / `spherical` on the device.

    python scripts/time_regularization.py [--batch 32] [--step-batch 16] [--steps 12] [--json OUT.json]

1. The MMD (rave_mmd_fwd, rave_mmd_bwd) against the reference's ATen expression (rave/blocks.py:761-774, which
   materialises three N x N x D difference tensors) on the same device, at N = 1024, 2048, 4096 rows and D = 16:
   forward, and forward + backward.  Each side is captured once into a CUDA graph and replayed
   (scripts/_timing.py); the kernel side also reports the largest deviation of its MMD from the ATen value.
2. The sphere projection (rave_sphere_norm_fwd + _bwd) at the v2 latent shape [B, 16, 32] against the reference's
   `z / torch.norm(z, dim=1)` and its autograd backward.
3. The training step of v2_wasserstein against v2 at step-batch x 65536 samples, bf16, whole-step CUDA graphs (GraphedTrainer):
   the phase-1 G-step, then the phase-2 cycle (one D-step and three G-steps), the two configurations alternated.
The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:          # noqa: BLE001  (the numbers are still printed)
        return f"unknown ({e})"


def aten_mmd(z, prior):
    """WasserteinEncoder.reparametrize's regulariser as the reference computes it."""
    x = z.permute(0, 2, 1).reshape(-1, z.shape[1])

    def k(a, b):
        return (-((a[:, None] - b[None]).pow(2).mean(2) / a.shape[-1])).exp().mean()
    return k(x, x) + k(prior, prior) - 2 * k(x, prior)


def time_mmd(res):
    import torch
    from _timing import graph_time_us
    from rave_b200 import ops
    D = 16
    for N in (1024, 2048, 4096):
        B, L = 32, N // 32
        g = torch.Generator(device="cuda").manual_seed(N)
        zs = [torch.randn(B, D, L, device="cuda", generator=g).requires_grad_(True) for _ in range(2)]
        ps = [torch.randn(N, D, device="cuda", generator=g) for _ in range(2)]
        one = torch.ones((), device="cuda")
        row = dict(N=N, D=D)
        row["kernel_fwd_us"] = graph_time_us(lambda i: ops.mmd(zs[i % 2].detach(), ps[i % 2]), n=10)
        row["aten_fwd_us"] = graph_time_us(lambda i: aten_mmd(zs[i % 2].detach(), ps[i % 2]), n=4)
        row["kernel_fwd_bwd_us"] = graph_time_us(
            lambda i: torch.autograd.grad(ops.mmd(zs[i % 2], ps[i % 2])[0], [zs[i % 2]], one), n=10)
        row["aten_fwd_bwd_us"] = graph_time_us(
            lambda i: torch.autograd.grad(aten_mmd(zs[i % 2], ps[i % 2]), [zs[i % 2]], one), n=4)
        with torch.no_grad():
            ref = aten_mmd(zs[0].double(), ps[0].double())
            got = ops.mmd(zs[0].detach(), ps[0])[0]
        row["abs_err_vs_fp64"] = abs(float(got) - float(ref))
        row["mmd"] = float(ref)
        print(f"MMD N={N:5d} D={D}: fwd {row['kernel_fwd_us']:8.1f} us (ATen {row['aten_fwd_us']:8.1f}), "
              f"fwd+bwd {row['kernel_fwd_bwd_us']:8.1f} us (ATen {row['aten_fwd_bwd_us']:8.1f}); "
              f"|mmd - fp64| {row['abs_err_vs_fp64']:.2e} (mmd {row['mmd']:.3e})", flush=True)
        res["mmd"].append(row)


def time_sphere(res, B):
    import torch
    from _timing import graph_time_us
    from rave_b200 import ops
    zs = [torch.randn(B, 16, 32, device="cuda").requires_grad_(True) for _ in range(2)]
    gy = torch.randn(B, 16, 32, device="cuda")
    row = dict(shape=[B, 16, 32])
    row["kernel_fwd_bwd_us"] = graph_time_us(lambda i: torch.autograd.grad(ops.sphere_norm(zs[i % 2]), [zs[i % 2]], gy))
    row["aten_fwd_bwd_us"] = graph_time_us(
        lambda i: torch.autograd.grad(zs[i % 2] / torch.norm(zs[i % 2], p=2, dim=1, keepdim=True), [zs[i % 2]], gy))
    print(f"sphere projection [B={B}, 16, 32] fwd+bwd: {row['kernel_fwd_bwd_us']:.1f} us "
          f"(ATen {row['aten_fwd_bwd_us']:.1f} us)", flush=True)
    res["sphere"] = row


def time_steps(res, B, steps, rounds=3):
    import torch
    import rave_b200
    from rave_b200 import configs
    from rave_b200.graphs import GraphedTrainer
    rave_b200.set_precision("bf16")
    x = (0.5 * torch.randn(B, 1, 65536, device="cuda")).clamp(-1, 1)
    trainers = {}
    for name in ("v2", "v2_wasserstein"):
        for phase2 in (False, True):
            torch.manual_seed(0)
            m = configs.build_rave(name).cuda().train()
            m.warmed_up = phase2
            if name == "v2_wasserstein":
                m.beta_factor = 100.0
            trainers[(name, phase2)] = GraphedTrainer(m, x)
    out = {f"{n} phase{2 if p else 1}": [] for n, p in trainers}
    for _ in range(rounds):
        for key, tr in trainers.items():
            # phase 1: G-steps only; phase 2: the reference's cycle, one D-step every four steps
            idx = [1 + 4 * i for i in range(steps)] if not key[1] else list(range(steps))
            tr.step(x, idx[0])
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in idx:
                tr.step(x, i)
            e1.record()
            torch.cuda.synchronize()
            out[f"{key[0]} phase{2 if key[1] else 1}"].append(e0.elapsed_time(e1) / steps)
    for k, v in out.items():
        print(f"{k}: {', '.join(f'{t:.2f}' for t in v)} ms/step (B={B} x 65536, bf16, graphed)", flush=True)
    res["steps_ms"] = out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32, help="batch of the sphere projection's latent")
    ap.add_argument("--step-batch", type=int, default=16,
                    help="batch of the timed training steps (four graphed full-size models stay resident)")
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("time_regularization.py measures on a CUDA device; none found")
    res = dict(card=card(), mmd=[])
    print("card:", res["card"], flush=True)
    time_mmd(res)
    time_sphere(res, args.batch)
    time_steps(res, args.step_batch, args.steps)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

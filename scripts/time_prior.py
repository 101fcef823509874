"""The latent prior's training step (VariationalPrior, prior_v1.gin) on the device, at train_prior's defaults.

    python scripts/time_prior.py [--batch 8] [--samples 262144] [--latent-size 16] [--json OUT.json]

1. The whole graphed step (GraphedPriorTrainer, bf16): frozen v2 encode + latent classes + prior forward / backward +
   FusedAdam, replayed from one CUDA graph.
2. Its split: the frozen encode + latent classes alone (captured on their own), and the rest (prior forward + backward
   + Adam) as the difference.
3. The reference's arithmetic on stock torch (cuDNN, TF32 allowed as scripts/train.py allows it): the oracle port of the
   encoder (oracle/rave_oracle.py) and of the prior (oracle/prior_oracle.py, stacked one-hot, grouped convs,
   F.cross_entropy), autograd and torch.optim.Adam, on the same device, captured the same way.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--samples", type=int, default=262144)
    ap.add_argument("--latent-size", type=int, default=16)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    import rave_b200
    from _timing import graph_time_us
    from rave_b200 import configs
    from rave_b200.prior import GraphedPriorTrainer
    from oracle import prior_oracle as P
    from oracle import rave_oracle as O

    if not torch.cuda.is_available():
        raise SystemExit("time_prior.py needs a CUDA device")
    res = dict(card=card(), batch=a.batch, samples=a.samples, latent_size=a.latent_size)
    print("card:", res["card"])
    torch.manual_seed(0)
    m = configs.build_rave("v2")
    prior = configs.build_prior(m, latent_size=a.latent_size).cuda()
    xs = [(0.3 * torch.randn(a.batch, 1, a.samples, device="cuda")).clamp(-1, 1) for _ in range(2)]
    rave_b200.set_precision("bf16")
    try:
        tr = GraphedPriorTrainer(prior, xs[0])
        for i in range(3):
            tr.step(xs[i % 2])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n = 20
        e0.record()
        for i in range(n):
            tr.step(xs[i % 2])
        e1.record()
        torch.cuda.synchronize()
        res["graphed_step_ms"] = e0.elapsed_time(e1) / n
        res["graph_launches"] = tr.launches
        res["encode_classes_ms"] = graph_time_us(lambda i: prior.latent_classes(xs[i % 2]), n=4) / 1e3
    finally:
        rave_b200.set_precision("fp32")
    res["prior_fwd_bwd_adam_ms"] = res["graphed_step_ms"] - res["encode_classes_ms"]
    print(f"graphed bf16 step: {res['graphed_step_ms']:.3f} ms ({tr.launches} library launches); frozen encode + "
          f"classes {res['encode_classes_ms']:.3f} ms; prior forward + backward + Adam {res['prior_fwd_bwd_adam_ms']:.3f} ms")

    # the reference's arithmetic on stock torch
    try:
        torch.backends.cuda.matmul.allow_tf32 = True
        torch.backends.cudnn.allow_tf32 = True
        cfg = O.v2_config()
        sd = {k: v.detach() for k, v in m.state_dict().items()}
        hk = sd["pqmf.hk"]
        D, R = prior.latent_size, P.PRIOR_V1["resolution"]
        psd = {k: v.detach().clone().requires_grad_(True) for k, v in prior.state_dict().items()
               if not k.startswith("synth.")}
        opt = torch.optim.Adam(list(psd.values()), lr=torch.tensor(1e-4, device="cuda"), capturable=True)

        def ref_encode(i):
            with torch.no_grad():
                z = O.encoder_v2(O.pqmf_encode(xs[i % 2], hk), sd, "encoder.encoder.", cfg)
                eps = torch.randn(z.shape[0], z.shape[1] // 2, z.shape[2], device="cuda")
                return P.latent_classes(z, eps, sd["latent_mean"], sd["latent_pca"], D, R)

        def ref_step(i):
            cls = ref_encode(i)
            loss = P.loss(cls, psd, P.PRIOR_V1, D)
            grads = torch.autograd.grad(loss, list(psd.values()), allow_unused=True)
            for p, g in zip(psd.values(), grads):
                p.grad = g
            opt.step()
        res["reference_encode_classes_ms"] = graph_time_us(ref_encode, n=2) / 1e3
        res["reference_step_ms"] = graph_time_us(ref_step, n=2) / 1e3
        print(f"reference arithmetic (torch / cuDNN, TF32): step {res['reference_step_ms']:.3f} ms, of which encode + "
              f"classes {res['reference_encode_classes_ms']:.3f} ms")
    except Exception as e:          # noqa: BLE001  (the library's numbers above stand on their own)
        res["reference_error"] = repr(e)
        print("reference timing failed:", repr(e))
    print(json.dumps(res))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

"""The exported model's encode / decode (rave_b200.ExportedRAVE) of v2, discrete and v2_spherical on the device, bf16
eval mode, at B = 8 examples of 2^20 samples.

    python scripts/time_export.py [--batch 8] [--samples 1048576] [--json OUT.json]

Per configuration and direction: the whole call; the latent processing alone (csrc/export.cu); the same latent
arithmetic written in torch on the same device (the reference's formulas of scripts/export.py, and for the discrete
model the residual-VQ loop of rave_b200/quantization.py: one distance GEMM, argmax, gather and subtraction per stage);
the latent share of the call; and how far the two latent outputs agree.  CUDA events around 10 calls after 3 warm-up
calls.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:          # noqa: BLE001  (the numbers are still printed)
        return f"unknown ({e})"


def timed(fn, n=10, warm=3):
    import torch
    for _ in range(warm):
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
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--samples", type=int, default=2 ** 20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    import torch.nn.functional as F
    import rave_b200
    from oracle import export_oracle as EO
    from rave_b200 import configs
    from rave_b200.export import ExportedRAVE

    if not torch.cuda.is_available():
        raise SystemExit("time_export.py needs a CUDA device")
    res = dict(card=card(), batch=a.batch, samples=a.samples, rows=[])
    print("card:", res["card"])
    rave_b200.set_precision("bf16")
    torch.backends.cuda.matmul.allow_tf32 = False       # the reference's fp32 distance GEMM
    torch.set_grad_enabled(False)
    try:
        for name in ("v2", "discrete", "v2_spherical"):
            torch.manual_seed(0)
            m = configs.build_rave(name).cuda()
            del m.discriminator
            L = m.latent_size
            m.latent_pca.copy_(torch.linalg.qr(torch.randn(L, L, device="cuda", dtype=torch.float64))[0].float())
            m.latent_mean.copy_(0.1 * torch.randn(L, device="cuda"))
            m.fidelity.copy_(1 - 0.9 ** torch.arange(1, L + 1, device="cuda", dtype=torch.float32))
            if name == "discrete":
                for q, vq in enumerate(m.encoder.rvq.layers):
                    vq._codebook.embed.copy_(torch.randn_like(vq._codebook.embed) * 0.7 ** q)
            ex = ExportedRAVE(m)
            x = (0.3 * torch.randn(a.batch, 1, a.samples, device="cuda")).clamp(-1, 1)
            raw = m.encode(x).float()
            B, C, T = raw.shape
            eps = torch.randn(B, L, T, device="cuda") if ex.kind == "variational" else None
            z = ex.post_process_latent(raw, eps)
            n_noise = (L - ex.latent_size) if ex.kind == "variational" else ex.n_noise
            noise = torch.randn(B, n_noise, T, device="cuda") if n_noise else None
            mean, pca = m.latent_mean, m.latent_pca

            if ex.kind == "variational":
                def ref_post():
                    mu, scale = raw.chunk(2, 1)
                    s = eps * (F.softplus(scale) + 1e-4) + mu - mean.unsqueeze(-1)
                    return F.conv1d(s, pca.unsqueeze(-1))[:, :ex.latent_size]

                def ref_pre():
                    return F.conv1d(torch.cat([z, noise], 1), pca.T.unsqueeze(-1)) + mean.unsqueeze(-1)
            elif ex.kind == "discrete":
                def ref_post():
                    return m.encoder.rvq.encode(raw).float()

                def ref_pre():
                    k = torch.clamp(z, 0, m.encoder.rvq.layers[0].codebook_size - 1).long()
                    return torch.cat([m.encoder.rvq.decode(k), noise], 1)
            else:
                def ref_post():
                    return EO.sphere_to_angles(raw)

                def ref_pre():
                    return EO.angles_to_sphere(z)

            zr, pr, pn = ref_post(), ref_pre(), ex.pre_process_latent(z, noise)
            if ex.kind == "discrete":
                agree_enc = f"codes equal {(zr == z).float().mean().item():.6f}"
            else:
                agree_enc = f"max |diff| {(zr - z).abs().max().item():.2e}"
            agree_dec = f"max |diff| {(pr - pn).abs().max().item():.2e}"
            t_enc = timed(lambda: ex.encode(x, eps))
            t_dec = timed(lambda: ex.decode(z, noise))
            t_post = timed(lambda: ex.post_process_latent(raw, eps))
            t_pre = timed(lambda: ex.pre_process_latent(z, noise))
            t_rpost, t_rpre = timed(ref_post), timed(ref_pre)
            for d, call, lat, ref, agree in (("encode", t_enc, t_post, t_rpost, agree_enc),
                                             ("decode", t_dec, t_pre, t_rpre, agree_dec)):
                row = dict(config=name, direction=d, frames=B * T, latent_size=ex.latent_size, call_ms=call,
                           latent_ms=lat, torch_latent_ms=ref, share=lat / call, agreement=agree)
                if ex.kind == "discrete" and d == "encode":
                    Q, K = len(m.encoder.rvq.layers), m.encoder.rvq.layers[0].codebook_size
                    row["rvq_gflop"] = 2.0 * B * T * K * C * Q / 1e9
                    row["rvq_tflops"] = row["rvq_gflop"] / lat
                res["rows"].append(row)
                print(json.dumps(row))
            del m, ex, x, raw
            torch.cuda.empty_cache()
    finally:
        rave_b200.set_precision("fp32")
    print(f"\n{res['card']}, B = {a.batch} x {a.samples} samples, bf16 eval")
    print(f"{'config':14s}{'call':>8s}{'latent':>14s}{'frames':>8s}{'call ms':>10s}{'latent ms':>11s}"
          f"{'torch ms':>10s}{'share':>8s}  agreement")
    for r in res["rows"]:
        print(f"{r['config']:14s}{r['direction']:>8s}{r['latent_size']:>14d}{r['frames']:>8d}{r['call_ms']:>10.3f}"
              f"{r['latent_ms']:>11.4f}{r['torch_latent_ms']:>10.4f}{100 * r['share']:>7.2f}%  {r['agreement']}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

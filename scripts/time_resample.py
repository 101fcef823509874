"""The export's resampler (rave_b200.resampler, csrc/resample.cu) on the device at export sizes: B = 8 examples of 2^20
samples at the target rate, mono and stereo, ratios 2 and 3.

    python scripts/time_resample.py [--batch 8] [--samples 1048576] [--json OUT.json]

Per ratio, channel count and direction: the kernel time (CUDA events around 20 launches after 3 warm-up launches, the
kernel and the torch arm alternated over 5 rounds, medians reported), the bytes it must move (input read once, output
written once) over 3.35 TB/s, and the same arithmetic through torch.nn.functional.conv1d in float32 on the device
(TF32 off, as printed: the reference's fp32 conv, plus the permute / reshape its up path needs).  Then the share of the
resampling in a full v2 `ExportedRAVE.forward` with target_sr = 2 sr (bf16 eval).  The card name and power limit are
read in the same run."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.time_export import card  # noqa: E402

HBM = 3.35e12


def events_ms(fn, n=20, warm=3):
    import torch
    for _ in range(warm):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def alternate(fns, rounds=5):
    times = [[] for _ in fns]
    for _ in range(rounds):
        for i, fn in enumerate(fns):
            times[i].append(events_ms(fn))
    return [statistics.median(t) for t in times]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--samples", type=int, default=2 ** 20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    import torch.nn.functional as F
    import rave_b200
    from rave_b200 import configs
    from rave_b200.export import ExportedRAVE
    from rave_b200.resampler import Resampler

    if not torch.cuda.is_available():
        raise SystemExit("time_resample.py needs a CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    res = dict(card=card(), batch=a.batch, samples=a.samples, cudnn_allow_tf32=torch.backends.cudnn.allow_tf32,
               rows=[])
    print("card:", res["card"], "| cudnn.allow_tf32:", res["cudnn_allow_tf32"])
    torch.set_grad_enabled(False)
    sr = 48000
    for ratio in (2, 3):
        rs = Resampler(ratio * sr, sr).cuda()
        wd, wu = rs.downsample.weight.detach(), rs.upsample.weight.detach()
        for C in (1, 2):
            x = 0.3 * torch.randn(a.batch, C, a.samples, device="cuda")
            xm = rs.to_model_sampling_rate(x)

            def torch_down():
                return F.conv1d(F.pad(x.reshape(-1, 1, x.shape[-1]), rs.downsample._pad), wd,
                                stride=ratio).reshape(a.batch, C, -1)

            def torch_up():
                y = F.conv1d(F.pad(xm.reshape(-1, 1, xm.shape[-1]), rs.upsample._pad), wu)
                return y.permute(0, 2, 1).reshape(a.batch, C, -1)

            for d, ours, ref, inp in (("down", lambda: rs.to_model_sampling_rate(x), torch_down, x),
                                      ("up", lambda: rs.from_model_sampling_rate(xm), torch_up, xm)):
                y = ours()
                diff = (y - ref()).abs().max().item()
                t_k, t_t = alternate([ours, ref])
                nbytes = 4 * (inp.numel() + y.numel())
                row = dict(ratio=ratio, channels=C, direction=d, in_samples=inp.numel(), out_samples=y.numel(),
                           kernel_us=1e3 * t_k, conv1d_us=1e3 * t_t, bytes=nbytes, tb_per_s=nbytes / (t_k * 1e-3) / 1e12,
                           hbm_share=nbytes / HBM / (t_k * 1e-3), max_abs_diff_vs_conv1d=diff)
                res["rows"].append(row)
                print(json.dumps(row))
            del x, xm
    # share of a full forward
    rave_b200.set_precision("bf16")
    try:
        torch.manual_seed(0)
        m = configs.build_rave("v2", sampling_rate=sr).cuda()
        del m.discriminator
        ex = ExportedRAVE(m, target_sr=2 * sr)
        x = (0.3 * torch.randn(a.batch, 1, a.samples, device="cuda")).clamp(-1, 1)
        xm = ex.resampler.to_model_sampling_rate(x)
        ym = m.decode(ex.pre_process_latent(ex.encode(x)))
        t_fwd, t_down, t_up = alternate([lambda: ex(x), lambda: ex.resampler.to_model_sampling_rate(x),
                                         lambda: ex.resampler.from_model_sampling_rate(ym)], rounds=3)
        res["forward"] = dict(forward_ms=t_fwd, down_ms=t_down, up_ms=t_up, share=(t_down + t_up) / t_fwd)
        print(json.dumps(res["forward"]))
        del m, ex, x, xm, ym
    finally:
        rave_b200.set_precision("fp32")

    print(f"\n{res['card']}, B = {a.batch} x {a.samples} samples at the target rate, cudnn.allow_tf32 "
          f"{res['cudnn_allow_tf32']}")
    print(f"{'ratio':>5s}{'C':>3s}{'dir':>6s}{'kernel us':>11s}{'TB/s':>7s}{'of HBM':>8s}{'conv1d us':>11s}{'max diff':>10s}")
    for r in res["rows"]:
        print(f"{r['ratio']:>5d}{r['channels']:>3d}{r['direction']:>6s}{r['kernel_us']:>11.1f}{r['tb_per_s']:>7.2f}"
              f"{100 * r['hbm_share']:>7.1f}%{r['conv1d_us']:>11.1f}{r['max_abs_diff_vs_conv1d']:>10.1e}")
    f = res["forward"]
    print(f"v2 ExportedRAVE.forward, target_sr = 2 sr: {f['forward_ms']:.2f} ms; down {1e3 * f['down_ms']:.1f} us + "
          f"up {1e3 * f['up_ms']:.1f} us = {100 * f['share']:.2f}% of it")
    if a.json:
        with open(a.json, "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()

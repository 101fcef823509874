"""D-step forward + backward of the multi-scale spectral discriminator (configs/spectral_discriminator.gin: scales
4096 / 2048 / 1024 / 512 / 256, EncodecConvNet capacity 32) at the bench shape: B = 32 x 65536, real + fake = 64 rows.

    python scripts/time_spectral_disc.py [--batch 32] [--iters 10] [--json OUT.json]

Two arms, per scale and in total:
  engine : rave_b200 in bf16 mode (framing kernel + cuFFT, every conv a one-layer wgmma chain, fused feature taps);
  cudnn  : the same arithmetic as the oracle restatement (oracle/spectral_oracle.py::multi_scale_spectral_discriminator) on
           CUDA tensors, torch.stft + F.conv2d on cuDNN with TF32 allowed.
The loss is the hinge term of a D-step on the scores (rave/core.py:151-155); as in the training step the input needs no
gradient.  Every shape is warmed up, then timed with CUDA events over --iters iterations.
Algorithmic work, from the layer shapes: GFLOP = forward convs + weight gradients + data gradients of every conv but the
first; MB = every conv's input and output read or written once in fp32 per pass (forward: input, output, post-activation
feature; backward: data gradient in and out, weight gradient reading input and output gradient).  The bound is the larger
of GFLOP over the data-sheet peak (bf16 989 TFLOP/s for the engine, TF32 495 TFLOP/s for cuDNN) and MB over 3.35 TB/s;
"roofline" is that bound's time over the measured time.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
from functools import partial

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SCALES = [4096, 2048, 1024, 512, 256]
PEAK = {"engine": 989e12, "cudnn": 495e12}
BW = 3.35e12
# (kf, kt), stride along frequency, time dilation, Cin, Cout of the EncodecConvNet convs (rave/discriminator.py:54-67)
GEOMETRY = lambda cap: [((9, 3), 1, 1, 2, cap), ((9, 3), 2, 1, cap, cap), ((9, 3), 2, 2, cap, cap),
                        ((9, 3), 2, 4, cap, cap), ((3, 3), 1, 1, cap, cap), ((3, 3), 1, 1, cap, 1)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:
        return f"unknown ({type(e).__name__})"


def work(rows, T, n_fft, cap):
    """(flops, bytes) of one D-step forward + backward of one scale."""
    frames = 1 + (T - n_fft) // (n_fft // 4)
    Fq = n_fft // 2 + 1
    fl = by = 0.0
    for i, ((kf, kt), sf, _, cin, cout) in enumerate(GEOMETRY(cap)):
        Fo = (Fq + 2 * (kf // 2) - kf) // sf + 1
        mac = 2.0 * rows * frames * Fo * cout * cin * kf * kt
        fl += mac * (2 if i == 0 else 3)
        n_in, n_out = rows * frames * Fq * cin, rows * frames * Fo * cout
        by += 4.0 * (n_in + 2 * n_out) + 4.0 * (2 * n_out + 2 * n_in)
        Fq = Fo
    fl += 2.0 * rows * frames * 5 * n_fft * max(n_fft.bit_length() - 1, 1)      # the FFT, 5 N log2 N
    by += 4.0 * rows * T + 8.0 * rows * frames * (n_fft // 2 + 1)
    return fl, by


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--T", type=int, default=65536)
    ap.add_argument("--capacity", type=int, default=32)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("time_spectral_disc.py measures on the GPU; no CUDA device found")
    import rave_b200
    from rave_b200.discriminator import EncodecConvNet, MultiScaleSpectralDiscriminator
    from oracle import spectral_oracle as S
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    rows = 2 * a.batch
    torch.manual_seed(0)
    disc = MultiScaleSpectralDiscriminator(SCALES, partial(EncodecConvNet, capacity=a.capacity)).cuda()
    params = {k: v.detach().clone().requires_grad_("window" not in k) for k, v in disc.state_dict().items()}
    x = (0.5 * torch.randn(rows, 1, a.T, device="cuda")).clamp(-1, 1)

    def hinge(score):
        return torch.relu(1 - score[:a.batch]).mean() + torch.relu(1 + score[a.batch:]).mean()

    def engine_step(i):
        net, spec = disc.nets[i], disc.specs[i]
        feats = net.forward_cl(torch.view_as_real(spec.frames_spectrum(x[:, 0])))
        hinge(feats[-1]).backward()

    def cudnn_step(i):
        s = S.spectrogram(x, SCALES[i])
        feats = S.encodec_convnet(torch.cat([s.real, s.imag], 1), params, f"nets.{i}.")
        hinge(feats[-1]).backward()

    def timed(fn, i):
        for _ in range(3):
            fn(i)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            fn(i)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.iters

    gpu = card()
    print(f"card: {gpu}")
    print(f"D-step forward + backward, {rows} rows x {a.T} samples, EncodecConvNet capacity {a.capacity}, "
          f"{a.iters} timed iterations per shape after 3 warm-up iterations")
    res = {"card": gpu, "rows": rows, "T": a.T, "capacity": a.capacity, "scales": {}}
    hdr = f"{'scale':>6} {'arm':>7} {'ms':>9} {'GFLOP':>9} {'MB':>9} {'bound':>8} {'roofline':>9}"
    print(hdr)
    tot = {"engine": [0.0, 0.0, 0.0], "cudnn": [0.0, 0.0, 0.0]}
    for i, n in enumerate(SCALES):
        fl, by = work(rows, a.T, n, a.capacity)
        res["scales"][n] = {}
        for arm in ("engine", "cudnn"):
            if arm == "engine":
                rave_b200.set_precision("bf16")
            try:
                ms = timed(engine_step if arm == "engine" else cudnn_step, i)
            finally:
                rave_b200.set_precision("fp32")
            t_c, t_m = fl / PEAK[arm], by / BW
            bound = "tensor" if t_c >= t_m else "memory"
            frac = max(t_c, t_m) / (ms * 1e-3)
            res["scales"][n][arm] = dict(ms=ms, gflop=fl / 1e9, mb=by / 1e6, bound=bound, roofline=frac)
            tot[arm][0] += ms
            tot[arm][1] += fl
            tot[arm][2] += by
            print(f"{n:>6} {arm:>7} {ms:>9.2f} {fl / 1e9:>9.1f} {by / 1e6:>9.1f} {bound:>8} {frac:>9.3f}")
            for p in list(disc.parameters()) + list(params.values()):
                p.grad = None
            torch.cuda.empty_cache()
    for arm in ("engine", "cudnn"):
        ms, fl, by = tot[arm]
        t_c, t_m = fl / PEAK[arm], by / BW
        frac = max(t_c, t_m) / (ms * 1e-3)
        bound = "tensor" if t_c >= t_m else "memory"
        res[arm] = dict(ms=ms, gflop=fl / 1e9, mb=by / 1e6, bound=bound, roofline=frac)
        print(f"{'total':>6} {arm:>7} {ms:>9.2f} {fl / 1e9:>9.1f} {by / 1e6:>9.1f} {bound:>8} {frac:>9.3f}")
    res["cudnn_over_engine"] = tot["cudnn"][0] / tot["engine"][0]
    print(f"cuDNN TF32 time / engine time: {res['cudnn_over_engine']:.2f}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

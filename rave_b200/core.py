"""Loss helpers -- the subset of rave/core.py the training step calls (SURVEY.md section 8f.1,
a "next" row: cuFFT-backed `torch.stft` + elementwise reductions run on the device through
PyTorch for now; the conv / PQMF hot path they consume is native).
"""
from typing import Callable, Optional, Sequence

import numpy as np
import torch
import torch.nn as nn


def mod_sigmoid(x):
    return 2 * torch.sigmoid(x) ** 2.3 + 1e-7


def get_augmented_latent_size(latent_size: int, noise_augmentation: int):
    return latent_size + noise_augmentation


def hinge_gan(score_real, score_fake):
    """rave/core.py:151-155."""
    loss_dis = (torch.relu(1 - score_real) + torch.relu(1 + score_fake)).mean()
    loss_gen = -score_fake.mean()
    return loss_dis, loss_gen


def ls_gan(score_real, score_fake):
    loss_dis = ((score_real - 1).pow(2) + score_fake.pow(2)).mean()
    loss_gen = (score_fake - 1).pow(2).mean()
    return loss_dis, loss_gen


def nonsaturating_gan(score_real, score_fake):
    score_real = torch.clamp(torch.sigmoid(score_real), 1e-7, 1 - 1e-7)
    score_fake = torch.clamp(torch.sigmoid(score_fake), 1e-7, 1 - 1e-7)
    loss_dis = -(torch.log(score_real) + torch.log(1 - score_fake)).mean()
    loss_gen = -torch.log(score_fake).mean()
    return loss_dis, loss_gen


def valid_signal_crop(x, left_rf, right_rf):
    """rave/core.py:220-225."""
    dim = x.shape[1]
    x = x[..., left_rf.item() // dim:]
    if right_rf.item():
        x = x[..., :-right_rf.item() // dim]
    return x


def mean_difference(target, value, norm: str = "L1", relative: bool = False):
    """rave/core.py:236-252.  L1 on CUDA fp32 tensors: both sums from one library pass (ops.l1_stats)."""
    if (norm == "L1" and target.is_cuda and target.dtype == torch.float32 and value.dtype == torch.float32
            and target.shape == value.shape and target.numel() > 0):
        from . import ops
        st = ops.l1_stats(target, value)
        return st[0] / st[1] if relative else st[0] / target.numel()
    diff = target - value
    if norm == "L1":
        diff = diff.abs().mean()
        if relative:
            diff = diff / target.abs().mean()
        return diff
    elif norm == "L2":
        diff = (diff * diff).mean()
        if relative:
            diff = diff / (target * target).mean()
        return diff
    raise Exception(f"Norm must be either L1 or L2, got {norm}")


def mean_difference_halves(base, n_true: int, relative: bool = False):
    """mean_difference(real, fake, 'L1', relative) where real / fake are the two halves (dim 0) of ONE dense fp32 buffer
    whose padding (if any) is zero in both halves; `n_true` = the number of real feature elements (the mean's
    denominator, rave/core.py:244)."""
    from . import ops
    st = ops.l1_halves(base)
    return st[0] / st[1] if relative else st[0] / n_true


_STACKED_WEIGHTS = {}


def stacked_l1_terms(tapped, relative: bool = False):
    """sum_i w_i * mean_difference_i for features whose (sum |real - fake|, sum |real|) pairs already exist:
    `tapped` = [(sums[2], n_true, w)].  One stack, one multiply (or divide + multiply), one sum -- instead of a scalar
    division and an addition (and their backward launches) per feature.  The constant weight vector lives on the device,
    built once per (device, weights) outside any stream capture."""
    S = torch.stack([t[0] for t in tapped])                                  # [n, 2]
    key = (str(S.device), bool(relative), tuple((int(t[1]), float(t[2])) for t in tapped))
    w = _STACKED_WEIGHTS.get(key)
    if w is None:
        if S.is_cuda and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("stacked_l1_terms: first call for these features inside a stream capture (run one eager "
                               "step first: the weight vector is uploaded once)")
        vals = [t[2] if relative else t[2] / t[1] for t in tapped]
        w = _STACKED_WEIGHTS[key] = torch.tensor(vals, dtype=torch.float64).to(S.dtype).to(S.device)
    if relative:
        return ((S[:, 0] / S[:, 1]) * w).sum()
    return (S[:, 0] * w).sum()


class _StftWindow(nn.Module):
    """Holder of one scale's hann window (`stfts.<i>.window`, the key torchaudio.transforms.Spectrogram contributes)."""

    def __init__(self, n_fft: int) -> None:
        super().__init__()
        self.n_fft = n_fft
        self.register_buffer("window", torch.hann_window(n_fft))


class MultiScaleSTFT(nn.Module):
    """rave/core.py:269-319 (magnitude spectrogram, hann window, hop = n_fft/4, centred)."""

    def __init__(self, scales: Sequence[int], sample_rate: int, magnitude: bool = True,
                 normalized: bool = False, num_mels: Optional[int] = None) -> None:
        super().__init__()
        if num_mels is not None:
            raise NotImplementedError("mel scales need librosa, absent here; not used by v2/v3/discrete")
        self.scales = scales
        self.magnitude = magnitude
        self.normalized = normalized
        # the reference keeps one torchaudio Spectrogram per scale in `self.stfts` (rave/core.py:283-296), whose hann
        # `window` buffers are part of RAVE.state_dict(): same names here
        self.stfts = nn.ModuleList([_StftWindow(s) for s in scales])
        for s in scales:
            bw = torch.full((s // 2 + 1,), 0.5 * s)       # rfft backward as one c2r transform (ops.RfftFn)
            bw[0] = s
            bw[-1] = s
            self.register_buffer(f"rfft_bw_{s}", bw, persistent=False)

    def __getattr__(self, name):
        if name.startswith("window_"):                  # window_<n_fft>: the persistent buffer stfts[i].window
            s = int(name[7:])
            return self.stfts[list(self.scales).index(s)].window
        return super().__getattr__(name)

    def complex_stfts(self, x):
        x = x.reshape(-1, x.shape[-1])
        if x.is_cuda and x.dtype == torch.float32 and not self.normalized:
            # library framing kernel (pad + frame + window; adjoint = window + overlap-add + fold) and cuFFT for
            # the transform; like torch.stft the result is a [N, bins, frames] view of a [N, frames, bins] buffer
            from . import ops
            if all(x.shape[-1] > s // 2 for s in self.scales):
                return [ops.rfft(ops.stft_frames(x, getattr(self, f"window_{s}"), s, s // 4),
                                 getattr(self, f"rfft_bw_{s}")).transpose(-1, -2) for s in self.scales]
        return [torch.stft(x, s, hop_length=s // 4, win_length=s, window=getattr(self, f"window_{s}"),
                           center=True, pad_mode="reflect", normalized=self.normalized, onesided=True,
                           return_complex=True) for s in self.scales]

    def forward(self, x):
        return [y.abs() if self.magnitude else torch.stack([y.real, y.imag], -1) for y in self.complex_stfts(x)]


def htk_mel_filterbank(sample_rate: int, n_fft: int, n_mels: int) -> torch.Tensor:
    """[n_fft // 2 + 1, n_mels] triangular HTK filter bank, norm=None, f_min = 0, f_max = sample_rate // 2: the `fb`
    buffer of torchaudio.transforms.MelScale (torchaudio.functional.melscale_fbanks), computed in numpy."""
    # float32 throughout, as torchaudio computes it: the zero pattern (which bins feed which band) is then the same
    f32 = np.float32
    n_freqs = n_fft // 2 + 1
    all_freqs = np.linspace(0.0, float(sample_rate // 2), n_freqs).astype(f32)
    m_max = 2595.0 * np.log10(1.0 + (sample_rate // 2) / 700.0)
    m_pts = np.linspace(0.0, m_max, n_mels + 2).astype(f32)
    f_pts = f32(700.0) * (f32(10.0) ** (m_pts / f32(2595.0)) - f32(1.0))
    f_diff = f_pts[1:] - f_pts[:-1]
    slopes = f_pts[None, :] - all_freqs[:, None]
    down = -slopes[:, :-2] / f_diff[:-1]
    up = slopes[:, 2:] / f_diff[1:]
    return torch.from_numpy(np.maximum(f32(0.0), np.minimum(down, up)).astype(f32))


class _MelStft(nn.Module):
    """Holder of the periodic hann window (`spectrogram.window` of torchaudio.transforms.Spectrogram)."""

    def __init__(self, n_fft: int) -> None:
        super().__init__()
        self.register_buffer("window", torch.hann_window(n_fft))


class _MelScale(nn.Module):
    """Holder of the filter bank (`mel_scale.fb` of torchaudio.transforms.MelScale)."""

    def __init__(self, fb: torch.Tensor) -> None:
        super().__init__()
        self.register_buffer("fb", fb)


class MelSpectrogram(nn.Module):
    """torchaudio.transforms.MelSpectrogram(sr, n_fft, win_length=n_fft, hop_length, normalized=True, n_mels) as the
    hybrid configuration binds it (configs/hybrid.gin), fused with what RAVE._mel_encode does next
    (rave/model.py:238-242): `encode_log1p(x)` = log1p(mel(x)[..., :-1]) reshaped to [B, C * n_mels, frames - 1].
    Periodic hann window, centred reflect-padded frames, |X|^2 / sum(w^2), HTK bands.  Forward only: the encoder's
    input needs no gradient.  Same sub-modules / buffers as torchaudio's, so reference checkpoints load."""

    def __init__(self, sample_rate: int, n_fft: int = 2048, win_length: Optional[int] = None,
                 hop_length: Optional[int] = None, normalized: bool = True, n_mels: int = 128) -> None:
        super().__init__()
        if (win_length or n_fft) != n_fft or not normalized:
            raise NotImplementedError("MelSpectrogram: only win_length = n_fft and normalized=True are on the hot path")
        self.n_fft, self.hop_length, self.n_mels = n_fft, hop_length or n_fft // 2, n_mels
        self.spectrogram = _MelStft(n_fft)
        self.mel_scale = _MelScale(htk_mel_filterbank(sample_rate, n_fft, n_mels))

    def band_table(self):
        """(band [n_mels, 3] int32 = lo, hi, offset; packed weights) of the current `fb`, on its device; rebuilt only
        when the buffer changes (load_state_dict), so a captured step reads the same tensors."""
        fb = self.mel_scale.fb
        hit = self.__dict__.get("_bands")
        if hit is not None and hit[0] is fb and hit[1] == fb._version:
            return hit[2]
        if fb.is_cuda and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("MelSpectrogram: run one eager step before capturing a CUDA graph")
        f = fb.detach().cpu()
        rows, wts, off = [], [], 0
        for m in range(f.shape[1]):
            nz = torch.nonzero(f[:, m]).reshape(-1)
            lo, hi = (int(nz[0]), int(nz[-1]) + 1) if nz.numel() else (0, 0)
            rows.append((lo, hi, off))
            wts.append(f[lo:hi, m])
            off += hi - lo
        w = torch.cat(wts) if off else torch.zeros(1)
        table = (torch.tensor(rows, dtype=torch.int32).to(fb.device), w.contiguous().to(fb.device))
        self.__dict__["_bands"] = (fb, fb._version, table)
        return table

    def encode_log1p(self, x: torch.Tensor) -> torch.Tensor:
        from . import ops
        batch, channels, T = x.shape
        w = self.spectrogram.window
        if x.requires_grad and torch.is_grad_enabled():
            # differentiable path (the receptive-field probe): framing, rfft and the mel reduction each with their
            # library backward; training never asks for the input gradient and keeps the no-grad path below
            X = ops.rfft(ops.stft_frames(x.reshape(-1, T), w, self.n_fft, self.hop_length), self._rfft_bw())
            band, wts = self.band_table()
            return ops.MelLog1pFn.apply(X, band, wts, self.n_mels, 1.0 / float(self._win_energy()), batch, channels)
        with torch.no_grad():
            frames = ops.stft_frames(x.detach().reshape(-1, T), w, self.n_fft, self.hop_length)
            X = torch.fft.rfft(frames)
            band, wts = self.band_table()
            return ops.mel_log1p(X, band, wts, self.n_mels, 1.0 / float(self._win_energy()), batch, channels)

    def _rfft_bw(self):
        """Bin weights of ops.rfft's backward for n_fft (MultiScaleSTFT.rfft_bw_<n>), on the window's device."""
        w = self.spectrogram.window
        hit = self.__dict__.get("_rfft_bw_cache")
        if hit is None or hit.device != w.device:
            bw = torch.full((self.n_fft // 2 + 1,), 0.5 * self.n_fft)
            bw[0] = bw[-1] = self.n_fft
            hit = self.__dict__["_rfft_bw_cache"] = bw.to(w.device)
        return hit

    def _win_energy(self):
        w = self.spectrogram.window
        hit = self.__dict__.get("_energy")
        if hit is None or hit[0] is not w or hit[1] != w._version:
            hit = self.__dict__["_energy"] = (w, w._version, float(w.detach().double().square().sum().cpu()))
        return hit[2]


class AudioDistanceV1(nn.Module):
    """rave/core.py:322-344."""

    def __init__(self, multiscale_stft: Callable[[], nn.Module], log_epsilon: float) -> None:
        super().__init__()
        self.multiscale_stft = multiscale_stft()
        self.log_epsilon = log_epsilon

    def forward(self, x, y):
        mstft = self.multiscale_stft
        if (x.is_cuda and not x.requires_grad and isinstance(mstft, MultiScaleSTFT) and mstft.magnitude
                and x.dtype == torch.float32):
            # fused path: one kernel per scale for the whole |.|, log, L2-relative + L1 tail (and one for its
            # gradient) instead of ~40 ATen launches; cuFFT still does the transforms
            from . import ops
            distance = 0.
            for sx, sy in zip(mstft.complex_stfts(x), mstft.complex_stfts(y)):
                distance = distance + ops.spectral_distance(sx, sy, self.log_epsilon)
            return {"spectral_distance": distance}
        stfts_x = self.multiscale_stft(x)
        stfts_y = self.multiscale_stft(y)
        distance = 0.
        for sx, sy in zip(stfts_x, stfts_y):
            logx = torch.log(sx + self.log_epsilon)
            logy = torch.log(sy + self.log_epsilon)
            distance = distance + mean_difference(sx, sy, norm="L2", relative=True) \
                + mean_difference(logx, logy, norm="L1")
        return {"spectral_distance": distance}


def _is_recurrent(module) -> bool:
    """The modules rave/core.py:186-188 switches off for the probe (a recurrence makes the gradient's support unbounded)."""
    return hasattr(module, "gru_state") or hasattr(module, "temporal")


@torch.enable_grad()
def get_rave_receptive_field(model, n_channels=1):
    """rave/core.py:180-217: support of the input gradient of one output sample, doubling the probe length until both
    ends of the gradient are zero.  Recurrent modules are disabled for the probe; the probe runs on the fp32 kernels and
    the dense PQMF tables (exact non-zero counts, the reference's fp32 measurement) in eval mode.  The input gradient is taken with
    torch.autograd.grad, so no parameter `.grad` is created or cleared.  Precision, training flag and the recurrent
    modules are restored afterwards."""
    from . import engine, pqmf
    N = 2 ** 15
    device = next(iter(model.parameters())).device
    was_training, precision = model.training, engine.precision()
    recurrent = [m for m in model.modules() if _is_recurrent(m)]
    banks = [m for m in model.modules() if isinstance(m, pqmf.PQMF)]
    model.eval()
    engine.set_precision("fp32")
    for m in recurrent:
        m.disable()
    for m in banks:
        m.exact_taps = True
    try:
        while True:
            x = torch.randn(1, model.n_channels, N, requires_grad=True, device=device)
            z = model.encode(x)
            z = model.encoder.reparametrize(z)[0]
            y = model.decode(z)
            (grad,) = torch.autograd.grad(y[0, 0, N // 2], x, allow_unused=True)
            if grad is None:
                raise RuntimeError("get_rave_receptive_field: the output does not depend on the input (an encoder "
                                   "that detaches its output, e.g. a VariationalEncoder in phase 2)")
            left_grad, right_grad = grad.reshape(-1).chunk(2, 0)
            if left_grad[0] == 0 and right_grad[-1] == 0:
                break
            N *= 2
        left_rf = int((left_grad != 0).sum())
        right_rf = int((right_grad != 0).sum())
    finally:
        for m in recurrent:
            m.enable()
        for m in banks:
            m.exact_taps = False
        engine.set_precision(precision)
        model.train(was_training)
    return left_rf, right_rf


def latent_analysis(means: Sequence[torch.Tensor], latent_size: int):
    """The latent PCA of RAVE.validation_epoch_end (rave/model.py:464-488) over the posterior means [B, D, L] of an
    epoch, taken in list order: (latent_mean [D], components [D, D] (rows), fidelity [D]), all fp32.

    One rave_latent_moments per tensor accumulates the fp64 count, mean and centred scatter (Chan's merge: no
    X^T X - n m m^T cancellation on channels whose mean is large against their spread); the covariance M2 / (n - 1) is
    diagonalised once on the device in fp64.  Order and signs follow sklearn's PCA: eigenvalues descending, negatives
    clipped to zero, each component flipped so that its largest-magnitude entry is positive."""
    from . import ops
    D = int(latent_size)
    n = sum(int(m.shape[0]) * int(m.shape[-1]) for m in means)          # rows, from shapes: no device read
    if n < D:
        raise ValueError(f"latent_analysis: {n} latent rows for {D} components (PCA needs at least as many rows)")
    state = torch.zeros(1 + D + D * D, dtype=torch.float64, device=means[0].device)
    for m in means:
        ops.latent_moments(m, D, state)
    mean = state[1:1 + D]
    cov = state[1 + D:].reshape(D, D) / (n - 1)
    ev, vec = torch.linalg.eigh(cov)
    ev = ev.flip(0).clamp_min(0)
    comps = vec.flip(1).T.contiguous()
    pivot = comps.gather(1, comps.abs().argmax(1, keepdim=True))
    comps = comps * torch.where(pivot < 0, -1.0, 1.0)
    fidelity = torch.cumsum(ev / ev.sum(), 0)
    return mean.float(), comps.float(), fidelity.float()


# ---------------------------------------------------------------------------------------------
# FFT noise filtering helpers of NoiseGeneratorV2 (rave/core.py:48-81) -- cuFFT through torch,
# SURVEY row 8f.4 ("next"); the strided convs that feed them are on the library kernels.
# ---------------------------------------------------------------------------------------------

def amp_to_impulse_response(amp, target_size):
    """Zero-phase band amplitudes -> windowed, causal-shifted FIR of length `target_size`."""
    spec = torch.complex(amp, torch.zeros_like(amp))
    ir = torch.fft.irfft(spec)
    n = ir.shape[-1]
    ir = torch.roll(ir, n // 2, -1) * torch.hann_window(n, dtype=ir.dtype, device=ir.device)
    ir = nn.functional.pad(ir, (0, int(target_size) - int(n)))
    return torch.roll(ir, -n // 2, -1)


def fft_convolve(signal, kernel):
    """Linear convolution on the last axis via zero-padded rFFT, keeping the last half."""
    signal = nn.functional.pad(signal, (0, signal.shape[-1]))
    kernel = nn.functional.pad(kernel, (kernel.shape[-1], 0))
    out = torch.fft.irfft(torch.fft.rfft(signal) * torch.fft.rfft(kernel))
    return out[..., out.shape[-1] // 2:]

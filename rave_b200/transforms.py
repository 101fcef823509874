"""Training-batch transforms on the device: the reference's per-example dataset pipeline (`get_dataset`,
rave/dataset.py:207-262) on a collated batch of database chunks, in one CUDA kernel (csrc/augment.cu).

    transforms = get_transforms(sr=44100, n_signal=131072, normalize=True, augmentations=[RandomMute(0.1)])
    x = transforms(raw)            # raw [B, C, L] int16 or float32 on the GPU -> [B, C, n_signal] float32

Per example, in the reference's order: int16 -> float32 / 32767, RandomCrop(n_signal), RandomApply(p=.8) of
random_phase_mangle(x, 20, 2000, .99, sr_dataset), Dequantize(16), normalize_signal (option), the derivator (option),
the augmentations, the float32 cast.  All channels of an example share its draws.  The per-example draws come from the
current CUDA generator and the dequantisation noise from a counter-based Philox keyed by two integers drawn from it, so
a call never synchronises with the host and can be captured in a CUDA graph.
"""
import math
from typing import Iterable, Optional

import torch

from . import ops

PHASE_P = 0.8                       # RandomApply(random_phase_mangle, p=.8)
PHASE_MIN_F, PHASE_MAX_F = 20.0, 2000.0


class RandomMute:
    """RandomMute(prob) of rave/transforms.py:169-178: the whole example is multiplied by one Bernoulli(1 - prob)."""

    def __init__(self, prob: float = 0.1):
        assert 0. <= prob <= 1., "prob must be between 0. and 1."
        self.prob = prob


class RandomGain:
    """RandomGain of rave/transforms.py:148-166.  The reference computes a gain and returns its input unchanged, so this
    transform is the identity (DESIGN §5.9, quirk D10)."""

    def __init__(self, gain_range=(-6, 3), prob: float = 0.5, limit=True):
        assert 0. <= prob <= 1., "prob must be between 0. and 1."
        self.gain_range = gain_range
        self.prob = prob
        self.limit = limit


_NOT_BUILT = {
    "Compress": "sox `compand`, whose arithmetic cannot be pinned without sox",
    "RandomCompress": "sox `compand`, whose arithmetic cannot be pinned without sox",
    "FrequencyMasking": "no configuration of the reference uses it",
    "RandomPitch": "resample_poly with a random ratio is not built",
    "Resample": "resampling is not built",
}


def _keep_probability(augmentations) -> float:
    """P(keep) of the augmentations: the product of 1 - prob of every RandomMute (RandomGain is the identity).
    Augmentations are matched by class name, so the reference's own objects are accepted too."""
    keep = 1.0
    for a in augmentations:
        name = type(a).__name__
        if name == "RandomMute":
            keep *= 1.0 - float(a.prob)
        elif name == "RandomGain":
            pass
        elif name in _NOT_BUILT:
            raise NotImplementedError(f"{name}: {_NOT_BUILT[name]}")
        else:
            raise NotImplementedError(f"augmentation {name} is not built")
    return keep


def sample_draws(B: int, L: int, n_signal: int, sr: float, keep_prob: float = 1.0, device=None,
                 generator: Optional[torch.Generator] = None) -> torch.Tensor:
    """Per-example choices [B, 4] float64 = (crop offset, allpass applied, omega, keep) from B x 4 uniforms of
    `generator` (the current default generator of `device` when None):
      offset uniform in [0, L - n_signal], both ends inclusive (random.randint);
      applied with probability .8 (random() < p);
      omega = 2 pi f / sr, f log-uniform in [20, 2000] Hz (random_angle);
      keep with probability keep_prob (RandomMute's Bernoulli(1 - prob), all mutes combined)."""
    u = torch.rand(B, 4, dtype=torch.float64, device=device, generator=generator)
    span = L - n_signal
    lo, hi = math.log(PHASE_MIN_F), math.log(PHASE_MAX_F)
    return torch.stack([
        torch.floor(u[:, 0] * (span + 1)).clamp_(max=span),
        (u[:, 1] < PHASE_P).double(),
        torch.exp(u[:, 2] * (hi - lo) + lo) * (2 * math.pi) / sr,
        (u[:, 3] < keep_prob).double(),
    ], 1)


class Transforms:
    """The callable get_transforms returns."""

    def __init__(self, sr_dataset: int, n_signal: int, derivative: bool, normalize: bool, keep_prob: float,
                 n_channels: int):
        self.sr_dataset = sr_dataset
        self.n_signal = n_signal
        self.derivative = bool(derivative)
        self.normalize = bool(normalize)
        self.keep_prob = keep_prob
        self.n_channels = n_channels

    def __call__(self, raw: torch.Tensor, draws: Optional[torch.Tensor] = None, noise: Optional[torch.Tensor] = None,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """raw [B, n_channels, L] int16 (database chunks) or float32 on the GPU, L >= n_signal -> [B, n_channels,
        n_signal] float32, written into `out` when given (e.g. a GraphedTrainer's x_static).  `draws` [B, 4] float64
        replaces the sampled choices (sample_draws' layout) and `noise` [B, C, n_signal] float64 in [0, 1) the
        dequantisation uniforms."""
        if not isinstance(raw, torch.Tensor) or not raw.is_cuda:
            raise ValueError("transforms: raw must be a CUDA tensor")
        if raw.dtype not in (torch.int16, torch.float32):
            raise TypeError(f"transforms: raw must be int16 or float32, not {raw.dtype}")
        if raw.dim() != 3 or raw.shape[1] != self.n_channels:
            raise ValueError(f"transforms: raw must be [B, {self.n_channels}, L], got {tuple(raw.shape)}")
        B, C, L = raw.shape
        N = self.n_signal
        if L < N:
            raise ValueError(f"transforms: chunks of {L} samples are shorter than n_signal = {N}")
        if draws is None:
            draws = sample_draws(B, L, N, self.sr_dataset, self.keep_prob, device=raw.device)
        elif draws.shape != (B, 4) or draws.dtype != torch.float64 or draws.device != raw.device:
            raise ValueError("transforms: draws must be [B, 4] float64 on raw's device")
        if noise is not None and (noise.shape != (B, C, N) or noise.dtype != torch.float64
                                  or noise.device != raw.device):
            raise ValueError(f"transforms: noise must be [{B}, {C}, {N}] float64 on raw's device")
        if out is None:
            out = torch.empty(B, C, N, dtype=torch.float32, device=raw.device)
        elif (out.shape != (B, C, N) or out.dtype != torch.float32 or out.device != raw.device
              or not out.is_contiguous()):
            raise ValueError(f"transforms: out must be a contiguous [{B}, {C}, {N}] float32 tensor on raw's device")
        key = torch.randint(0, 1 << 62, (2,), dtype=torch.int64, device=raw.device)
        return ops.augment(raw.contiguous(), draws.contiguous(), key, out,
                           None if noise is None else noise.contiguous(), self.normalize, self.derivative)


def get_transforms(sr: int, n_signal: int, sr_dataset: Optional[int] = None, derivative: bool = False,
                   normalize: bool = False, rand_pitch=False, augmentations: Iterable = (),
                   n_channels: int = 1) -> Transforms:
    """The transform list of get_dataset(db_path, sr, n_signal, derivative, normalize, rand_pitch, augmentations,
    n_channels) for a database recorded at sr_dataset (its metadata's `sr`; None: sr)."""
    if rand_pitch:
        raise NotImplementedError(f"rand_pitch: RandomPitch: {_NOT_BUILT['RandomPitch']}")
    if sr_dataset is None:
        sr_dataset = sr
    if sr_dataset != sr:
        raise NotImplementedError(f"sr_dataset {sr_dataset} != sr {sr}: Resample: {_NOT_BUILT['Resample']}")
    keep_prob = _keep_probability(list(augmentations or ()))
    return Transforms(sr_dataset, n_signal, derivative, normalize, keep_prob, n_channels)

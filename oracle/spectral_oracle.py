"""TEST INFRASTRUCTURE -- restatement of the multi-scale spectral discriminator (rave/discriminator.py:12-74, 139-153;
configs/spectral_discriminator.gin) and of the training-step arithmetic with it, in plain torch, built on
oracle/rave_oracle.py.  Pinned against the unmodified reference by oracle/make_golden_spectral.py
(tests/golden/*spectral*.pt).

The fixtures are kept small: parameters of the training-step fixture are regenerated from a seed (seeded_params),
inputs from their seeds (step_batch / step_eps), and feature maps and gradients are stored as fixed seeded samples
(oracle/make_reference_pins.py::sample)."""
import math
from typing import List

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle import rave_oracle as O
from oracle.make_reference_pins import sample  # noqa: F401  (re-exported for the tests)

SCALES = (4096, 2048, 1024, 512, 256)          # configs/spectral_discriminator.gin:7
# (stride, dilation) of the six EncodecConvNet blocks, rave/discriminator.py:58-67
ENCODEC_GEOMETRY = [((1, 1), (1, 1)), ((2, 1), (1, 1)), ((2, 1), (1, 2)), ((2, 1), (1, 4)), ((1, 1), (1, 1)),
                    ((1, 1), (1, 1))]


def spectrogram(x: Tensor, n_fft: int) -> Tensor:
    """torchaudio Spectrogram(n_fft, hop_length=n_fft // 4, power=None, normalized=True, center=False)
    (rave/discriminator.py:12-20): hann (periodic) window, no padding, divided by ||window||_2; [B, C, F, T] complex."""
    B, C, T = x.shape
    win = torch.hann_window(n_fft, dtype=x.dtype, device=x.device)
    s = torch.stft(x.reshape(B * C, T), n_fft, hop_length=n_fft // 4, win_length=n_fft, window=win,
                   center=False, normalized=False, onesided=True, return_complex=True)
    s = s / win.pow(2.).sum().sqrt()
    return s.reshape(B, C, s.shape[-2], s.shape[-1])


def encodec_convnet(x: Tensor, sd, prefix: str) -> List[Tensor]:
    """EncodecConvNet (rave/discriminator.py:54-74) on [B, 2C, F, T]: rectified_2d_conv_block (23-51) = weight-normed
    Conv2d + LeakyReLU(.2); kernels (9, 3) x 4 then (3, 3) x 2, padding (k - 1) * dilation // 2.  Features are
    POST-activation; the last block (one channel, no activation) is the score."""
    feats = []
    for i, (stride, dil) in enumerate(ENCODEC_GEOMETRY):
        last = i == len(ENCODEC_GEOMETRY) - 1
        q = f"{prefix}net.{i}." if last else f"{prefix}net.{i}.0."
        w = O.wn_weight(sd, q)
        kf, kt = w.shape[2], w.shape[3]
        pad = ((kf - 1) * dil[0] // 2, (kt - 1) * dil[1] // 2)
        x = F.conv2d(x, w, sd[q + "bias"], stride, pad, dil)
        if not last:
            x = O.leaky_relu(x, 0.2)
        feats.append(x)
    return feats


def multi_scale_spectral_discriminator(x: Tensor, sd, prefix: str, scales=SCALES) -> List[List[Tensor]]:
    """rave/discriminator.py:139-153: per scale, cat([re, im], 1) of the spectrogram through its own EncodecConvNet."""
    out = []
    for i, n in enumerate(scales):
        s = spectrogram(x, n)
        out.append(encodec_convnet(torch.cat([s.real, s.imag], 1), sd, f"{prefix}nets.{i}."))
    return out


def combine_discriminators_v2_spectral(x: Tensor, sd, prefix: str = "discriminator.",
                                       scales=SCALES) -> List[List[Tensor]]:
    """CombineDiscriminators[MSD, MultiScaleSpectralDiscriminator] (configs/spectral_discriminator.gin:13-17 on top of
    configs/v2.gin; rave/discriminator.py:198-209)."""
    feats = O.multi_scale_discriminator(x, sd, prefix + "discriminators.0.")
    feats.extend(multi_scale_spectral_discriminator(x, sd, prefix + "discriminators.1.", scales))
    return feats


def train_step_losses(x: Tensor, sd, cfg: O.ArchConfig, eps: Tensor, receptive_field=(0, 0), fm_weight: float = 20.0):
    """Phase-2 forward arithmetic of RAVE.training_step (rave/model.py:292-399) with the MSD + spectral discriminator:
    (logged loss_gen terms, loss_dis), as oracle/rave_oracle.py::train_step_losses computes them for v2."""
    hk = sd["pqmf.hk"]
    x_mb = O.pqmf_encode(x, hk, cfg.pad_mode)
    z = O.encoder_v2(x_mb, sd, "encoder.encoder.", cfg).detach()      # warmed up: blocks.py:743-744
    zs, reg = O.reparametrize(z, eps)
    y_mb = O.generator_v2(zs, sd, "decoder.", cfg)
    y = O.pqmf_decode(y_mb, hk, cfg.n_channels, cfg.pad_mode)[..., :x.shape[-1]]
    y_mb = y_mb[..., :x_mb.shape[-1]]
    x_mb_c, y_mb_c = x_mb, y_mb
    if receptive_field[0] + receptive_field[1]:
        x_mb_c = O.valid_signal_crop(x_mb, *receptive_field)
        y_mb_c = O.valid_signal_crop(y_mb, *receptive_field)
    fm, loss_dis, loss_adv = O.gan_losses(combine_discriminators_v2_spectral(torch.cat([x, y], 0), sd), 1, True)
    losses = {
        "multiband_spectral_distance": O.audio_distance_v1(x_mb_c, y_mb_c),
        "fullband_spectral_distance": O.audio_distance_v1(x, y),
        "regularization": reg,
        "feature_matching": fm_weight * fm,
        "adversarial": loss_adv,
    }
    return losses, loss_dis


def step_batch(B: int, T: int, seed: int) -> Tensor:
    """The training-step fixture's batch (oracle/make_golden.py::make_input with seed 500 + seed)."""
    g = torch.Generator(device="cpu").manual_seed(500 + seed)
    return (0.5 * torch.randn(B, 1, T, generator=g)).clamp(-1, 1)


def step_eps(B: int, latent: int, Lz: int, seed: int) -> Tensor:
    """The reparametrisation noise the reference's training_step draws first after torch.manual_seed(seed)."""
    return torch.randn(B, latent, Lz, generator=torch.Generator().manual_seed(seed))


def seeded_params(shapes, seed):
    """{key: tensor} drawn in key order from one CPU generator at the scale of a default initialisation: weights
    N(0, 1 / fan_in), biases N(0, 0.01^2), and every weight-norm magnitude `weight_g` set to the norm of its direction
    `weight_v` (the effective weight is then weight_v, as right after torch.nn.utils.weight_norm)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for k, s in shapes:
        s = tuple(s)
        fan_in = math.prod(s[1:]) if len(s) > 1 else 1
        scale = 1.0 / math.sqrt(fan_in) if len(s) > 1 else 0.01
        out[k] = torch.randn(s, generator=g) * scale
    for k in out:
        if k.endswith("weight_g"):
            v = out[k[:-1] + "v"]
            out[k] = v.reshape(v.shape[0], -1).norm(dim=1).reshape(out[k].shape)
    return out

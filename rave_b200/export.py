"""`ExportedRAVE`: the compact latent interface of a trained model, as the reference's export exposes it
(`ScriptedRAVE` and its four subclasses, scripts/export.py:75-409), without TorchScript or nn~ registration.

`encode` returns the compact latent and `decode` takes one:
  * VariationalEncoder: the posterior sample, centred on `latent_mean`, projected onto the first `latent_size` PCA rows;
    decode fills the dropped dimensions with standard normal noise and inverts the projection;
  * DiscreteEncoder: the residual-VQ codes as floats; decode clamps them, sums the codebook rows and appends the
    `noise_augmentation` noise channels;
  * WasserteinEncoder: encode is the identity; decode appends the noise channels;
  * SphericalEncoder: the `latent_size - 1` hyperspherical angles in [-1, 1) of the raw encoder output; decode maps them
    back to unit vectors.
With a trained `VariationalPrior` of the model (the export's `--prior`), `prior(temp)` generates the prior's latent
frame by frame with its state kept from call to call (scripts/export.py TraceModel, csrc/prior_sample.cu), and
`decode(prior(temp))` plays it.

The latent arithmetic runs on csrc/export.cu.  With `target_sr` (the export's `--sr`), the model runs in a host at
`target_sr = ratio * sr`: encode resamples its input down to the model's rate first, decode resamples the model's output
up before the crop (rave_b200/resampler.py, csrc/resample.cu).  Neither call synchronises with the host, so
`encode` -> `decode` can be captured in a CUDA graph.

Random draws (the posterior's eps, the decode noise) come from the current CUDA generator on the model's device unless
`eps` / `noise` inject them.  The reference draws the decode noise on the CPU: same distribution, different stream (as in
`Prior.decode_classes`).

`set_stereo_mode` is not provided: its batch folding only makes sense inside nn~, which passes the two channels of a
stereo stream as two batch rows.
"""
import math
from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from . import blocks, ops
from .resampler import Resampler


def _kind(encoder) -> str:
    if isinstance(encoder, blocks.VariationalEncoder):
        return "variational"
    if isinstance(encoder, blocks.DiscreteEncoder):
        return "discrete"
    if isinstance(encoder, blocks.WasserteinEncoder):
        return "wasserstein"
    if isinstance(encoder, blocks.SphericalEncoder):
        return "spherical"
    raise ValueError(f"Encoder type {encoder.__class__.__name__} not supported")


def variational_latent_size(fidelity: torch.Tensor, f: float) -> int:
    """scripts/export.py:120-122: the first index whose cumulative explained variance exceeds f (at least 1), rounded
    up to a power of two.  argmax of an all-False mask is 0, so an untrained model (fidelity all zero) gives 1."""
    size = max(int(np.argmax(fidelity.detach().cpu().numpy() > f)), 1)
    return 2 ** math.ceil(math.log2(size))


class ExportedRAVE(nn.Module):
    """The exported model's encode / decode / forward around a trained `RAVE` (put in eval mode, as the export does).

    `channels`: number of output channels of decode (default: the model's).  More than the model has: every example is
    decoded ceil(channels / n_channels) times, each time with its own noise, and the decodes are stacked along the
    channel axis (the reference does this for one example; with a larger batch it slices the batch instead).  Fewer:
    the first channels are kept.  `fidelity`: explained variance that sets `latent_size` of a variational model.
    `target_sr`: the host's sample rate, a multiple of the model's `sr` (ratios 2 and 3 can be built); `sr` becomes
    `target_sr` and `encode_ratio` counts samples at that rate.  `prior`: a `VariationalPrior` trained on this model
    (its `synth`), registered as `prior_module`; `prior(temp)` generates from it.

    Style transfer of a model with AdaIN layers: set `learn_target`, `learn_source`, `reset_target`, `reset_source`;
    they are applied through `RAVE.update_adain` before `encode` and before a `decode` that `forward` did not call, and
    the two resets clear after each application (scripts/export.py:213-230)."""

    def __init__(self, model, channels: Optional[int] = None, fidelity: float = .95, target_sr: Optional[int] = None,
                 prior=None):
        super().__init__()
        model.eval()
        self.model = model
        if prior is not None:
            from .prior import VariationalPrior
            if not isinstance(prior, VariationalPrior):
                raise ValueError(f"prior must be a VariationalPrior, got {prior.__class__.__name__}")
            if prior.synth is not model:
                raise ValueError("the prior was not trained on this model (prior.synth is not model)")
            if prior.latent_size > model.latent_size:
                raise ValueError(f"the prior's latent_size {prior.latent_size} exceeds the model's {model.latent_size}")
            self.prior_module = prior.eval()
        else:
            self.prior_module = None
        self._prior_state = None
        self.resampler = None
        if target_sr is not None and target_sr != model.sr:
            if target_sr % model.sr:
                raise ValueError(f"target_sr {target_sr} is not a multiple of the model's sampling rate {model.sr}")
            self.resampler = Resampler(target_sr, model.sr).to(model.latent_pca.device)
        self.kind = _kind(model.encoder)
        self.n_channels = model.n_channels
        self.target_channels = channels or self.n_channels
        self.full_latent_size = model.latent_size
        self.is_using_adain = any(isinstance(m, blocks.AdaptiveInstanceNormalization) for m in model.modules())
        if self.is_using_adain and self.n_channels != self.target_channels:
            raise ValueError("AdaIN requires the original number of channels")
        self.learn_target = False
        self.learn_source = False
        self.reset_target = False
        self.reset_source = False

        enc = model.encoder
        if self.kind == "variational":
            self.latent_size = variational_latent_size(model.fidelity, fidelity)
            if self.latent_size > self.full_latent_size:
                raise ValueError(f"fidelity {fidelity} gives {self.latent_size} latent dimensions, more than the "
                                 f"model's {self.full_latent_size}")
        elif self.kind == "discrete":
            self.latent_size = enc.num_quantizers
            if any(not isinstance(vq.project_in, nn.Identity) for vq in enc.rvq.layers):
                raise ValueError("the residual VQ's codebook dimension must equal the latent size")
        elif self.kind == "wasserstein":
            self.latent_size = self.full_latent_size
        else:
            self.latent_size = self.full_latent_size - 1
        self.n_noise = getattr(enc, "noise_augmentation", 0) if self.kind in ("discrete", "wasserstein") else 0

        dev = model.latent_pca.device
        x_len = 2 ** 14
        z = self.encode(torch.zeros(1, self.n_channels, x_len, device=dev))
        self.encode_ratio = x_len // z.shape[-1]

    @property
    def sr(self) -> int:
        """The sampling rate encode takes and decode returns: target_sr with a resampler, else the model's."""
        return self.resampler.target_sr if self.resampler is not None else self.model.sr

    # ------------------------------------------------------------------ latent arithmetic
    def _codebooks(self):
        return torch.stack([vq.codebook for vq in self.model.encoder.rvq.layers]).float()

    def post_process_latent(self, z, eps=None):
        z = z.float()
        if self.kind == "variational":
            B, L2, T = z.shape
            eps = self._draw(eps, (B, L2 // 2, T), z.device, "eps")
            return ops.latent_project(z, eps, self.model.latent_mean.float(), self.model.latent_pca.float(),
                                      self.latent_size)
        if self.kind == "discrete":
            return ops.rvq_encode(z, self._codebooks()).float()
        if self.kind == "wasserstein":
            return z
        return ops.sphere_to_angles(z)

    def pre_process_latent(self, z, noise=None):
        z = z.float()
        B, _, T = z.shape
        if self.kind == "variational":
            noise = self._draw(noise, (B, self.full_latent_size - z.shape[1], T), z.device, "noise")
            return ops.latent_unproject(z, noise, self.model.latent_mean.float(), self.model.latent_pca.float())
        if self.kind == "spherical":
            return ops.angles_to_sphere(z)
        noise = self._draw(noise, (B, self.n_noise, T), z.device, "noise") if self.n_noise else None
        if self.kind == "discrete":
            return ops.rvq_decode(z, self._codebooks(), noise)
        return z if noise is None else torch.cat([z, noise], 1)

    @staticmethod
    def _draw(given, shape, device, name):
        if given is None:
            return torch.randn(shape, device=device)
        if tuple(given.shape) != tuple(shape):
            raise ValueError(f"{name} has shape {tuple(given.shape)}, expected {tuple(shape)}")
        return given.to(device=device, dtype=torch.float32)

    # ------------------------------------------------------------------ style transfer flags
    def _update_adain(self):
        self.model.update_adain(self.learn_target, self.learn_source, self.reset_target, self.reset_source)
        self.reset_source = False
        self.reset_target = False

    # ------------------------------------------------------------------ interface
    @torch.no_grad()
    def encode(self, x, eps: Optional[torch.Tensor] = None):
        """x [B, n_channels, N] -> compact latent [B, latent_size, N / encode_ratio].  `eps` [B, L, T]: the posterior's
        standard normal draw of a variational model."""
        if self.is_using_adain:
            self._update_adain()
        if self.resampler is not None:
            x = self.resampler.to_model_sampling_rate(x.float())
        return self.post_process_latent(self.model.encode(x), eps)

    @torch.no_grad()
    def decode(self, z, noise: Optional[torch.Tensor] = None):
        """Compact latent [B, latent_size, T] -> audio [B, target_channels, T * encode_ratio].  `noise`: the draw of
        pre_process_latent for the ceil(target_channels / n_channels) B decoded rows (row b r + i is decode i of
        example b): [B r, L - latent_size, T] (variational) or [B r, noise_augmentation, T]."""
        return self._decode(z, noise, from_forward=False)

    @torch.no_grad()
    def prior(self, temp, uniform: Optional[torch.Tensor] = None, dither: Optional[torch.Tensor] = None):
        """temp [B, 1, T] -> the prior's next T latent frames [B, D, T] float32 (D = prior.latent_size), continuing the
        stream the last call left (scripts/export.py TraceModel.forward at a `--streaming` export).  Each row's
        temperature for the call is softplus(mean_t temp[b, 0, t]) / ln 2 (1 for an input of 0); each step divides the
        logits by it, draws the class by inverse CDF at `uniform` [B, T, D], decodes it with the dither `dither`
        [B, T, D] and shifts it diagonally, so dim d lags the newest frame by D - 1 - d frames (0.0 before the first).
        The draws default to `torch.rand` on the current CUDA generator, uniform first.  The output is in the prior's
        latent coordinates; `decode` fills the other dimensions.  B <= 64 rows, each with its own state; a call whose B
        or device differs from the state's raises ValueError until `reset_prior()`."""
        if self.prior_module is None:
            raise RuntimeError("this ExportedRAVE was built without a prior")
        if temp.dim() != 3 or temp.shape[1] != 1:
            raise ValueError(f"temp has shape {tuple(temp.shape)}, expected [B, 1, T]")
        pm = self.prior_module
        params = pm._trained_parameters()
        B, _, T = temp.shape
        D, dev = pm.latent_size, params[0].device
        if self._prior_state is None:
            if dev.type == "cuda" and torch.cuda.is_current_stream_capturing():
                raise ops._lib.RaveB200Error("prior: the stream is being captured; the state's frame graph is "
                                             "captured and replayed by the call, so it cannot run inside a capture")
            self._prior_state = ops.PriorStream(params, pm.cycle_size, B, pm.quantized_normal.resolution, D)
        elif (self._prior_state.B, self._prior_state.device) != (B, dev):
            raise ValueError(f"the prior's state has {self._prior_state.B} rows on {self._prior_state.device}, the call "
                             f"{B} on {dev}: call reset_prior() first")
        uniform = torch.rand(B, T, D, device=dev) if uniform is None else self._draw(uniform, (B, T, D), dev, "uniform")
        dither = torch.rand(B, T, D, device=dev) if dither is None else self._draw(dither, (B, T, D), dev, "dither")
        return self._prior_state(params, temp.to(device=dev, dtype=torch.float32), uniform, dither)

    def reset_prior(self):
        """Return the prior's generation to its initial state (next call starts a new stream, at any B)."""
        self._prior_state = None

    @torch.no_grad()
    def forward(self, x, eps: Optional[torch.Tensor] = None, noise: Optional[torch.Tensor] = None):
        return self._decode(self.encode(x, eps), noise, from_forward=True)

    def _decode(self, z, noise, from_forward: bool):
        if self.is_using_adain and not from_forward:
            self._update_adain()
        B, T = z.shape[0], z.shape[-1]
        reps = math.ceil(self.target_channels / self.n_channels) if self.target_channels > self.n_channels else 1
        if reps > 1:
            z = z.repeat_interleave(reps, 0)
        y = self.model.decode(self.pre_process_latent(z, noise))
        if self.resampler is not None:
            y = self.resampler.from_model_sampling_rate(y.float())
        if y.shape[-1] > T * self.encode_ratio:
            y = y[..., :T * self.encode_ratio]
        if reps > 1:
            y = y.reshape(B, reps * self.n_channels, y.shape[-1])
        return y[:, :self.target_channels] if self.target_channels != y.shape[1] else y

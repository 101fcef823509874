"""Encoder / generator / latent-head modules -- the module surface of rave/blocks.py with the
arithmetic on librave_b200.so.

Class names, constructor arguments, sub-module layout (hence `state_dict` keys: SURVEY.md
App. B.3) and call signatures follow the reference so that `RAVE(...)` can be assembled from the
same bindings; `forward` never touches an ATen conv: every `activation -> conv (-> + skip)` group
is one kernel launch (see cc.CachedSequential / Residual).
"""
from typing import Callable, Optional, Sequence, Union

import numpy as np
import torch
import torch.nn as nn
from torch.nn.utils.weight_norm import WeightNorm

from . import cc, core, ops
from ._lib import RaveB200Error


# ---------------------------------------------------------------------------------------------
# normalization (rave/blocks.py:15-22; configs/v1.gin:41 binds mode='weight_norm')
# ---------------------------------------------------------------------------------------------

class _config:
    normalization_mode = "weight_norm"


class CudaWeightNorm(WeightNorm):
    """torch.nn.utils.weight_norm's hook object with `compute_weight` on our kernel.  Being a
    `WeightNorm` instance keeps `torch.nn.utils.remove_weight_norm` working
    (tests/test_configs.py:87-89, scripts/export.py:561-563)."""

    def compute_weight(self, module):
        g = getattr(module, self.name + "_g")
        v = getattr(module, self.name + "_v")
        return ops.weight_norm(v, g)

    @staticmethod
    def apply(module, name: str = "weight", dim: int = 0):
        if dim != 0:
            raise RaveB200Error("weight_norm: only dim=0 is on the hot path")
        for hook in module._forward_pre_hooks.values():
            if isinstance(hook, WeightNorm) and hook.name == name:
                raise RuntimeError(f"Cannot register two weight_norm hooks on the same parameter {name}")
        fn = CudaWeightNorm(name, dim)
        weight = getattr(module, name)
        del module._parameters[name]
        with torch.no_grad():
            g = torch.norm_except_dim(weight, 2, dim)   # initialisation only (g = ||v||)
        module.register_parameter(name + "_g", nn.Parameter(g.data))
        module.register_parameter(name + "_v", nn.Parameter(weight.data))
        setattr(module, name, weight.data)               # w == v at init; recomputed every forward
        module.register_forward_pre_hook(fn)
        return fn


def weight_norm(module: nn.Module, name: str = "weight", dim: int = 0) -> nn.Module:
    CudaWeightNorm.apply(module, name, dim)
    return module


def normalization(module: nn.Module, mode: Optional[str] = None):
    mode = mode if mode is not None else _config.normalization_mode
    if mode == "identity":
        return module
    elif mode == "weight_norm":
        return weight_norm(module)
    raise Exception(f"Normalization mode {mode} not supported")


# ---------------------------------------------------------------------------------------------
# activations
# ---------------------------------------------------------------------------------------------

class Snake(nn.Module):
    """x + sin^2(alpha x) / (alpha + 1e-9), alpha [dim, 1] (rave/blocks.py:852-860)."""

    def __init__(self, dim: int) -> None:
        super().__init__()
        self.alpha = nn.Parameter(torch.ones(dim, 1))

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return ops.activation(x, ops.ACT_SNAKE, 0.0, self.alpha.reshape(-1))


def leaky_relu(dim: int, alpha: float):
    return nn.LeakyReLU(alpha)


def _default_activation(dim):
    return nn.LeakyReLU(.2)


class AdaptiveInstanceNormalization(nn.Module):
    """Identity in training (rave/blocks.py:901-902).  In eval mode it learns the running mean / std of its input over
    time as the target (`learn_y`) or source (`learn_x`) statistics, and once both were learned maps the stream from
    source to target statistics: the style transfer, driven by `update_adain`.  `forward` is the reference's arithmetic
    (the fp32 path); the v3 chains on the wgmma engine run it as two kernels per layer (engine.plan_sequential,
    csrc/adain.cu) that read the same buffers and flags on the device."""

    def __init__(self, dim: int) -> None:
        super().__init__()
        for s in ("x", "y"):
            self.register_buffer(f"mean_{s}", torch.zeros(cc.MAX_BATCH_SIZE, dim, 1))
            self.register_buffer(f"std_{s}", torch.ones(cc.MAX_BATCH_SIZE, dim, 1))
            self.register_buffer(f"learn_{s}", torch.zeros(1))
            self.register_buffer(f"num_update_{s}", torch.zeros(1))

    def update(self, target, source, num_updates):
        bs = source.shape[0]
        target[:bs] += (source - target[:bs]) / (num_updates + 1)

    def reset_x(self):
        self.mean_x.zero_()
        self.std_x.zero_().add_(1)
        self.num_update_x.zero_()

    def reset_y(self):
        self.mean_y.zero_()
        self.std_y.zero_().add_(1)
        self.num_update_y.zero_()

    def transfer(self, x):
        bs = x.shape[0]
        x = (x - self.mean_x[:bs]) / (self.std_x[:bs] + 1e-5)
        return x * self.std_y[:bs] + self.mean_y[:bs]

    def forward(self, x):
        if self.training:
            return x
        if self.learn_y:
            self.update(self.mean_y, x.mean(-1, keepdim=True), self.num_update_y)
            self.update(self.std_y, x.std(-1, keepdim=True), self.num_update_y)
            self.num_update_y += 1
            return x
        if self.learn_x:
            self.update(self.mean_x, x.mean(-1, keepdim=True), self.num_update_x)
            self.update(self.std_x, x.std(-1, keepdim=True), self.num_update_x)
            self.num_update_x += 1
        if self.num_update_x and self.num_update_y:
            x = self.transfer(x)
        return x


def update_adain(root: nn.Module, learn_target: bool = False, learn_source: bool = False, reset_target: bool = False,
                 reset_source: bool = False) -> int:
    """Style-transfer controls of every AdaptiveInstanceNormalization under `root` (scripts/export.py:213-230,
    `ScriptedRAVE.update_adain`): both learn flags are cleared, then set from `learn_target` (learn_y) and
    `learn_source` (learn_x); then `reset_target` / `reset_source` restore the y / x statistics and counters.  Only
    in-place device writes (no host sync, no host-to-device copy), so it may sit between the replays of a captured
    CUDA graph.  Returns the number of AdaIN layers touched."""
    n = 0
    for m in root.modules():
        if isinstance(m, AdaptiveInstanceNormalization):
            m.learn_x.zero_()
            m.learn_y.zero_()
            if learn_target:
                m.learn_y.add_(1)
            if learn_source:
                m.learn_x.add_(1)
            if reset_target:
                m.reset_y()
            if reset_source:
                m.reset_x()
            n += 1
    return n


# ---------------------------------------------------------------------------------------------
# residual dilated units (rave/blocks.py:31-45, 83-112)
# ---------------------------------------------------------------------------------------------

class Residual(nn.Module):
    """x + module(x).  When `module` is a DilatedUnit the skip add is fused into the epilogue of
    the unit's last conv kernel."""

    def __init__(self, module, cumulative_delay=0):
        super().__init__()
        additional_delay = module.cumulative_delay
        self.aligned = cc.AlignBranches(module, nn.Identity(), delays=[additional_delay, 0])
        self.cumulative_delay = additional_delay + cumulative_delay

    def forward(self, x):
        module = self.aligned.branches[0]
        if isinstance(module, DilatedUnit) and not self.aligned._cached:
            return module(x, res=x)
        x_net, x_res = self.aligned(x)
        return x_net + x_res


class DilatedUnit(nn.Module):
    """act -> Conv1d(dim, dim, k, dilation) -> act -> Conv1d(dim, dim, 1)."""

    def __init__(self, dim: int, kernel_size: int, dilation: int,
                 activation: Callable[[int], nn.Module] = _default_activation) -> None:
        super().__init__()
        net = [
            activation(dim),
            normalization(cc.Conv1d(dim, dim, kernel_size=kernel_size, dilation=dilation,
                                    padding=cc.get_padding(kernel_size, dilation=dilation))),
            activation(dim),
            normalization(cc.Conv1d(dim, dim, kernel_size=1)),
        ]
        self.net = cc.CachedSequential(*net)
        self.cumulative_delay = net[1].cumulative_delay

    def forward(self, x: torch.Tensor, res: Optional[torch.Tensor] = None) -> torch.Tensor:
        return self.net(x, res=res)


# ---------------------------------------------------------------------------------------------
# v1 architecture (rave/blocks.py:48-240, 322-503; configs/v1.gin).  Not in any BASELINE config: the blocks run on the
# generic library kernels (activation fused into the following conv's operand load, residual add into its epilogue);
# BatchNorm1d / repeat_interleave / stack-sum are the reference's own torch calls.  Same constructor arguments,
# sub-module layout and state_dict keys as the reference.
# ---------------------------------------------------------------------------------------------

class SampleNorm(nn.Module):
    """rave/blocks.py:25-28."""

    def forward(self, x):
        return x / torch.norm(x, 2, 1, keepdim=True)


class ResidualLayer(nn.Module):
    """rave/blocks.py:48-80: x + [act -> Conv1d(dim, dim, k, dilation d)] for d in dilations."""

    def __init__(self, dim, kernel_size, dilations, cumulative_delay=0,
                 activation: Callable[[int], nn.Module] = _default_activation):
        super().__init__()
        net = []
        for d in dilations:
            net.append(activation(dim))
            net.append(normalization(cc.Conv1d(dim, dim, kernel_size, dilation=d,
                                               padding=cc.get_padding(kernel_size, dilation=d))))
        self.net = Residual(cc.CachedSequential(*net), cumulative_delay=cumulative_delay)
        self.cumulative_delay = self.net.cumulative_delay

    def forward(self, x):
        if self.net.aligned._cached:
            return self.net(x)
        # the skip add rides on the epilogue of the last conv (CachedSequential.forward(x, res=x))
        return self.net.aligned.branches[0](x, res=x)


class ResidualBlock(nn.Module):
    """rave/blocks.py:115-141."""

    def __init__(self, dim, kernel_size, dilations_list, cumulative_delay=0) -> None:
        super().__init__()
        layers = [ResidualLayer(dim, kernel_size, dilations) for dilations in dilations_list]
        self.net = cc.CachedSequential(*layers, cumulative_delay=cumulative_delay)
        self.cumulative_delay = self.net.cumulative_delay

    def forward(self, x):
        for layer in self.net:
            x = layer(x)
        return x


class ResidualStack(nn.Module):
    """rave/blocks.py:144-160 (v1.gin:63-65: kernel_sizes [3], dilations_list [[1, 1], [3, 1], [5, 1]])."""

    def __init__(self, dim, kernel_sizes=(3,), dilations_list=((1, 1), (3, 1), (5, 1)), cumulative_delay=0) -> None:
        super().__init__()
        blocks = [ResidualBlock(dim, k, dilations_list) for k in kernel_sizes]
        self.net = cc.AlignBranches(*blocks, cumulative_delay=cumulative_delay)
        self.cumulative_delay = self.net.cumulative_delay

    def forward(self, x):
        x = self.net(x)
        return torch.stack(x, 0).sum(0)


class UpsampleLayer(nn.Module):
    """rave/blocks.py:163-192."""

    def __init__(self, in_dim, out_dim, ratio, cumulative_delay=0,
                 activation: Callable[[int], nn.Module] = _default_activation):
        super().__init__()
        net = [activation(in_dim)]
        if ratio > 1:
            net.append(normalization(cc.ConvTranspose1d(in_dim, out_dim, 2 * ratio, stride=ratio, padding=ratio // 2)))
        else:
            net.append(normalization(cc.Conv1d(in_dim, out_dim, 3, padding=cc.get_padding(3))))
        self.net = cc.CachedSequential(*net)
        self.cumulative_delay = self.net.cumulative_delay + cumulative_delay * ratio

    def forward(self, x):
        return self.net(x)


class NoiseGenerator(nn.Module):
    """rave/blocks.py:195-240 (v1.gin:67-70: ratios [4, 4, 4], noise_bands 5)."""

    def __init__(self, in_size, data_size, ratios=(4, 4, 4), noise_bands=5):
        super().__init__()
        net = []
        channels = [in_size] * len(ratios) + [data_size * noise_bands]
        for i, r in enumerate(ratios):
            net.append(cc.Conv1d(channels[i], channels[i + 1], 3, padding=cc.get_padding(3, r), stride=r))
            if i != len(ratios) - 1:
                net.append(nn.LeakyReLU(.2))
        self.net = cc.CachedSequential(*net)
        self.data_size = data_size
        self.cumulative_delay = 0
        self.register_buffer("target_size", torch.tensor(np.prod(ratios)).long())
        self._target_size = int(np.prod(ratios))          # host copy: no device sync per forward

    def forward(self, x, noise: Optional[torch.Tensor] = None):
        """`noise` (optional, uniform in [-1, 1), shape of the impulse responses) lets a parity test inject the draw."""
        amp = core.mod_sigmoid(self.net(x) - 5)
        amp = amp.permute(0, 2, 1)
        amp = amp.reshape(amp.shape[0], amp.shape[1], self.data_size, -1)
        ir = core.amp_to_impulse_response(amp, self._target_size)
        if noise is None:
            noise = self.__dict__.get("_noise_override")          # parity tests inject the draw (Generator calls forward(x))
        if noise is None:
            noise = torch.rand_like(ir) * 2 - 1
        noise = core.fft_convolve(noise, ir).permute(0, 2, 1, 3)
        return noise.reshape(noise.shape[0], noise.shape[1], -1)


class Generator(nn.Module):
    """rave/blocks.py:322-423 (v1 decoder: upsampling stacks, then waveform / loudness / filtered-noise branches)."""

    def __init__(self, latent_size, capacity, data_size, ratios, loud_stride, use_noise, n_channels: int = 1,
                 recurrent_layer: Optional[Callable[[], nn.Module]] = None):
        super().__init__()
        net = [normalization(cc.Conv1d(latent_size, 2 ** len(ratios) * capacity, 7, padding=cc.get_padding(7)))]
        if recurrent_layer is not None:
            net.append(recurrent_layer(dim=2 ** len(ratios) * capacity, cumulative_delay=0))
        for i, r in enumerate(ratios):
            in_dim = 2 ** (len(ratios) - i) * capacity
            out_dim = 2 ** (len(ratios) - i - 1) * capacity
            net.append(UpsampleLayer(in_dim, out_dim, r))
            net.append(ResidualStack(out_dim))
        self.net = cc.CachedSequential(*net)
        wave_gen = normalization(cc.Conv1d(out_dim, data_size * n_channels, 7, padding=cc.get_padding(7)))
        loud_gen = normalization(cc.Conv1d(out_dim, 1, 2 * loud_stride + 1, stride=loud_stride,
                                           padding=cc.get_padding(2 * loud_stride + 1, loud_stride)))
        branches = [wave_gen, loud_gen]
        if use_noise:
            branches.append(NoiseGenerator(out_dim, data_size * n_channels))
        self.synth = cc.AlignBranches(*branches, cumulative_delay=self.net.cumulative_delay)
        self.use_noise = use_noise
        self.loud_stride = loud_stride
        self.cumulative_delay = self.synth.cumulative_delay
        self.register_buffer("warmed_up", torch.tensor(0))

    def set_warmed_up(self, state: bool):
        state = bool(state)
        if self.__dict__.get("_warmed_up_host") != state:
            self.warmed_up = torch.tensor(int(state), device=self.warmed_up.device)
            self.__dict__["_warmed_up_host"] = state

    def forward(self, x):
        x = self.net(x)
        if self.use_noise:
            waveform, loudness, noise = self.synth(x)
        else:
            waveform, loudness = self.synth(x)
            noise = torch.zeros_like(waveform)
        if self.loud_stride != 1:
            loudness = loudness.repeat_interleave(self.loud_stride)
        loudness = loudness.reshape(x.shape[0], 1, -1)
        waveform = torch.tanh(waveform) * core.mod_sigmoid(loudness)
        if self.__dict__.get("_warmed_up_host", None) is None:
            self.__dict__["_warmed_up_host"] = bool(self.warmed_up)
        if self.__dict__["_warmed_up_host"] and self.use_noise:
            waveform = waveform + noise
        return waveform


class Encoder(nn.Module):
    """rave/blocks.py:426-503 (v1 encoder: BatchNorm1d / SampleNorm, strided convs k = 2 r + 1, grouped output conv)."""

    def __init__(self, data_size, capacity, latent_size, ratios, n_out, sample_norm, repeat_layers, n_channels: int = 1,
                 recurrent_layer: Optional[Callable[[], nn.Module]] = None, spectrogram=None):
        super().__init__()
        data_size = data_size or n_channels
        net = [cc.Conv1d(data_size * n_channels, capacity, 7, padding=cc.get_padding(7))]
        for i, r in enumerate(ratios):
            in_dim = 2 ** i * capacity
            out_dim = 2 ** (i + 1) * capacity
            net.append(SampleNorm() if sample_norm else nn.BatchNorm1d(in_dim))
            net.append(nn.LeakyReLU(.2))
            net.append(cc.Conv1d(in_dim, out_dim, 2 * r + 1, padding=cc.get_padding(2 * r + 1, r), stride=r))
            for _ in range(repeat_layers - 1):
                net.append(SampleNorm() if sample_norm else nn.BatchNorm1d(out_dim))
                net.append(nn.LeakyReLU(.2))
                net.append(cc.Conv1d(out_dim, out_dim, 3, padding=cc.get_padding(3)))
        net.append(nn.LeakyReLU(.2))
        if recurrent_layer is not None:
            net.append(recurrent_layer(dim=out_dim, cumulative_delay=0))
            net.append(nn.LeakyReLU(.2))
        net.append(cc.Conv1d(out_dim, latent_size * n_out, 5, padding=cc.get_padding(5), groups=n_out))
        self.net = cc.CachedSequential(*net)
        self.cumulative_delay = self.net.cumulative_delay

    def forward(self, x):
        return self.net(x)


class NoiseGeneratorV2(nn.Module):
    """v2_small's filtered-noise branch (rave/blocks.py:243-292, configs/v2_small.gin:42-57): strided
    convs (library kernels) -> band amplitudes -> FIR via irfft -> uniform noise -> FFT convolution
    (torch/cuFFT: SURVEY 8f.4).  `forward(x, noise=None)`: a caller may inject the uniform noise
    (parity tests: CPU and CUDA Philox streams differ)."""

    def __init__(self, in_size: int, hidden_size: int, data_size: int, ratios, noise_bands: int,
                 n_channels: int = 1, activation: Callable[[int], nn.Module] = _default_activation):
        super().__init__()
        from .core import amp_to_impulse_response, fft_convolve, mod_sigmoid  # noqa: F401
        self.n_channels = n_channels
        channels = [in_size]
        channels.extend((len(ratios) - 1) * [hidden_size])
        channels.append(data_size * noise_bands * n_channels)
        net = []
        for i, r in enumerate(ratios):
            net.append(cc.Conv1d(channels[i], channels[i + 1], 2 * r, padding=(r, 0), stride=r))
            if i != len(ratios) - 1:
                net.append(activation(channels[i + 1]))
        self.net = nn.Sequential(*net)
        self.data_size = data_size
        self.noise_bands = noise_bands
        self._target = int(np.prod(ratios))            # host copy of `target_size` (no device sync per forward)
        self.register_buffer("target_size", torch.tensor(self._target).long())
        # every step of amp_to_impulse_response is linear in the amplitudes: its matrix, from the identity
        from .core import amp_to_impulse_response
        self.register_buffer("_ir_matrix", amp_to_impulse_response(torch.eye(noise_bands), self._target).t().contiguous(),
                             persistent=False)          # [target, bands]

    def forward(self, x, noise: Optional[torch.Tensor] = None):
        from .core import amp_to_impulse_response, fft_convolve, mod_sigmoid
        h = x
        mods = list(self.net)
        i = 0
        while i < len(mods):               # conv, then `activation -> conv` pairs fused
            m = mods[i]
            if isinstance(m, cc.Conv1d):
                h = m(h)
                i += 1
            else:
                h = mods[i + 1](h, act=m)
                i += 2
        C = self.n_channels * self.data_size
        if h.is_cuda and self._target <= 16 and self.noise_bands <= 64:
            # one library kernel for mod_sigmoid -> impulse response -> causal convolution with the noise block
            if noise is None:
                noise = torch.rand(h.shape[0], h.shape[2], C, self._target, device=h.device) * 2 - 1
            return ops.noise_fir(h, self._ir_matrix, noise, C)
        amp = mod_sigmoid(h - 5)
        amp = amp.permute(0, 2, 1)
        amp = amp.reshape(amp.shape[0], amp.shape[1], C, -1)
        ir = amp_to_impulse_response(amp, self._target)
        if noise is None:
            noise = torch.rand_like(ir) * 2 - 1
        out = fft_convolve(noise, ir).permute(0, 2, 1, 3)
        return out.reshape(out.shape[0], out.shape[1], -1)


class GRU(nn.Module):
    """rave/blocks.py:295-319 (configs/hybrid.gin: GeneratorV2.recurrent_layer, num_layers 2): nn.GRU over the time
    axis of [B, C, T], on rave_gru_fwd / rave_gru_bwd and GEMMs (ops.gru).  `gru_state` is the reference's (unused)
    buffer; `disable()` makes the module an identity."""

    def __init__(self, latent_size: int, num_layers: int) -> None:
        super().__init__()
        self.gru = nn.GRU(input_size=latent_size, hidden_size=latent_size, num_layers=num_layers, batch_first=True)
        self.register_buffer("gru_state", torch.tensor(0))
        self.enabled = True

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if not self.enabled:
            return x
        return ops.gru(x, self.gru)

    def disable(self):
        self.enabled = False

    def enable(self):
        self.enabled = True


def normalize_dilations(dilations, ratios):
    if isinstance(dilations[0], int):
        dilations = [dilations for _ in ratios]
    return dilations


# ---------------------------------------------------------------------------------------------
# EncoderV2 / GeneratorV2 (rave/blocks.py:514-714)
# ---------------------------------------------------------------------------------------------

class EncoderV2(nn.Module):

    def __init__(self, data_size: Union[int, None], capacity: int, ratios: Sequence[int],
                 latent_size: int, n_out: int, kernel_size: int, dilations: Sequence[int],
                 keep_dim: bool = False, recurrent_layer: Optional[Callable[[], nn.Module]] = None,
                 n_channels: int = 1,
                 activation: Callable[[int], nn.Module] = _default_activation,
                 adain: Optional[Callable[[int], nn.Module]] = None, spectrogram=None,
                 unit_activation: Optional[Callable[[int], nn.Module]] = None) -> None:
        super().__init__()
        dilations_list = normalize_dilations(dilations, ratios)
        data_size = data_size or n_channels
        # configs/snake.gin:10-11 rebinds DilatedUnit.activation together with the encoder's
        unit_activation = unit_activation or activation

        net = [
            normalization(cc.Conv1d(data_size * n_channels, capacity, kernel_size=kernel_size * 2 + 1,
                                    padding=cc.get_padding(kernel_size * 2 + 1))),
        ]
        num_channels = capacity
        for r, dils in zip(ratios, dilations_list):
            for d in dils:
                if adain is not None:
                    net.append(adain(dim=num_channels))
                net.append(Residual(DilatedUnit(dim=num_channels, kernel_size=kernel_size, dilation=d,
                                                activation=unit_activation)))
            net.append(activation(num_channels))
            out_channels = num_channels * r if keep_dim else num_channels * 2
            net.append(normalization(cc.Conv1d(num_channels, out_channels, kernel_size=2 * r, stride=r,
                                               padding=cc.get_padding(2 * r, r))))
            num_channels = out_channels

        net.append(activation(num_channels))
        net.append(normalization(cc.Conv1d(num_channels, latent_size * n_out, kernel_size=kernel_size,
                                           padding=cc.get_padding(kernel_size))))
        if recurrent_layer is not None:
            net.append(recurrent_layer(latent_size * n_out))
        self.net = cc.CachedSequential(*net)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.net(x)


class GeneratorV2(nn.Module):

    def __init__(self, capacity: int, ratios: Sequence[int], latent_size: int, kernel_size: int,
                 dilations: Sequence[int], keep_dim: bool = False, data_size: Union[int, None] = None,
                 recurrent_layer: Optional[Callable[[], nn.Module]] = None, n_channels: int = 1,
                 amplitude_modulation: bool = False, noise_module=None,
                 activation: Callable[[int], nn.Module] = _default_activation,
                 adain: Optional[Callable[[int], nn.Module]] = None,
                 unit_activation: Optional[Callable[[int], nn.Module]] = None) -> None:
        super().__init__()
        data_size = n_channels if data_size is None else data_size * n_channels
        dilations_list = normalize_dilations(dilations, ratios)[::-1]
        ratios = ratios[::-1]
        unit_activation = unit_activation or activation
        if keep_dim:
            num_channels = int(np.prod(ratios)) * capacity
        else:
            num_channels = 2 ** len(ratios) * capacity

        net = []
        if recurrent_layer is not None:
            net.append(recurrent_layer(latent_size))
        net.append(normalization(cc.Conv1d(latent_size, num_channels, kernel_size=kernel_size,
                                           padding=cc.get_padding(kernel_size))))
        for r, dils in zip(ratios, dilations_list):
            out_channels = num_channels // r if keep_dim else num_channels // 2
            net.append(activation(num_channels))
            net.append(normalization(cc.ConvTranspose1d(num_channels, out_channels, 2 * r, stride=r,
                                                        padding=r // 2)))
            num_channels = out_channels
            for d in dils:
                if adain is not None:
                    net.append(adain(num_channels))
                net.append(Residual(DilatedUnit(dim=num_channels, kernel_size=kernel_size, dilation=d,
                                                activation=unit_activation)))
        net.append(activation(num_channels))

        waveform_module = normalization(
            cc.Conv1d(num_channels, data_size * 2 if amplitude_modulation else data_size,
                      kernel_size=kernel_size * 2 + 1, padding=cc.get_padding(kernel_size * 2 + 1)))

        self.noise_module = None
        self.waveform_module = None
        if noise_module is not None:
            self.waveform_module = waveform_module
            self.noise_module = noise_module(out_channels, n_channels=n_channels)
        else:
            net.append(waveform_module)
        self.net = cc.CachedSequential(*net)
        self.amplitude_modulation = amplitude_modulation

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = self.net(x)
        noise = 0.
        if self.noise_module is not None:
            noise = self.noise_module(x)
            x = self.waveform_module(x)
        if self.amplitude_modulation and self.noise_module is None:
            return ops.am_tanh(x)                       # x*sigmoid(a) -> tanh, one kernel
        if self.amplitude_modulation:
            x, amplitude = x.split(x.shape[1] // 2, 1)
            x = x * torch.sigmoid(amplitude)
        x = x + noise
        return torch.tanh(x)

    def set_warmed_up(self, state: bool):
        pass


# ---------------------------------------------------------------------------------------------
# latent heads (rave/blocks.py:717-745, 794-850)
# ---------------------------------------------------------------------------------------------

class VariationalEncoder(nn.Module):

    def __init__(self, encoder, beta: float = 1.0, n_channels=1):
        super().__init__()
        self.encoder = encoder(n_channels=n_channels)
        self.beta = beta
        self.register_buffer("warmed_up", torch.tensor(0))
        self._warmed_up_host = None      # host mirror of the buffer: no device->host sync per step

    def reparametrize(self, z, eps: Optional[torch.Tensor] = None):
        """`eps` lets a caller inject the noise (parity tests; the CPU and CUDA Philox streams
        differ); default draws it like the reference (blocks.py:731)."""
        mean, scale = z.chunk(2, 1)
        if eps is None:
            eps = torch.randn_like(mean)
        if z.is_cuda and z.dim() == 3 and z.dtype == torch.float32:
            # one library pass instead of ~14 elementwise / reduction launches (sum over channels, mean over the rest)
            zs, kl_sum = ops.reparam(z, eps)
            return zs, self.beta * (kl_sum / (z.shape[0] * z.shape[2]))
        std = nn.functional.softplus(scale) + 1e-4
        var = std * std
        logvar = torch.log(var)
        z = eps * std + mean
        kl = (mean * mean + var - logvar - 1).sum(1).mean()
        return z, self.beta * kl

    def set_warmed_up(self, state: bool):
        state = bool(state)
        if self._warmed_up_host is None or self._warmed_up_host != state:
            self.warmed_up = torch.tensor(int(state), device=self.warmed_up.device)
            self._warmed_up_host = state

    def _is_warmed_up(self) -> bool:
        if self._warmed_up_host is None:          # e.g. right after load_state_dict: read the buffer once
            self._warmed_up_host = bool(self.warmed_up)
        return self._warmed_up_host

    def forward(self, x: torch.Tensor):
        z = self.encoder(x)
        if self._is_warmed_up():
            z = z.detach()
        return z


class WasserteinEncoder(nn.Module):
    """rave/blocks.py:748-791 (configs/wasserstein.gin; the reference's spelling): a Wasserstein auto-encoder whose
    regulariser is the MMD between the latent rows z[b, :, t] and a standard normal sample of the same shape, and whose
    latent may be extended by `noise_augmentation` channels of standard normal noise."""

    def __init__(self, encoder_cls, noise_augmentation: int = 0, n_channels: int = 1):
        super().__init__()
        self.encoder = encoder_cls(n_channels=n_channels)
        self.register_buffer("warmed_up", torch.tensor(0))
        self.noise_augmentation = noise_augmentation
        self._warmed_up_host = None      # host mirror of the buffer, as in VariationalEncoder

    def compute_mean_kernel(self, x, y):
        kernel_input = (x[:, None] - y[None]).pow(2).mean(2) / x.shape[-1]
        return torch.exp(-kernel_input).mean()

    def compute_mmd(self, x, y):
        x_kernel = self.compute_mean_kernel(x, x)
        y_kernel = self.compute_mean_kernel(y, y)
        xy_kernel = self.compute_mean_kernel(x, y)
        return x_kernel + y_kernel - 2 * xy_kernel

    def reparametrize(self, z, eps: Optional[tuple] = None):
        """`eps` = (prior [B·L, D], noise [B, noise_augmentation, L] or None) lets a caller inject both draws (parity
        tests: the CPU and CUDA Philox streams differ); by default they are drawn in the reference's order, the prior
        sample first.  CUDA fp32 input runs the MMD kernels (rave_mmd_fwd / _bwd), other input the reference's
        expression."""
        B, D, L = z.shape
        prior, noise = eps if eps is not None else (None, None)
        if prior is None:
            prior = torch.randn(B * L, D, device=z.device, dtype=z.dtype)
        if z.is_cuda and z.dtype == torch.float32:
            reg = ops.mmd(z, prior)[0]
        else:
            reg = self.compute_mmd(z.permute(0, 2, 1).reshape(-1, D), prior).mean()
        if self.noise_augmentation:
            if noise is None:
                noise = torch.randn(B, self.noise_augmentation, L, device=z.device, dtype=z.dtype)
            z = torch.cat([z, noise], 1)
        return z, reg

    def set_warmed_up(self, state: bool):
        state = bool(state)
        if self._warmed_up_host is None or self._warmed_up_host != state:
            self.warmed_up = torch.tensor(int(state), device=self.warmed_up.device)
            self._warmed_up_host = state

    def _is_warmed_up(self) -> bool:
        if self._warmed_up_host is None:          # e.g. right after load_state_dict: read the buffer once
            self._warmed_up_host = bool(self.warmed_up)
        return self._warmed_up_host

    def forward(self, x: torch.Tensor):
        z = self.encoder(x)
        if self._is_warmed_up():
            z = z.detach()
        return z


class SphericalEncoder(nn.Module):
    """rave/blocks.py:833-849 (configs/spherical.gin).  Its `set_warmed_up` does nothing: the encoder keeps training in
    phase 2."""

    def __init__(self, encoder_cls, n_channels: int = 1) -> None:
        super().__init__()
        self.encoder = encoder_cls(n_channels=n_channels)

    def reparametrize(self, z):
        if z.is_cuda and z.dtype == torch.float32:
            return ops.sphere_norm(z), z.new_zeros(())
        norm_z = z / torch.norm(z, p=2, dim=1, keepdim=True)
        return norm_z, torch.zeros_like(z).mean()

    def set_warmed_up(self, state: bool):
        pass

    def forward(self, x):
        return self.encoder(x)


class DiscreteEncoder(nn.Module):
    """rave/blocks.py:794-830 (quirk D3: `enabled` is never switched on by the reference's own
    training code, so RVQ is bypassed unless the caller sets it)."""

    def __init__(self, encoder_cls, vq_cls, num_quantizers, noise_augmentation: int = 0,
                 n_channels: int = 1):
        super().__init__()
        self.encoder = encoder_cls(n_channels=n_channels)
        self.rvq = vq_cls()
        self.num_quantizers = num_quantizers
        self.register_buffer("warmed_up", torch.tensor(0))
        self.register_buffer("enabled", torch.tensor(0))
        self.noise_augmentation = noise_augmentation

    def _enabled_host(self) -> bool:
        """Host copy of the `enabled` buffer (re-read only when the buffer was written: no device sync per step, and a
        captured CUDA graph never touches it)."""
        t = self.enabled
        hit = self.__dict__.get("_enabled_cache")
        if hit is None or hit[0] is not t or hit[1] != t._version:
            hit = self.__dict__["_enabled_cache"] = (t, t._version, bool(t.item()))
        return hit[2]

    def reparametrize(self, z):
        if self._enabled_host():
            z, diff, _ = self.rvq(z)
        else:
            diff = torch.zeros_like(z).mean()
        if self.noise_augmentation:
            noise = torch.randn(z.shape[0], self.noise_augmentation, z.shape[-1], device=z.device, dtype=z.dtype)
            z = torch.cat([z, noise], 1)
        return z, diff

    def set_warmed_up(self, state: bool):
        # host mirror as in VariationalEncoder: the buffer is rewritten only when the flag changes (a tensor built from a
        # Python int is a pageable host->device copy, which a CUDA-graph capture rejects)
        state = bool(state)
        if self.__dict__.get("_warmed_up_host") != state:
            self.warmed_up = torch.tensor(int(state), device=self.warmed_up.device)
            self.__dict__["_warmed_up_host"] = state

    def forward(self, x):
        return self.encoder(x)

"""v1/v2 discriminators -- module surface of rave/discriminator.py:77-209 on librave_b200.so.

`ConvNet` accepts the same `conv` argument the reference's gin files bind (`@torch.nn.Conv1d`,
`@nn.Conv2d` with kernel (5,1): configs/v1.gin:84-86, configs/v2.gin:53-55) and maps it to a
subclass with identical parameters / state_dict keys whose forward launches our kernels.  A
(k,1) Conv2d over the folded signal [B,C,L/p,p] is a Conv1d along L/p with the period axis as
extra batch (SURVEY.md K12): the fold is kept as a *view* of a [B,p,C,L/p] tensor, so the only
copy is the 1-channel input.
"""
from typing import Callable, Optional, Sequence, Type

import numpy as np

import torch
import torch.nn as nn

from . import cc, ops
from .blocks import normalization
from ._lib import RaveB200Error

# streams the feature-matching discriminator chains are issued on (CombineDiscriminators.forward_fm); RAVE.compute_losses
# also moves the spectral losses to a side stream when it is above 1.  1 = everything on the current stream
DISC_STREAMS = 8


class DiscConv1d(nn.Conv1d):
    """nn.Conv1d (symmetric int padding, bias) on the library kernels; optional fused pre-activation."""

    def forward(self, x, act=None):
        code = cc._act_code(act)
        p = self.padding[0]
        return ops.conv1d(x, self.weight, self.bias, None, self.stride[0], self.dilation[0], (p, p),
                          code[0], code[1], None)


class DiscConv2dK1(nn.Conv2d):
    """nn.Conv2d with kernel (k,1), stride (s,1), padding (p,0): conv1d along H, W folded into batch.
    Input/outputs are [B,C,H,W] tensors (the output is a permuted view of a [B,W,C,H'] buffer)."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        if self.kernel_size[1] != 1 or self.stride[1] != 1 or self.padding[1] != 0 or self.groups != 1:
            raise RaveB200Error("only (k,1) 2-D convolutions are on the hot path")

    def forward(self, x, act=None):
        code = cc._act_code(act)
        B, C, H, W = x.shape
        xw = x.permute(0, 3, 1, 2).reshape(B * W, C, H)   # free when x came from a previous layer
        p = self.padding[0]
        y = ops.conv1d(xw, self.weight.squeeze(-1), self.bias, None, self.stride[0], self.dilation[0],
                       (p, p), code[0], code[1], None)
        return y.view(B, W, y.shape[1], y.shape[2]).permute(0, 2, 3, 1)


class TimeStackedConv2d(nn.Conv2d):
    """nn.Conv2d with unit time stride and 'same' time padding whose kt time taps (time t + j dt - pt for tap j) become
    kt x Cin input channels of ONE conv along frequency over rows (b, t): in bf16 mode a one-layer chain of the wgmma
    engine (forward, dgrad and wgrad on the tensor cores), channel-last on both sides.  Subclasses say which axis of
    kernel_size / padding / stride / dilation is time, check their arguments and keep their fp32 `forward`."""

    TIME_AXIS: int            # set by the subclass: 0 or 1, frequency is the other one

    def cout_ok(self) -> bool:
        return self.out_channels % 16 == 0

    def _tc_chain_spec(self, C):
        """One-layer engine chain of this conv along frequency, planned on an engine.ParamProxy: the (j, c) channel
        order is a permuted VIEW of the parameter, so the weight-norm backward of the chain reaches weight_v / weight_g
        through autograd."""
        from . import engine
        t, f = self.TIME_AXIS, 1 - self.TIME_AXIS
        kt, pf = self.kernel_size[t], self.padding[f]
        cin = kt * C
        proxy = self.__dict__.get("_tc_proxy")
        if proxy is None:
            spec = engine.LayerSpec("conv", None, cin, self.out_channels, self.kernel_size[f], self.stride[f], 1, (pf, pf),
                                    ops.ACT_NONE, 0.0, None, True, True)
            spec.cin_pad = (-cin) % 16
            spec.cout_pad = (-self.out_channels) % 16
            proxy = engine.ParamProxy(self, spec, self._tc_refresh_proxy)
        if proxy.spec.Cin != cin:
            raise RaveB200Error(f"{type(self).__name__}: planned for {proxy.spec.Cin // kt} input channels, called "
                                f"with {C}")
        self._tc_refresh_proxy()
        return proxy.spec

    def _tc_refresh_proxy(self):
        """(Re)build the proxy's (j, c)-ordered views of the parameters (a permuted reshape is a copy: it goes stale
        when the parameters move, so engine.refresh_static_prep calls this before it rewrites the static layouts)."""
        proxy = self.__dict__["_tc_proxy"]
        t, f = self.TIME_AXIS, 1 - self.TIME_AXIS
        shape = (self.out_channels, proxy.spec.Cin, self.kernel_size[f])
        order = (0, 2 + t, 1, 2 + f)                      # [Cout][Cin][.][.] -> [Cout][kt][Cin][kf]
        if hasattr(self, "weight_v"):
            proxy.weight_v = self.weight_v.permute(order).reshape(shape)
            proxy.weight_g = self.weight_g.reshape(self.out_channels, 1, 1)
        else:
            proxy.weight = self.weight.permute(order).reshape(shape)
        proxy.bias = self.bias

    def stacked_geometry(self, Fq: int, C: int):
        """(Fp, Cp) of this conv's time-stacked operand for an input of Fq positions and C channels."""
        spec = self._tc_chain_spec(C)
        return Fq + (-Fq) % spec.stride, self.kernel_size[self.TIME_AXIS] * C + spec.cin_pad

    def forward_cl(self, x_cl, xs=None):
        """Channel-last in, channel-last out: x_cl [B, T, F, C] fp32 (a view with dense (f, c) rows) -> the chain's own
        output buffer [(b t), Fo, Cout(+pad to 16)] fp32, which IS [B, T, Fo, Cout] channel-last: no layout pass on
        either side of the conv.  `xs`: the time-stacked bf16 operand when the producer already wrote it
        (ops.leaky_fm_stack: the previous layer's feature tap)."""
        from . import engine
        B, T, Fq, C = x_cl.shape
        spec = self._tc_chain_spec(C)
        t = self.TIME_AXIS
        Fp, Cp = self.stacked_geometry(Fq, C)
        if xs is None:
            xs = ops.time_stack_nhwc(x_cl, self.kernel_size[t], self.padding[t], Cp, Fp, *_dil_arg(self.dilation[t]))
        elif tuple(xs.shape) != (B * T, Fp, Cp) or xs.dtype != engine.ACT_DTYPE:
            raise RaveB200Error(f"{type(self).__name__}.forward_cl: the pre-stacked operand does not match this conv's "
                                f"geometry")
        (out,) = engine.run_chain(xs, [spec], Fq)
        if out.shape[1] != engine.chain_lengths([spec], Fq)[0]:
            raise RaveB200Error(f"{type(self).__name__}: the one-layer chain's output pitch is its length")
        return out


def _dil_arg(dt: int):
    """Trailing time-dilation argument of ops.time_stack_nhwc / ops.leaky_fm_stack: left out when it is 1, their default
    (the CPU emulation of these two calls, tests/tc_emulator.py, takes no dilation)."""
    return () if dt == 1 else (dt,)


def _feature_tap(out, slope, B):
    """Post-activation feature of a chain output (rows = [real; fake] when the batch B is even): LeakyReLU and the two L1
    feature-matching sums in one pass (ops.leaky_fm), or the plain activation for an unpaired batch."""
    if B % 2 == 0 and out.dtype == torch.float32 and out.is_contiguous():
        return ops.leaky_fm(out, slope)
    return ops.activation(out, ops.ACT_LEAKY, slope), None


def _feature_tap_stack(out, slope, B, T, nxt, fuse: bool = True):
    """_feature_tap that, with `fuse`, also writes the time-stacked operand of the next conv `nxt` (a TimeStackedConv2d)
    in the same pass when the geometry allows it (kt = 3, pt = its time dilation, no channel padding on either side):
    returns (a, stats, xs | None)."""
    C = out.shape[2]
    if (fuse and nxt is not None and B % 2 == 0 and out.dtype == torch.float32 and out.is_contiguous()
            and nxt.in_channels == C and C % 4 == 0 and out.shape[0] == B * T):
        kt, pt, dt = (v[nxt.TIME_AXIS] for v in (nxt.kernel_size, nxt.padding, nxt.dilation))
        if kt == 3 and pt == dt:
            Fp, Cp = nxt.stacked_geometry(out.shape[1], C)
            if Cp == 3 * C:
                return ops.leaky_fm_stack(out, slope, T, Fp, *_dil_arg(dt))
    a, st = _feature_tap(out, slope, B)
    return a, st, None


def _map_conv(conv):
    if conv is nn.Conv1d or conv is DiscConv1d:
        return DiscConv1d
    if conv is nn.Conv2d or conv is DiscConv2dK1:
        return DiscConv2dK1
    raise RaveB200Error(f"unsupported conv class for the discriminator hot path: {conv}")


class ConvNet(nn.Module):
    """rave/discriminator.py:77-119.  Features = PRE-activation output of every conv."""

    def __init__(self, in_size, out_size, capacity, n_layers, kernel_size, stride, conv) -> None:
        super().__init__()
        conv = _map_conv(conv)
        channels = [in_size]
        channels += list(capacity * 2 ** np.arange(n_layers))
        if isinstance(stride, int):
            stride = n_layers * [stride]
        net = []
        for i in range(n_layers):
            if not isinstance(kernel_size, int):
                pad = (cc.get_padding(kernel_size[0], stride[i], mode="centered")[0], 0)
                s = (stride[i], 1)
            else:
                pad = cc.get_padding(kernel_size, stride[i], mode="centered")[0]
                s = stride[i]
            net.append(normalization(conv(int(channels[i]), int(channels[i + 1]), kernel_size, stride=s,
                                          padding=pad)))
            net.append(nn.LeakyReLU(.2))
        net.append(conv(int(channels[-1]), out_size, 1))
        self.net = nn.Sequential(*net)

    def _tc_specs(self):
        from . import engine
        if "_tc_specs_cache" not in self.__dict__:
            specs = engine.plan_convnet(self.net)
            if specs is not None and not engine.chain_supported(specs):
                specs = None
            self.__dict__["_tc_specs_cache"] = specs
        return self.__dict__["_tc_specs_cache"]

    def _chain_input(self, x, specs):
        """Operand of the chain and the `src` argument of engine.run_chain.  A first layer that reads the signal in
        place (engine.raw_input_ok: every shipped config, mono or stereo) gets the raw fp32 rows, [B(*W), pitch] for
        mono and [B(*W), C, pitch] otherwise; any other first layer the zero-padded channel-last bf16 stream."""
        from . import engine
        first = specs[0]
        if x.dim() == 3:
            B, C, L = x.shape
            W = 1
        else:
            B, C, L, W = x.shape
        rpad = (-L) % first.stride              # row pitch: a multiple of the first layer's stride
        if engine.raw_input_ok(first, C):
            rows = x.unsqueeze(-1) if x.dim() == 3 else x          # [B, C, L, W]
            rows = rows.permute(0, 3, 1, 2).reshape(B * W, C, L)
            if C == 1:
                return nn.functional.pad(rows.reshape(B * W, L), (0, rpad)).contiguous(), None, B, W, L
            return nn.functional.pad(rows, (0, rpad)).contiguous(), (1, 1), B, W, L
        rows = x.transpose(1, 2) if x.dim() == 3 else x.permute(0, 3, 2, 1).reshape(B * W, L, C)
        xa = nn.functional.pad(rows, (0, first.cin_pad, 0, rpad)).to(engine.ACT_DTYPE).contiguous()
        return xa, None, B, W, L

    def forward_fm(self, x, period: int = 1, pool: int = 1, fake_grad_only: bool = False):
        """Fused feature-matching path (bf16 engine): x = cat([real, fake]) RAW signal [B, C, T] -> (stats [n-1, 2],
        counts, score, score_stats [3, 2], n_score) with stats[i] = (sum|h_r - h_f|, sum|h_r|) of hidden feature i,
        counts[i] = its number of elements per half, score = the last conv's output in the reference's shape,
        score_stats = the six sums of the score tail (engine.TcChainFn), n_score = score elements per half.
        `period` > 1: this ConvNet sees MultiPeriodDiscriminator.fold(x, period); `pool` > 1: it sees x average-
        pooled by `pool` (MultiScaleDiscriminator) -- in both cases the first layer reads x in place."""
        from . import engine
        specs = self._tc_specs()
        first = specs[0]
        if x.dim() != 3 or not engine.raw_input_ok(first, x.shape[1]):
            raise RuntimeError("forward_fm expects a signal [B, C, T] and a first layer that reads its C channels in "
                               "place (engine.raw_input_ok)")
        B, C, T = x.shape
        W = period
        L = (T + period - 1) // period if period > 1 else T // pool
        xr = x.reshape(B, T) if C == 1 else x.contiguous()
        stats, score_stats, last = engine.run_chain(xr, specs, L, fm=True, src=(period, pool),
                                                    fake_grad_only=fake_grad_only)
        lens = engine.chain_lengths(specs, L)
        counts = [(B // 2) * W * Lo * s.Cout for s, Lo in zip(specs[:-1], lens[:-1])]
        o = last[:, :lens[-1], :specs[-1].Cout]
        if period == 1:
            score = o.permute(0, 2, 1)
        else:
            score = o.reshape(B, W, lens[-1], specs[-1].Cout).permute(0, 3, 2, 1)
        # score_stats [3, 2] (engine.TcChainFn) is meaningful when the score has one channel; n_score = its
        # number of elements per half
        n_score = (B // 2) * W * lens[-1] if specs[-1].Cout == 1 else 0
        return stats, counts, score, score_stats, n_score

    def _forward_tc(self, x, specs):
        """bf16 tensor-core path: the whole ConvNet as one chain in channel-last layout; features come
        back as permuted views with the reference's shapes."""
        from . import engine
        xa, src, B, W, L = self._chain_input(x, specs)
        outs = engine.run_chain(xa, specs, L, src=src)
        lens = engine.chain_lengths(specs, L)
        features = []
        for s, o, Lo in zip(specs, outs, lens):
            o = o[:, :Lo, :s.Cout]
            if x.dim() == 3:
                features.append(o.permute(0, 2, 1))
            else:
                features.append(o.reshape(B, W, Lo, s.Cout).permute(0, 3, 2, 1))
        return features

    def forward(self, x):
        from . import engine
        if engine.precision() == "bf16" and x.is_cuda:
            specs = self._tc_specs()
            if specs is not None:
                return self._forward_tc(x, specs)
        features = []
        pending_act = None
        for layer in self.net:
            if isinstance(layer, nn.LeakyReLU):
                pending_act = layer            # fused into the next conv's operand load
                continue
            x = layer(x, act=pending_act)
            pending_act = None
            features.append(x)
        return features


class MultiScaleDiscriminator(nn.Module):
    """rave/discriminator.py:122-136."""

    def __init__(self, n_discriminators, convnet, n_channels=1) -> None:
        super().__init__()
        self.layers = nn.ModuleList([convnet(in_size=n_channels) for _ in range(n_discriminators)])

    def fm_jobs(self):
        # scale i sees avg_pool1d(., 2) applied i times = the mean over 2^i consecutive samples (floor lengths agree)
        return [(layer, {"pool": 2 ** i}) for i, layer in enumerate(self.layers)]

    def forward_fm(self, x, fake_grad_only: bool = False):
        return [layer.forward_fm(x, fake_grad_only=fake_grad_only, **kw) for layer, kw in self.fm_jobs()]

    def forward(self, x):
        features = []
        for layer in self.layers:
            features.append(layer(x))
            x = nn.functional.avg_pool1d(x, 2)
        return features


class MultiPeriodDiscriminator(nn.Module):
    """rave/discriminator.py:174-195."""

    def __init__(self, periods, convnet, n_channels=1) -> None:
        super().__init__()
        self.periods = periods
        self.layers = nn.ModuleList([convnet(in_size=n_channels) for _ in periods])

    def forward(self, x):
        features = []
        for layer, n in zip(self.layers, self.periods):
            features.append(layer(self.fold(x, n)))
        return features

    def fm_jobs(self):
        return [(layer, {"period": n}) for layer, n in zip(self.layers, self.periods)]

    def forward_fm(self, x, fake_grad_only: bool = False):
        return [layer.forward_fm(x, fake_grad_only=fake_grad_only, **kw) for layer, kw in self.fm_jobs()]

    def fold(self, x, n):
        pad = (n - (x.shape[-1] % n)) % n
        x = nn.functional.pad(x, (0, pad))
        return x.reshape(*x.shape[:2], -1, n)


class CombineDiscriminators(nn.Module):
    """rave/discriminator.py:198-209."""

    def __init__(self, discriminators: Sequence[Type[nn.Module]], n_channels=1) -> None:
        super().__init__()
        self.discriminators = nn.ModuleList(disc_cls(n_channels=n_channels) for disc_cls in discriminators)

    def forward(self, x):
        features = []
        for disc in self.discriminators:
            features.extend(disc(x))
        return features

    def supports_fused_fm(self, x) -> bool:
        """True when every sub-discriminator can run the fused feature-matching path on `x`."""
        from . import engine
        if engine.precision() != "bf16" or not x.is_cuda or x.dim() != 3:
            return False
        for disc in self.discriminators:
            if not hasattr(disc, "forward_fm"):
                return False
            for layer in disc.layers:
                if not isinstance(layer, ConvNet) or layer._tc_specs() is None:
                    return False
                specs = layer._tc_specs()
                if not engine.raw_input_ok(specs[0], x.shape[1]):
                    return False
                # the statistics are read from the bf16 operand a = LeakyReLU(h) of the NEXT layer: every hidden feature
                # needs a LeakyReLU consumer and un-padded channels (tiny test capacities have Cout % 16 != 0)
                for s, nxt in zip(specs[:-1], specs[1:]):
                    if s.cout_pad or nxt.pre_act != ops.ACT_LEAKY:
                        return False
        return True

    def forward_fm(self, x, fake_grad_only: bool = False):
        """fake_grad_only: the caller will only use the gradient with respect to the FAKE half of x (generator step,
        frozen discriminator): the backward then runs on that half alone (engine.TcChainFn.backward)."""
        jobs = []
        for disc in self.discriminators:
            jobs.extend(disc.fm_jobs())
        ns = DISC_STREAMS
        if ns <= 1 or not x.is_cuda:
            return [layer.forward_fm(x, fake_grad_only=fake_grad_only, **kw) for layer, kw in jobs]
        # The nets are independent chains of persistent kernels: issued on a few streams, the tail of one kernel (CTAs
        # finishing at different times) and the prologue of the next overlap with another net's work instead of leaving
        # SMs idle; autograd replays every chain's backward on the stream its forward ran on.
        cur = torch.cuda.current_stream()
        if getattr(self, "_fm_streams", None) is None or len(self._fm_streams) != ns:
            self._fm_streams = [torch.cuda.Stream() for _ in range(ns)]
        out = [None] * len(jobs)
        for j, (layer, kw) in enumerate(jobs):
            st = self._fm_streams[j % ns]
            st.wait_stream(cur)
            x.record_stream(st)
            with torch.cuda.stream(st):
                out[j] = layer.forward_fm(x, fake_grad_only=fake_grad_only, **kw)
        for st in self._fm_streams:
            cur.wait_stream(st)
        for res in out:
            for t in res:
                if torch.is_tensor(t):
                    t.record_stream(cur)
        return out


# ---------------------------------------------------------------------------------------------------------------------
# Multi-scale spectral discriminator (rave/discriminator.py:12-74, 139-153; configs/spectral_discriminator.gin): one
# EncodecConvNet of weight-normed 2-D convs over the complex STFT [B, (re | im) x C, F, T] of each scale.  A (kf, kt)
# conv with unit time stride is ONE library conv1d along frequency over rows (b, t) whose channels are the kt time-
# shifted copies (by multiples of the time dilation) of the input channels (`SpectralConv2d`).  In bf16 mode each scale
# runs channel-last from end to end on the wgmma engine, like the Descript MRD.
# ---------------------------------------------------------------------------------------------------------------------

class _Spectrogram(nn.Module):
    """torchaudio.transforms.Spectrogram(n_fft, hop_length=n_fft // 4, power=None, normalized=True, center=False) of the
    reference: its only state_dict entry is the hann `window`.  On CUDA tensors the framing is a library kernel
    (no padding, scaled by 1 / ||window||_2) and cuFFT transforms; returns the complex [B, C, F, T]."""

    def __init__(self, n_fft: int):
        super().__init__()
        self.n_fft, self.hop = n_fft, n_fft // 4
        window = torch.hann_window(n_fft)
        self.register_buffer("window", window)
        self.scale = float(1.0 / window.pow(2.).sum().sqrt())
        bw = torch.full((n_fft // 2 + 1,), 0.5 * n_fft)
        bw[0] = n_fft
        bw[-1] = n_fft
        self.register_buffer("rfft_bw", bw, persistent=False)

    def frames_spectrum(self, x):
        """x [N, T] CUDA -> complex [N, frames, bins]: the channel-last (time, frequency) layout of the engine path."""
        return ops.rfft(ops.stft_frames_valid(x, self.window, self.n_fft, self.hop, self.scale), self.rfft_bw)

    def forward(self, x):
        B, C, T = x.shape
        if x.is_cuda:
            z = self.frames_spectrum(x.reshape(B * C, T)).transpose(-1, -2)
        else:
            z = torch.stft(x.reshape(B * C, T), self.n_fft, hop_length=self.hop, win_length=self.n_fft,
                           window=self.window, center=False, normalized=False, onesided=True,
                           return_complex=True) * self.scale
        return z.reshape(B, C, z.shape[-2], z.shape[-1])


def spectrogram(n_fft: int):
    """rave/discriminator.py:12-20."""
    return _Spectrogram(n_fft)


class SpectralConv2d(TimeStackedConv2d):
    """nn.Conv2d with kernel (kf, kt), stride (sf, 1), dilation (1, dt), padding (pf, dt (kt - 1) / 2) on [B, C, F, T]
    tensors, on the library's conv1d kernels (TimeStackedConv2d, time on the last axis).  Same parameters / state_dict
    keys as nn.Conv2d."""

    TIME_AXIS = 1

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        kt, dt = self.kernel_size[1], self.dilation[1]
        if self.stride[1] != 1 or self.dilation[0] != 1 or self.groups != 1 or self.padding_mode != "zeros" \
                or 2 * self.padding[1] != dt * (kt - 1):
            raise RaveB200Error("SpectralConv2d: unit time stride, 'same' time padding, no groups / frequency dilation")

    def forward(self, x):
        B, C, Fq, T = x.shape
        kf, kt = self.kernel_size
        pf, pt = self.padding
        dt = self.dilation[1]
        if self.tc_ready(x):
            out = self.forward_cl(x.permute(0, 3, 2, 1))
            return out[..., :self.out_channels].reshape(B, T, out.shape[1], self.out_channels).permute(0, 3, 2, 1)
        xp = nn.functional.pad(x, (pt, pt))
        xi = torch.stack([xp[..., j * dt:j * dt + T] for j in range(kt)], 1)          # [B, kt, C, F, T]
        xi = xi.permute(0, 4, 1, 2, 3).reshape(B * T, kt * C, Fq)                      # rows (b, t), channels (j, c)
        w = self.weight.permute(0, 3, 1, 2).reshape(self.out_channels, kt * C, kf)
        y = ops.conv1d(xi, w, self.bias, None, self.stride[0], 1, (pf, pf), ops.ACT_NONE, 0.0, None)
        return y.view(B, T, self.out_channels, y.shape[-1]).permute(0, 2, 3, 1)

    def tc_ready(self, x) -> bool:
        from . import engine
        return engine.precision() == "bf16" and x.is_cuda and engine.ACT_DTYPE == torch.bfloat16


def rectified_2d_conv_block(capacity, kernel_sizes, strides=None, dilations=None, in_size=None, out_size=None,
                            activation: bool = True):
    """rave/discriminator.py:23-51 (weight norm through blocks.normalization, configs/v1.gin:41)."""
    if dilations is None:
        paddings = kernel_sizes[0] // 2, kernel_sizes[1] // 2
    else:
        fks = (kernel_sizes[0] - 1) * dilations[0], (kernel_sizes[1] - 1) * dilations[1]
        paddings = fks[0] // 2, fks[1] // 2
    conv = normalization(SpectralConv2d(in_size or capacity, out_size or capacity, kernel_size=kernel_sizes,
                                        stride=strides or (1, 1), dilation=dilations or (1, 1), padding=paddings))
    if not activation:
        return conv
    return nn.Sequential(conv, nn.LeakyReLU(.2))


class EncodecConvNet(nn.Module):
    """rave/discriminator.py:54-74.  Features are the POST-activation output of every block, the last one (no
    activation) is the score."""

    def __init__(self, capacity: int, n_channels: int = 1) -> None:
        super().__init__()
        self.net = nn.Sequential(
            rectified_2d_conv_block(capacity, (9, 3), in_size=2 * n_channels),
            rectified_2d_conv_block(capacity, (9, 3), (2, 1), (1, 1)),
            rectified_2d_conv_block(capacity, (9, 3), (2, 1), (1, 2)),
            rectified_2d_conv_block(capacity, (9, 3), (2, 1), (1, 4)),
            rectified_2d_conv_block(capacity, (3, 3)),
            rectified_2d_conv_block(capacity, (3, 3), out_size=1, activation=False),
        )

    def convs(self):
        return [layer[0] if isinstance(layer, nn.Sequential) else layer for layer in self.net]

    def forward(self, x):
        features = []
        for layer in self.net:
            if isinstance(layer, nn.Sequential):
                h = layer[0](x)
                x = ops.activation(h.contiguous(), ops.ACT_LEAKY, layer[1].negative_slope)
            else:
                x = layer(x)
            features.append(x)
        return features

    def forward_cl(self, x0):
        """bf16 engine mode: x0 = view_as_real(spectrum) [B, T, F, 2] is already the channel-last input of the first
        conv; every conv's output buffer passes through the feature tap, which also writes the next conv's operand.
        Features are NCHW views [B, C, F, T] of the tapped buffers, carrying `_cl_base` / `_fm_stats`."""
        B, T = x0.shape[0], x0.shape[1]
        convs = self.convs()
        fmap = []
        cur, xs = x0, None
        for i, (layer, conv) in enumerate(zip(self.net, convs)):
            out = conv.forward_cl(cur, xs)                                 # [(b t), Fo, Cout(+pad)]
            Fo = out.shape[1]
            if isinstance(layer, nn.Sequential):
                nxt = convs[i + 1] if i + 1 < len(convs) else None
                a, st, xs = _feature_tap_stack(out, layer[1].negative_slope, B, T, nxt)
                cur = a.view(B, T, Fo, out.shape[2])
                feat = cur.permute(0, 3, 2, 1)
                feat._cl_base = a
                feat._fm_stats = st
            else:
                feat = out.view(B, T, Fo, out.shape[2])[..., :conv.out_channels].permute(0, 3, 2, 1)
            fmap.append(feat)
        return fmap


class MultiScaleSpectralDiscriminator(nn.Module):
    """rave/discriminator.py:139-153."""

    def __init__(self, scales: Sequence[int], convnet: Callable[..., nn.Module], n_channels: int = 1) -> None:
        super().__init__()
        self.specs = nn.ModuleList([spectrogram(n) for n in scales])
        self.nets = nn.ModuleList([convnet(n_channels=n_channels) for _ in scales])

    def engine_ready(self, x) -> bool:
        """bf16 engine path: mono CUDA input, 16-aligned widths, at least one frame at every scale."""
        first = [net.convs()[0] for net in self.nets]
        return (x.dim() == 3 and x.shape[1] == 1 and all(c.tc_ready(x) and c.cout_ok() for c in first)
                and x.shape[-1] >= max(s.n_fft for s in self.specs))

    def forward(self, x):
        features = []
        if self.engine_ready(x):
            for spec, net in zip(self.specs, self.nets):
                features.append(net.forward_cl(torch.view_as_real(spec.frames_spectrum(x[:, 0]))))
            return features
        for spec, net in zip(self.specs, self.nets):
            spec_x = spec(x)
            features.append(net(torch.cat([spec_x.real, spec_x.imag], 1)))
        return features

"""v3 discriminator -- module surface of rave/descript_discriminator.py (MPD + MRD; MSD is defined by
the reference but never instantiated: `rates=[]`, and its constructor call would raise, quirk D4).

MPD (77 % of the v3 discriminator FLOPs, SURVEY 8a15) runs on the library's conv kernels: a (5,1)
Conv2d over the period-folded signal is a Conv1d along the folded axis with the period as extra batch.
MRD (banded complex STFT -> (3,9) Conv2d stacks, SURVEY row 8f.3) runs on the library too: the STFT is the framing
kernel of csrc/spectral.cu (+ cuFFT for the transform, as for the spectral losses), and a (kt, kf) Conv2d with unit
time stride is ONE library conv1d along frequency over rows [(b, t)] whose channels are the kt time-shifted copies of
the input channels (`DiscConv2d`): out[b,:,t,:] = sum_dt conv1d_f(x[b,:,t+dt-pt,:], W[:,:,dt,:]).
Features are POST-activation (descript_discriminator.py:59-61).  No cuDNN on this path.
"""
import os

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib, ops
from .blocks import weight_norm
from .discriminator import DiscConv2dK1


def WNConv2dK1(*args, **kwargs):
    """WNConv2d of the reference for (k,1) kernels, on the library kernels."""
    act = kwargs.pop("act", True)
    conv = weight_norm(DiscConv2dK1(*args, **kwargs))
    if not act:
        return conv
    return nn.Sequential(conv, nn.LeakyReLU(0.1))


class DiscConv2d(nn.Conv2d):
    """nn.Conv2d with kernel (kt, kf), stride (1, sf), padding (pt, pf) on the library's conv1d kernel: the kt time taps
    become kt x Cin input channels of a conv along frequency (rows = (batch, time) pairs).  Same parameters / state_dict
    keys as nn.Conv2d; input and output are [B, C, T, F] tensors."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        if self.stride[0] != 1 or self.groups != 1 or self.dilation != (1, 1) or self.padding_mode != "zeros" \
                or 2 * self.padding[0] != self.kernel_size[0] - 1:
            raise _lib.RaveB200Error("DiscConv2d: unit time stride, 'same' time padding, no groups / dilation")

    def forward(self, x):
        from . import engine
        B, C, T, Fq = x.shape
        kt, kf = self.kernel_size
        pt, pf = self.padding
        if self.tc_ready(x, C):
            return self._forward_tc(x, B, C, T, Fq)
        xp = F.pad(x, (0, 0, pt, pt))
        xi = torch.stack([xp[:, :, dt:dt + T] for dt in range(kt)], 1)            # [B, kt, C, T, F]
        xi = xi.permute(0, 3, 1, 2, 4).reshape(B * T, kt * C, Fq)                 # rows (b, t), channels (dt, c)
        w = self.weight.permute(0, 2, 1, 3).reshape(self.out_channels, kt * C, kf)
        y = ops.conv1d(xi, w, self.bias, None, self.stride[1], 1, (pf, pf), ops.ACT_NONE, 0.0, None)
        return y.view(B, T, self.out_channels, y.shape[-1]).permute(0, 2, 1, 3)

    def _tc_chain_spec(self, C):
        """One-layer engine chain of this conv along frequency; the (dt, c) channel order is a permuted VIEW of the
        parameter, so the weight-norm backward of the chain reaches weight_v / weight_g through autograd."""
        from . import engine
        kt, kf = self.kernel_size
        pt, pf = self.padding
        cin = kt * C
        proxy = self.__dict__.get("_tc_proxy")
        if proxy is None:
            proxy = self.__dict__["_tc_proxy"] = _ParamView()
            if self.__dict__.get("_tc_proxy_static"):       # engine.enable_static_prep ran before the first forward
                proxy.__dict__["_tc_static"] = {}
            spec = engine.LayerSpec("conv", proxy, cin, self.out_channels, kf, self.stride[1], 1, (pf, pf),
                                    ops.ACT_NONE, 0.0, None, True, True)
            spec.cin_pad = (-cin) % 16
            spec.cout_pad = (-self.out_channels) % 16
            self.__dict__["_tc_spec"] = spec
        spec = self.__dict__["_tc_spec"]
        if spec.Cin != cin:
            raise _lib.RaveB200Error(f"DiscConv2d: planned for {spec.Cin // kt} input channels, called with {C}")
        self._tc_refresh_proxy()
        return spec

    def _tc_refresh_proxy(self):
        """(Re)build the proxy's (dt, c)-ordered views of the parameters (a permuted reshape is a copy: it goes stale
        when the parameters move, so engine.refresh_static_prep calls this before it rewrites the static layouts)."""
        proxy = self.__dict__["_tc_proxy"]
        kf = self.kernel_size[1]
        co = self.out_channels
        cin = self.__dict__["_tc_spec"].Cin
        if hasattr(self, "weight_v"):
            proxy.weight_v = self.weight_v.permute(0, 2, 1, 3).reshape(co, cin, kf)
            proxy.weight_g = self.weight_g.reshape(co, 1, 1)
        else:
            proxy.weight = self.weight.permute(0, 2, 1, 3).reshape(co, cin, kf)
        proxy.bias = self.bias

    def _forward_tc(self, x, B, C, T, Fq):
        """bf16 mode: the same conv along frequency as a one-layer chain of the wgmma engine (forward, dgrad and wgrad
        on the tensor cores; 23 % of the v3 discriminator FLOPs ran on the fp32 CUDA-core kernels: 176 ms of a 280 ms
        G-step).  NCHW in, NCHW (view) out; the MRD itself stays channel-last between layers (`forward_cl`)."""
        from . import engine
        spec = self._tc_chain_spec(C)
        kt, pt, co = self.kernel_size[0], self.padding[0], self.out_channels
        # rows (b, t), positions f, channels (dt, c): channel-last bf16 operand of the engine, in one library pass
        rpad = (-Fq) % spec.stride
        x_cl = ops.time_stack_cl(x, kt, pt, kt * C + spec.cin_pad, Fq + rpad)
        (out,) = engine.run_chain(x_cl, [spec], Fq)
        Fo = engine.chain_lengths([spec], Fq)[0]
        return out[:, :Fo, :co].reshape(B, T, Fo, co).permute(0, 3, 1, 2)

    def cout_ok(self) -> bool:
        return self.out_channels % 16 == 0

    def tc_ready(self, x, C) -> bool:
        from . import engine
        return (engine.precision() == "bf16" and x.is_cuda and engine.ACT_DTYPE == torch.bfloat16
                and self.kernel_size[0] * C <= 112)

    def stacked_geometry(self, Fq: int, C: int):
        """(Fp, Cp) of this conv's time-stacked operand for an input of Fq positions and C channels."""
        spec = self._tc_chain_spec(C)
        return Fq + (-Fq) % spec.stride, self.kernel_size[0] * C + spec.cin_pad

    def forward_cl(self, x_cl, xs=None):
        """Channel-last in, channel-last out: x_cl [B, T, F, C] fp32 (a view with dense (f, c) rows) -> the chain's own
        output buffer [(b t), Fo, Cout(+pad to 16)] fp32, which IS [B, T, Fo, Cout] channel-last: no layout pass on
        either side of the conv.  `xs`: the time-stacked bf16 operand when the producer already wrote it
        (ops.leaky_fm_stack: the previous layer's feature tap)."""
        from . import engine
        B, T, Fq, C = x_cl.shape
        spec = self._tc_chain_spec(C)
        kt, pt = self.kernel_size[0], self.padding[0]
        Fp, Cp = self.stacked_geometry(Fq, C)
        if xs is None:
            xs = ops.time_stack_nhwc(x_cl, kt, pt, Cp, Fp)
        elif tuple(xs.shape) != (B * T, Fp, Cp) or xs.dtype != engine.ACT_DTYPE:
            raise _lib.RaveB200Error("DiscConv2d.forward_cl: the pre-stacked operand does not match this conv's geometry")
        (out,) = engine.run_chain(xs, [spec], Fq)
        Fo = engine.chain_lengths([spec], Fq)[0]
        if out.shape[1] != Fo:
            raise _lib.RaveB200Error("DiscConv2d: the one-layer chain's output pitch is its length")
        return out


def _feature_tap(out, slope, B):
    """Post-activation feature of a chain output (rows = [real; fake] when the batch B is even): LeakyReLU and the two L1
    feature-matching sums in one pass (ops.leaky_fm), or the plain activation for an unpaired batch."""
    if B % 2 == 0 and out.dtype == torch.float32 and out.is_contiguous():
        return ops.leaky_fm(out, slope)
    return ops.activation(out, ops.ACT_LEAKY, slope), None


def _feature_tap_stack(out, slope, B, T, nxt):
    """_feature_tap that also writes the time-stacked operand of the next MRD conv `nxt` (a DiscConv2d) in the same pass,
    when the geometry allows it (kt = 3, pt = 1, no channel padding on either side): returns (a, stats, xs | None)."""
    C = out.shape[2]
    if (nxt is not None and B % 2 == 0 and out.dtype == torch.float32 and out.is_contiguous() and os.environ.get(
            "RAVE_FUSE_TAP_STACK", "1") != "0" and nxt.kernel_size[0] == 3 and nxt.padding[0] == 1
            and nxt.in_channels == C and C % 4 == 0 and out.shape[0] == B * T):
        Fp, Cp = nxt.stacked_geometry(out.shape[1], C)
        if Cp == 3 * C:
            return ops.leaky_fm_stack(out, slope, T, Fp)
    a, st = _feature_tap(out, slope, B)
    return a, st, None


class _ParamView:
    """Attribute holder standing in for a conv module inside a one-layer engine chain (engine._layer_params reads
    weight_v / weight_g / bias or weight / bias; the prepared-weight cache lives in its __dict__)."""


def WNConv2d(*args, **kwargs):
    """WNConv2d of the reference for general (kt, kf) kernels (MRD), on the library kernels."""
    act = kwargs.pop("act", True)
    conv = weight_norm(DiscConv2d(*args, **kwargs))
    if not act:
        return conv
    return nn.Sequential(conv, nn.LeakyReLU(0.1))


class MPD(nn.Module):
    """rave/descript_discriminator.py:30-66."""

    def __init__(self, period, n_channels: int = 1):
        super().__init__()
        self.period = period
        self.convs = nn.ModuleList([
            WNConv2dK1(n_channels, 32, (5, 1), (3, 1), padding=(2, 0)),
            WNConv2dK1(32, 128, (5, 1), (3, 1), padding=(2, 0)),
            WNConv2dK1(128, 512, (5, 1), (3, 1), padding=(2, 0)),
            WNConv2dK1(512, 1024, (5, 1), (3, 1), padding=(2, 0)),
            WNConv2dK1(1024, 1024, (5, 1), 1, padding=(2, 0)),
        ])
        self.conv_post = WNConv2dK1(1024, 1, kernel_size=(3, 1), padding=(1, 0), act=False)

    def pad_to_period(self, x):
        t = x.shape[-1]
        # quirk D8: a FULL extra period is appended when t % period == 0
        return F.pad(x, (0, self.period - t % self.period), mode="reflect")

    def _tc_specs(self):
        """Plan of the whole MPD as ONE tensor-core chain (bf16 mode): conv -> LeakyReLU(0.1) -> ... -> conv_post, every
        conv's fp32 output kept (the features are its activation).  The period axis folds into the batch, the Cin = 1
        first layer reads the folded signal in place (engine.TcChainFn)."""
        from . import engine
        if "_tc_specs_cache" not in self.__dict__:
            mods = []
            for layer in self.convs:
                mods += [layer[0], layer[1]]
            mods.append(self.conv_post)
            specs = engine.plan_convnet(nn.Sequential(*mods))
            if specs is not None and not engine.chain_supported(specs):
                specs = None
            self.__dict__["_tc_specs_cache"] = specs
        return self.__dict__["_tc_specs_cache"]

    def _forward_tc(self, x, specs):
        from . import engine
        from .discriminator import ConvNet
        B, C, L, W = x.shape
        xa, _, _, _ = ConvNet._chain_input(None, x, specs)
        outs = engine.run_chain(xa, specs, L)
        lens = engine.chain_lengths(specs, L)
        fmap = []
        for i, (s, o, Lo) in enumerate(zip(specs, outs, lens)):
            # features are POST-activation (descript_discriminator.py:59-61): one elementwise pass over the chain's own
            # [(b w), pitch, C] buffer (rows beyond Lo stay zero), the [B, C, L, W] feature is a VIEW of it
            a, st = _feature_tap(o, self.convs[i][1].negative_slope, B) if i < len(self.convs) else (o, None)
            h = a[:, :Lo, :s.Cout].unflatten(0, (B, W)).permute(0, 3, 2, 1)
            if i < len(self.convs) and not s.cout_pad:
                h._cl_base = a          # dense buffer behind the view (core.mean_difference_halves)
                h._fm_stats = st        # (sum |real - fake|, sum |real|) of this feature, when B is even
            fmap.append(h)
        return fmap

    def forward(self, x):
        from . import engine
        fmap = []
        x = self.pad_to_period(x)
        x = x.reshape(x.shape[0], x.shape[1], -1, self.period)
        if engine.precision() == "bf16" and x.is_cuda and x.shape[1] == 1:
            specs = self._tc_specs()
            if specs is not None:
                return self._forward_tc(x, specs)
        pre = None          # activation of the previous layer, fused into the next conv's operand load
        for layer in self.convs:
            conv, act = layer[0], layer[1]
            h = conv(x, act=None)
            x = ops.activation(h, ops.ACT_LEAKY, act.negative_slope)   # the (post-activation) feature
            fmap.append(x)
        x = self.conv_post(x)
        fmap.append(x)
        return fmap


BANDS = [(0.0, 0.1), (0.1, 0.25), (0.25, 0.5), (0.5, 0.75), (0.75, 1.0)]


class MRD(nn.Module):
    """rave/descript_discriminator.py:118-184 on the library kernels (see the module docstring)."""

    def __init__(self, window_length: int, hop_factor: float = 0.25, sample_rate: int = 44100,
                 bands: list = BANDS, n_channels: int = 1):
        super().__init__()
        self.window_length = window_length
        self.hop_factor = hop_factor
        self.sample_rate = sample_rate
        n_fft = window_length // 2 + 1
        self.bands = [(int(b[0] * n_fft), int(b[1] * n_fft)) for b in bands]
        ch = 32
        convs = lambda: nn.ModuleList([
            WNConv2d(2 * n_channels, ch, (3, 9), (1, 1), padding=(1, 4)),
            WNConv2d(ch, ch, (3, 9), (1, 2), padding=(1, 4)),
            WNConv2d(ch, ch, (3, 9), (1, 2), padding=(1, 4)),
            WNConv2d(ch, ch, (3, 9), (1, 2), padding=(1, 4)),
            WNConv2d(ch, ch, (3, 3), (1, 1), padding=(1, 1)),
        ])
        self.band_convs = nn.ModuleList([convs() for _ in range(len(self.bands))])
        self.conv_post = WNConv2d(ch, 1, (3, 3), (1, 1), padding=(1, 1), act=False)
        # torchaudio.transforms.Spectrogram(n_fft = win_length = window_length, hop, centred, power=None) holds a hann
        # `window` buffer under `stft.window`: same key here
        self.stft = _StftHolder(window_length, int(hop_factor * window_length))

    def spectrogram(self, x):
        B, C, T = x.shape
        st = self.stft
        if x.is_cuda and T > st.n_fft // 2:
            # framing kernel (reflect pad + frame + window; adjoint = overlap-add) + one rfft: [N, frames, bins]
            z = ops.rfft(ops.stft_frames(x.reshape(B * C, T), st.window, st.n_fft, st.hop), st.rfft_bw)
        else:
            z = torch.stft(x.reshape(B * C, T), st.n_fft, hop_length=st.hop, win_length=st.n_fft, window=st.window,
                           center=True, pad_mode="reflect", normalized=False, onesided=True,
                           return_complex=True).transpose(-1, -2)
        z = torch.view_as_real(z)                                           # [(b c), t, f, p]
        t, f = z.shape[1], z.shape[2]
        x = z.reshape(B, C, t, f, 2).permute(0, 1, 4, 2, 3).reshape(B, 2 * C, t, f)   # "b c f t p -> b (c p) t f"
        return [x[..., lo:hi] for lo, hi in self.bands]

    def _forward_cl(self, x):
        """bf16 engine mode: the whole MRD channel-last.  The complex spectrogram [B, t, f, (re, im)] is already the
        channel-last input of the first conv; every conv's output buffer is the next conv's input and -- after the one
        LeakyReLU pass -- the feature (an NCHW *view*, torch's channels_last layout)."""
        B, C, T = x.shape
        st = self.stft
        z = ops.rfft(ops.stft_frames(x.reshape(B * C, T), st.window, st.n_fft, st.hop), st.rfft_bw)
        x0 = torch.view_as_real(z)                                          # [B, t, f, 2]: "b (c p) t f" for c = 1
        t = x0.shape[1]
        fmap, outs = [], []
        for (lo, hi), stack in zip(self.bands, self.band_convs):
            cur = x0[:, :, lo:hi, :]
            xs_next = None
            for li, layer in enumerate(stack):
                conv = layer[0]
                out = conv.forward_cl(cur, xs_next)                          # [(b t), Fo, 32]
                # the tap of every layer but the stack's last also writes the next conv's time-stacked operand
                nxt = stack[li + 1][0] if li + 1 < len(stack) else None
                a, st, xs_next = _feature_tap_stack(out, layer[1].negative_slope, B, t, nxt)
                cur = a.view(B, t, out.shape[1], out.shape[2])
                feat = cur.permute(0, 3, 1, 2)
                feat._cl_base = a
                feat._fm_stats = st
                fmap.append(feat)
            outs.append(cur)
        out = self.conv_post.forward_cl(torch.cat(outs, dim=2))              # [(b t), F, 16]: one score channel + padding
        fmap.append(out.view(B, t, out.shape[1], out.shape[2])[..., :self.conv_post.out_channels].permute(0, 3, 1, 2))
        return fmap

    def forward(self, x):
        if (x.is_cuda and x.shape[1] == 1 and x.shape[-1] > self.stft.n_fft // 2
                and self.conv_post.tc_ready(x, 32) and self.band_convs[0][0][0].cout_ok()):
            return self._forward_cl(x)
        fmap = []
        outs = []
        for band, stack in zip(self.spectrogram(x), self.band_convs):
            for layer in stack:
                h = layer[0](band)
                band = ops.activation(h.contiguous(), ops.ACT_LEAKY, layer[1].negative_slope)   # post-activation feature
                fmap.append(band)
            outs.append(band)
        x = self.conv_post(torch.cat(outs, dim=-1))
        fmap.append(x)
        return fmap


class _StftHolder(nn.Module):
    """State of torchaudio.transforms.Spectrogram that reaches the state_dict (`window`), plus the rfft backward
    weights of ops.RfftFn."""

    def __init__(self, n_fft: int, hop: int):
        super().__init__()
        self.n_fft, self.hop = n_fft, hop
        self.register_buffer("window", torch.hann_window(n_fft))
        bw = torch.full((n_fft // 2 + 1,), 0.5 * n_fft)
        bw[0] = n_fft
        bw[-1] = n_fft
        self.register_buffer("rfft_bw", bw, persistent=False)


class DescriptDiscriminator(nn.Module):
    """rave/descript_discriminator.py:187-217."""

    def __init__(self, rates: list = [], periods: list = [2, 3, 5, 7, 11], fft_sizes: list = [2048, 1024, 512],
                 sample_rate: int = 44100, bands: list = BANDS, n_channels: int = 1):
        super().__init__()
        if rates:
            raise NotImplementedError("MSD is dead code in the reference (descript_discriminator.py:191,201)")
        discs = [MPD(p, n_channels=n_channels) for p in periods]
        discs += [MRD(f, sample_rate=sample_rate, bands=bands, n_channels=n_channels) for f in fft_sizes]
        self.discriminators = nn.ModuleList(discs)

    def preprocess(self, y):
        y = y - y.mean(dim=-1, keepdims=True)
        return 0.8 * y / (y.abs().max(dim=-1, keepdim=True)[0] + 1e-9)

    def forward(self, x):
        x = self.preprocess(x)
        return [d(x) for d in self.discriminators]

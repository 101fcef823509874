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
        """Channel-last operand of the chain.  Cin = 1 (every shipped config): the raw fp32 rows
        [B(*W), pitch] for the small-channel first-layer kernel; otherwise the zero-padded bf16 stream."""
        from . import engine
        first = specs[0]
        if x.dim() == 3:
            B, C, L = x.shape
            W = 1
            rows = x.transpose(1, 2)
        else:
            B, C, L, W = x.shape
            rows = x.permute(0, 3, 2, 1).reshape(B * W, L, C)
        rpad = (-L) % first.stride              # row pitch: a multiple of the first layer's stride
        if C == 1 and first.dil == 1:
            xa = nn.functional.pad(rows.reshape(B * W, L), (0, rpad)).contiguous()
        else:
            xa = nn.functional.pad(rows, (0, first.cin_pad, 0, rpad)).to(engine.ACT_DTYPE).contiguous()
        return xa, B, W, L

    def forward_fm(self, x, period: int = 1, pool: int = 1, fake_grad_only: bool = False):
        """Fused feature-matching path (bf16 engine): x = cat([real, fake]) RAW signal [B, 1, T] -> (stats [n-1, 2],
        counts, score, score_stats [3, 2], n_score) with stats[i] = (sum|h_r - h_f|, sum|h_r|) of hidden feature i,
        counts[i] = its number of elements per half, score = the last conv's output in the reference's shape,
        score_stats = the six sums of the score tail (engine.TcChainFn), n_score = score elements per half.
        `period` > 1: this ConvNet sees MultiPeriodDiscriminator.fold(x, period); `pool` > 1: it sees x average-
        pooled by `pool` (MultiScaleDiscriminator) -- in both cases the first layer reads x in place."""
        from . import engine
        specs = self._tc_specs()
        first = specs[0]
        if x.dim() != 3 or x.shape[1] != 1 or first.Cin != 1 or first.dil != 1:
            raise RuntimeError("forward_fm expects a mono signal [B, 1, T] and a Cin = 1 first layer")
        B, _, T = x.shape
        W = period
        L = (T + period - 1) // period if period > 1 else T // pool
        stats, score_stats, last = engine.run_chain(x.reshape(B, T), specs, L, fm=True, src=(period, pool),
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
        xa, B, W, L = self._chain_input(x, specs)
        outs = engine.run_chain(xa, specs, L)
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
        if engine.precision() != "bf16" or not x.is_cuda or x.dim() != 3 or x.shape[1] != 1:
            return False
        for disc in self.discriminators:
            if not hasattr(disc, "forward_fm"):
                return False
            for layer in disc.layers:
                if not isinstance(layer, ConvNet) or layer._tc_specs() is None:
                    return False
                specs = layer._tc_specs()
                first = specs[0]
                if first.Cin != 1 or first.dil != 1:
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

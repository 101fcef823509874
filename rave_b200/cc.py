"""Host-side mirror of the NON-cached operator layer the reference reaches through the
third-party package `cached-conv>=2.5.0` (requirements.txt:14; semantics: SURVEY.md App. A).

Same names / constructor arguments / attributes as `cached_conv` so the block definitions read
like the reference's (`cc.Conv1d`, `cc.ConvTranspose1d`, `cc.get_padding`, `cc.CachedSequential`,
`cc.AlignBranches`, `cc.CachedPadding1d`, `cc.MAX_BATCH_SIZE`, `cc.USE_BUFFER_CONV`,
`cc.use_cached_conv`), but `forward` launches the sm_90a kernels of librave_b200.so.

gin is not available: the two gin-configurable knobs the reference's configs bind
(`cc.Conv1d.bias = False`, configs/v1.gin:33-34; `cc.get_padding.mode = 'causal'`,
configs/causal.gin:5) are the fields of `cc.config`.
"""
import contextlib
from typing import Tuple

import torch
import torch.nn as nn

from . import ops

MAX_BATCH_SIZE = 64
USE_BUFFER_CONV = False


class _Config:
    conv_bias = False          # cc.Conv1d.bias / cc.ConvTranspose1d.bias
    padding_mode = "centered"  # cc.get_padding.mode
    cached = False             # cc.use_cached_conv: modules constructed afterwards are streaming (ring-buffer) variants


config = _Config()


@contextlib.contextmanager
def configure(conv_bias=None, padding_mode=None):
    old = (config.conv_bias, config.padding_mode)
    if conv_bias is not None:
        config.conv_bias = conv_bias
    if padding_mode is not None:
        config.padding_mode = padding_mode
    try:
        yield
    finally:
        config.conv_bias, config.padding_mode = old


def use_cached_conv(state: bool):
    """cached_conv.use_cached_conv: modules constructed AFTER this call are the streaming variants (SURVEY 8f.4; the
    reference flips it in export / real-time scripts only, `scripts/export.py:436`): every conv keeps the last
    `padding` input samples of each call in a ring buffer instead of zero-padding, so that consecutive calls on consecutive
    chunks reproduce the offline (non-cached, causal-shifted) result, delayed by `cumulative_delay` samples.
    [EXT: cached-conv 2.5.0 is not installable here; the arithmetic below follows its published design (left-only cached
    padding, stride alignment delay, overlap-add cache of the transposed conv, delay lines in AlignBranches) and is pinned
    by the property the reference's own tests check (tests/test_residual.py): streaming == offline up to the delay.]"""
    config.cached = bool(state)


def get_padding(kernel_size: int, stride: int = 1, dilation: int = 1, mode: str = None) -> Tuple[int, int]:
    """'same' padding as a (left, right) pair; `stride` is accepted but unused (App. A)."""
    mode = mode if mode is not None else config.padding_mode
    if kernel_size == 1:
        return (0, 0)
    p = (kernel_size - 1) * dilation + 1
    if mode == "centered":
        return ((p - 1) // 2, p // 2)
    if mode == "causal":
        return (p // 2 + (p - 1) // 2, 0)
    raise Exception(f"Padding mode {mode} is not valid")


def _act_code(act_module):
    """(code, slope, alpha) of an `activation(dim)` module, or None if it cannot be fused."""
    from .blocks import Snake  # local import: blocks imports cc
    if act_module is None:
        return (ops.ACT_NONE, 0.0, None)
    if isinstance(act_module, nn.LeakyReLU):
        return (ops.ACT_LEAKY, float(act_module.negative_slope), None)
    if isinstance(act_module, Snake):
        return (ops.ACT_SNAKE, 0.0, act_module.alpha)
    return None


class Conv1d(nn.Conv1d):
    """cc.Conv1d: explicit asymmetric padding tuple + nn.Conv1d parameters.  `forward(x, act=,
    res=)` optionally fuses the preceding activation module and a residual add into the kernel."""

    def __init__(self, *args, **kwargs):
        pad = kwargs.get("padding", (0, 0))
        if isinstance(pad, int):
            pad = (pad, pad)
        self._pad = tuple(pad)
        kwargs["padding"] = 0
        cd = kwargs.pop("cumulative_delay", 0) or 0
        if "bias" not in kwargs and len(args) < 8:
            kwargs["bias"] = config.conv_bias
        super().__init__(*args, **kwargs)
        self.cumulative_delay = 0
        self._cached = bool(config.cached)
        if self._cached:
            # streaming variant: ALL the padding on the left, served from the previous call's tail; a strided conv first
            # delays its input so that chunk boundaries stay aligned with the stride grid
            r_pad = self._pad[1]
            total = self._pad[0] + self._pad[1]
            st = self.stride[0]
            stride_delay = (st - ((r_pad + cd) % st)) % st
            self.cumulative_delay = (r_pad + stride_delay + cd) // st
            self.cache = CachedPadding1d(total)
            self.downsampling_delay = CachedPadding1d(stride_delay, crop=True)

    def script_cache(self):
        pass

    def forward(self, x, act=None, res=None):
        code = _act_code(act)
        if code is None:
            x = act(x)
            code = (ops.ACT_NONE, 0.0, None)
        alpha = code[2].reshape(-1) if code[2] is not None else None
        if self._cached:
            # (the fused activation is applied on the operand load, after the cache was prepended: pointwise, act(0) = 0)
            x = self.cache(self.downsampling_delay(x))
            w = self.weight
            return ops.conv1d(x, w, self.bias, res, self.stride[0], self.dilation[0], (0, 0), code[0], code[1], alpha) \
                if self.groups == 1 else self._grouped(x, res, (0, 0), code, alpha)
        if self.groups != 1:
            return self._grouped(x, res, self._pad, code, alpha)
        return ops.conv1d(x, self.weight, self.bias, res, self.stride[0], self.dilation[0], self._pad,
                          code[0], code[1], alpha)

    def _grouped(self, x, res, pad, code, alpha):
        """grouped conv (the v1 Encoder's last layer, rave/blocks.py:489-497: groups = n_out): one launch per group on
        its slice of the input / weight channels, same nn.Conv1d parameter layout [Cout, Cin / groups, K]"""
        g = self.groups
        cin, cout = self.in_channels // g, self.out_channels // g
        outs = []
        for i in range(g):
            xi = x[:, i * cin:(i + 1) * cin].contiguous()
            ai = alpha[i * cin:(i + 1) * cin].contiguous() if alpha is not None else None
            bi = self.bias[i * cout:(i + 1) * cout] if self.bias is not None else None
            ri = res[:, i * cout:(i + 1) * cout].contiguous() if res is not None else None
            outs.append(ops.conv1d(xi, self.weight[i * cout:(i + 1) * cout], bi, ri, self.stride[0],
                                   self.dilation[0], pad, code[0], code[1], ai))
        return torch.cat(outs, 1)


class ConvTranspose1d(nn.ConvTranspose1d):
    def __init__(self, *args, **kwargs):
        cd = kwargs.pop("cumulative_delay", 0) or 0
        if "bias" not in kwargs and len(args) < 8:
            kwargs["bias"] = config.conv_bias
        super().__init__(*args, **kwargs)
        if self.groups != 1 or self.output_padding[0] != 0 or self.dilation[0] != 1:
            raise NotImplementedError("only plain ConvTranspose1d is on the hot path")
        self.cumulative_delay = 0
        self._cached = bool(config.cached)
        if self._cached:
            # streaming variant: the un-cropped transposed conv of a chunk overlaps the next chunk's by K - stride samples
            # (overlap-add cache); the symmetric `padding` crop becomes a delay
            self.cumulative_delay = self.padding[0] + cd * self.stride[0]
            self.register_buffer("_tail", torch.zeros(0), persistent=False)

    def script_cache(self):
        pass

    def forward(self, x, act=None):
        code = _act_code(act)
        if code is None:
            x = act(x)
            code = (ops.ACT_NONE, 0.0, None)
        alpha = code[2].reshape(-1) if code[2] is not None else None
        if self._cached:
            y = ops.conv_transpose1d(x, self.weight, None, self.stride[0], 0, code[0], code[1], alpha)
            ov = self.kernel_size[0] - self.stride[0]
            if ov > 0:
                B = y.shape[0]
                if self._tail.numel() == 0 or self._tail.shape[0] < B or self._tail.shape[1:] != (y.shape[1], ov):
                    self._tail = torch.zeros(max(B, 1), y.shape[1], ov, dtype=y.dtype, device=y.device)
                head = y[..., :ov] + self._tail[:B]
                self._tail[:B] = y[..., -ov:].detach()
                y = torch.cat([head, y[..., ov:-ov]], -1)
            if self.bias is not None:
                y = y + self.bias.reshape(1, -1, 1)
            return y
        return ops.conv_transpose1d(x, self.weight, self.bias, self.stride[0], self.padding[0], code[0],
                                    code[1], alpha)


def _is_activation(m) -> bool:
    from .blocks import Snake
    return isinstance(m, (nn.LeakyReLU, Snake))


class CachedSequential(nn.Sequential):
    """cc.CachedSequential.  forward fuses every `activation -> conv` pair into one launch."""

    def __init__(self, *args, **kwargs):
        cumulative_delay = kwargs.pop("cumulative_delay", 0)
        stride = kwargs.pop("stride", 1)
        super().__init__(*args, **kwargs)
        self._cached = bool(config.cached)        # streaming variant: module by module (the ring buffers live in the convs)
        last = 0
        for m in reversed(list(self)):
            if hasattr(m, "cumulative_delay"):
                last = m.cumulative_delay
                break
        self.cumulative_delay = cumulative_delay * stride + last

    def _tc_plan(self):
        """Tensor-core plan of this sequence (None if a member is unsupported), cached per mode."""
        from . import engine
        key = self.training
        cache = self.__dict__.setdefault("_tc_plan_cache", {})
        if key not in cache:
            specs = engine.plan_sequential(list(self))
            if specs is not None and not engine.chain_supported(specs):
                specs = None
            cache[key] = specs
        return cache[key]

    def forward(self, x, res=None):
        from . import engine
        mode = engine.precision()
        x3 = mode == "bf16x3"
        if x3 and torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            mode = "fp32"          # the split-operand mode is a forward path: gradients run on the fp32 kernels
        if res is None and mode in ("bf16", "bf16x3") and x.is_cuda and x.dim() == 3 and not self._cached:
            specs = self._tc_plan()
            if specs is not None and (specs[0].kind != "conv" or x.shape[-1] % specs[0].stride == 0):
                (out,) = engine.run_chain(engine.to_channel_last(x, x3=x3), specs, x3=x3)
                Lout = engine.chain_lengths(specs, x.shape[-1])[-1]
                if out.shape[1] != Lout:
                    out = out[:, :Lout].contiguous()
                return engine.from_channel_last(out)
        mods = list(self)
        i = 0
        n = len(mods)
        while i < n:
            m = mods[i]
            last = i == n - 1
            if _is_activation(m) and i + 1 < n and isinstance(mods[i + 1], (Conv1d, ConvTranspose1d)):
                conv = mods[i + 1]
                if isinstance(conv, Conv1d):
                    x = conv(x, act=m, res=res if i + 1 == n - 1 else None)
                    if i + 1 == n - 1:
                        res = None
                else:
                    x = conv(x, act=m)
                i += 2
                continue
            if isinstance(m, Conv1d) and last and res is not None:
                x = m(x, res=res)
                res = None
            else:
                x = m(x)
            i += 1
        if res is not None:
            x = x + res
        return x


Sequential = CachedSequential


class AlignBranches(nn.Module):
    """Fan-out; in the streaming mode every branch input is delayed so that all branches come out aligned with the
    slowest one (`delays` = each branch's own cumulative delay)."""

    def __init__(self, *branches, delays=None, cumulative_delay=0, stride=1):
        super().__init__()
        self.branches = nn.ModuleList(branches)
        self.cumulative_delay = cumulative_delay
        self._cached = bool(config.cached)
        if self._cached:
            if delays is None:
                delays = [getattr(b, "cumulative_delay", 0) for b in branches]
            max_delay = max(delays) if len(delays) else 0
            self.paddings = nn.ModuleList([CachedPadding1d(max_delay - d, crop=True) for d in delays])
            self.cumulative_delay = int(cumulative_delay * stride) + max_delay

    def forward(self, x):
        if self._cached:
            return [b(p(x)) for b, p in zip(self.branches, self.paddings)]
        return [b(x) for b in self.branches]


class CachedPadding1d(nn.Module):
    """Ring buffer of the last `padding` samples of the previous call, prepended to the next one (zeros before the first
    call); `crop` drops the same number of samples at the end, i.e. a pure delay line.  Identity outside the streaming
    mode or when padding == 0."""

    def __init__(self, padding, crop=False):
        super().__init__()
        self.padding = int(padding)
        self.crop = crop
        self._on = bool(config.cached) and self.padding > 0
        if self._on:
            self.register_buffer("pad", torch.zeros(0), persistent=False)

    def forward(self, x):
        if not self._on:
            return x
        B, C, _ = x.shape
        if self.pad.numel() == 0 or self.pad.shape[0] < B or self.pad.shape[1] != C or self.pad.device != x.device:
            self.pad = torch.zeros(max(B, MAX_BATCH_SIZE), C, self.padding, dtype=x.dtype, device=x.device)
        y = torch.cat([self.pad[:B], x], -1)
        self.pad[:B] = y[..., -self.padding:].detach()
        if self.crop:
            y = y[..., :-self.padding]
        return y

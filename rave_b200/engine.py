"""Tensor-core execution engine: runs a whole conv chain (EncoderV2.net, GeneratorV2.net, a
discriminator ConvNet) on the wgmma kernels in the engine's own layout and precision.

Layout / precision ("bf16 mode", BASELINE config 3): every tensor between two convs is CHANNEL-LAST
([B][L][C]); the operand of each conv is the bf16 tensor `a = act(h)` written by the PRODUCER's
epilogue; the pre-activation stream `h` is written in fp32 only where a later layer needs it (residual
skip) or the caller does (discriminator features, chain output).  The module-boundary layout of the
reference ([B,C,L] fp32) is converted once on entry and once on exit of the chain.

One `torch.autograd.Function` per chain: forward and backward are explicit kernel sequences, so
autograd sees a single node and no intermediate is kept alive except the bf16 operands the backward
needs (LeakyReLU'(h) is recovered from the sign of a = act(h)).

Backward of layer i (operand a_in, output gradient g_i in h-space, bf16):
    wgrad : dWt = sum_rows g_i (x) a_in                 (rave_conv1d_tc_wgrad)
    dgrad : g_prev = (W^T g_i) * LeakyReLU'(a_in) + skip (rave_conv1d_tc_fwd with transposed taps,
                                                         `dact_src` = a_in, `res_bf16` = skip/external grad)
Strided convs' dgrad and ConvTranspose1d's forward are evaluated as `stride` interleaved phases,
each a stride-1 conv over the taps of that phase (no zero-insertion, no wasted MACs).
"""
from dataclasses import dataclass, field
from functools import partial
from typing import Dict, List, NamedTuple, Optional, Tuple

import torch
import torch.nn as nn

from . import _lib, ops

_state = {"precision": "fp32", "prep_epoch": 0}
ACT_DTYPE = torch.bfloat16   # storage type of operand / gradient streams (tests may widen it)

# output positions per tensor-core row of a raw first layer with 16-column operand rows (see RawFirstLayer); rows
# of 32 columns (multichannel, Cin*K > 16) take half as many; pitches that are not a multiple of it run with one
# position (plain W-channel rows)
C1_GROUP = 4
# Residual(DilatedUnit) blocks as ONE launch (csrc/unit_tc.cu) where the width allows it, else two launches per unit
FUSE_UNITS = True


def set_precision(mode: str) -> None:
    """'fp32'   : CUDA-core parity kernels ([B,C,L] fp32, per-layer autograd);
    'bf16'   : wgmma engine (bf16 operands, fp32 accumulate) for every chain it supports (~1e-2 rel-L2 end to end);
    'bf16x3' : the accurate fast mode -- the same wgmma kernels on split operands (x = hi + lo, three MMAs per
               product: hi*hi + lo*hi + hi*lo, fp32 accumulate), <= 1e-4 rel-L2 end to end like the fp32 path, for the
               FORWARD of the encoder / generator chains (no autograd graph: inference, validation, export warm-up);
               anything that needs gradients runs on the fp32 kernels in this mode."""
    if mode not in ("fp32", "bf16", "bf16x3"):
        raise ValueError(mode)
    _state["precision"] = mode


def precision() -> str:
    return _state["precision"]


def invalidate_prepared() -> None:
    """Drop every cached tap-major weight: call after parameters were changed behind autograd's back
    (CUDA-graph replays update them without bumping tensor versions)."""
    _state["prep_epoch"] += 1


@dataclass
class LayerSpec:
    kind: str                      # 'conv' | 'convT'
    module: nn.Module              # owner of weight(_v/_g) / bias
    Cin: int
    Cout: int
    K: int
    stride: int = 1
    dil: int = 1
    pad: Tuple[int, int] = (0, 0)  # conv: (left, right); convT: (padding, padding)
    pre_act: int = ops.ACT_NONE    # activation applied to this layer's INPUT (emitted by its producer)
    pre_slope: float = 0.2
    res_src: Optional[int] = None  # index of the layer whose output stream is added (residual skip)
    want_f32: bool = False         # fp32 stream needed (residual source or external output)
    is_output: bool = False        # returned to the caller (fp32, channel-last)
    cin_pad: int = 0               # zero-padded input channels (Cin=1 layers run with Cin=16)
    cout_pad: int = 0
    res_opnd: Optional[int] = None # index of the layer whose INPUT operand a = LeakyReLU(h_src) carries the
                                   # residual stream: the skip is recovered from it (no fp32 copy of h_src)
    pre_mod: Optional[nn.Module] = None   # the Snake module (owner of alpha) when pre_act == ACT_SNAKE
    res_raw: Optional[int] = None  # Snake units: index of the layer whose raw (pre-Snake) bf16 input IS the skip stream
    adain: Optional[nn.Module] = None     # eval-mode AdaptiveInstanceNormalization applied to this layer's raw input
                                          # stream (before its Snake): the first conv of a Residual(DilatedUnit)


def raw_input_ok(spec: LayerSpec, cin: int) -> bool:
    """True when a chain whose first layer is `spec` can read a raw fp32 signal of `cin` channels in place (TcChainFn:
    the Cin*K taps of a position fit one operand row of 16 columns for mono, 32 for more channels)."""
    return spec.kind == "conv" and spec.Cin == cin and spec.dil == 1 and spec.K * cin <= (16 if cin == 1 else 32)


def chain_supported(specs: List[LayerSpec]) -> bool:
    for s in specs:
        if s.pre_act not in (ops.ACT_NONE, ops.ACT_LEAKY, ops.ACT_SNAKE):
            return False
        cin = s.Cin + s.cin_pad
        cout = s.Cout + s.cout_pad
        if cin % 16 or cout % 16:
            return False
    return True


# ----------------------------------------------------------------------------------------------
# planning: walk a module list into LayerSpecs
# ----------------------------------------------------------------------------------------------

def split_recurrent(mods: List[nn.Module]):
    """(leading blocks.GRU or None, the modules after it): GeneratorV2's `recurrent_layer` (configs/hybrid.gin) opens
    its sequence; it runs on its own kernels (ops.gru) and the rest of the sequence is planned as a chain."""
    from . import blocks
    if mods and isinstance(mods[0], blocks.GRU):
        return mods[0], mods[1:]
    return None, mods


def plan_sequential(mods: List[nn.Module]) -> Optional[List[LayerSpec]]:
    """EncoderV2.net / GeneratorV2.net style sequences: activations (LeakyReLU or Snake), cc.Conv1d, cc.ConvTranspose1d,
    Residual(DilatedUnit), AdaIN (identity in training).  Returns None if something is unsupported.
    Snake (v3): the producer writes its pre-activation as bf16, a channel-last Snake kernel turns it into the next conv's
    operand (and keeps the raw stream for the backward and for the unit's skip).
    An eval-mode AdaIN in front of a Residual(DilatedUnit) of Snake units becomes `adain` of the unit's first conv: the
    chain learns from / transfers the raw stream there (forward only, see TcChainFn).  In front of anything else (a
    LeakyReLU unit) it is not run here.
    A leading GRU is not part of the plan (split_recurrent): the caller runs it first."""
    from . import blocks, cc
    mods = split_recurrent(list(mods))[1]
    specs: List[LayerSpec] = []
    NONE = (ops.ACT_NONE, 0.0, None)
    pending = NONE
    last_idx = -1            # index of the layer producing the current stream (-1 = chain input)
    adain = None             # eval-mode AdaIN waiting for the Residual(DilatedUnit) it feeds

    def act_of(m):
        if isinstance(m, nn.LeakyReLU):
            return (ops.ACT_LEAKY, float(m.negative_slope), None)
        if isinstance(m, blocks.Snake):
            return (ops.ACT_SNAKE, 0.0, m)
        return None

    def add_conv(conv, res_src=None):
        nonlocal pending, last_idx
        if isinstance(conv, cc.Conv1d):
            if conv.groups != 1:
                return False
            Cout, Cin, K = conv.out_channels, conv.in_channels, conv.kernel_size[0]
            spec = LayerSpec("conv", conv, Cin, Cout, K, conv.stride[0], conv.dilation[0], conv._pad,
                             pending[0], pending[1], res_src)
        else:
            Cin, Cout, K = conv.in_channels, conv.out_channels, conv.kernel_size[0]
            spec = LayerSpec("convT", conv, Cin, Cout, K, conv.stride[0], 1,
                             (conv.padding[0], conv.padding[0]), pending[0], pending[1], None)
        spec.pre_mod = pending[2]
        specs.append(spec)
        pending = NONE
        last_idx = len(specs) - 1
        return True

    for m in mods:
        if adain is not None and not isinstance(m, blocks.Residual):
            return None
        if isinstance(m, blocks.AdaptiveInstanceNormalization):
            if not m.training:
                adain = m
            continue
        a = act_of(m)
        if a is not None:
            pending = a
            continue
        if isinstance(m, (cc.Conv1d, cc.ConvTranspose1d)):
            if not add_conv(m):
                return None
            continue
        if isinstance(m, blocks.Residual):
            unit = m.aligned.branches[0]
            if not isinstance(unit, blocks.DilatedUnit):
                return None
            if pending[0] != ops.ACT_NONE:
                return None
            src = last_idx
            if src < 0:
                return None
            a0, c3, a1, c1 = list(unit.net)
            acts = [act_of(a0), act_of(a1)]
            if acts[0] is None or acts[1] is None or acts[0][0] != acts[1][0]:
                return None
            pending = acts[0]
            if not add_conv(c3):
                return None
            c3_idx = last_idx
            if adain is not None:
                if acts[0][0] != ops.ACT_SNAKE:
                    return None
                specs[-1].adain, adain = adain, None
            pending = acts[1]
            if not add_conv(c1, res_src=src):
                return None
            if acts[0][0] == ops.ACT_LEAKY:
                specs[-1].res_opnd = c3_idx       # h_src = unleaky(operand of conv3): no fp32 stream needed
            else:
                specs[-1].res_raw = c3_idx        # Snake is not invertible: the raw bf16 input of conv3 is the skip
            continue
        return None
    if pending[0] != ops.ACT_NONE or adain is not None or not specs:
        return None
    if specs[0].pre_act != ops.ACT_NONE:
        # a chain's operands are activated by their PRODUCER's epilogue; the chain input has no producer, so a
        # sequence that starts with an activation (DilatedUnit.net on its own) is not run here
        return None
    specs[-1].is_output = True
    specs[-1].want_f32 = True
    if specs[-1].Cout % 16:
        # narrow output conv (the raw-waveform generator's 64 -> 2): computed with zero weight rows up to a multiple of
        # 16 output channels, as plan_convnet does for score layers; the caller keeps the first Cout channels
        specs[-1].cout_pad = 16 - specs[-1].Cout % 16
    return specs


def plan_convnet(net: nn.Sequential) -> Optional[List[LayerSpec]]:
    """discriminator.ConvNet.net: [conv, LeakyReLU]*n + conv; every conv output is a feature.
    Works for DiscConv1d and DiscConv2dK1 (the latter over the folded [B*p, H, C] view)."""
    from . import discriminator as D
    specs: List[LayerSpec] = []
    pending = (ops.ACT_NONE, 0.0)
    for m in net:
        if isinstance(m, nn.LeakyReLU):
            pending = (ops.ACT_LEAKY, float(m.negative_slope))
            continue
        if isinstance(m, (D.DiscConv1d, D.DiscConv2dK1)):
            p = m.padding[0]
            spec = LayerSpec("conv", m, m.in_channels, m.out_channels, m.kernel_size[0], m.stride[0],
                             m.dilation[0], (p, p), pending[0], pending[1], None, True, True)
            if spec.Cin % 16:
                spec.cin_pad = 16 - spec.Cin % 16
            if spec.Cout % 16:
                spec.cout_pad = 16 - spec.Cout % 16
            specs.append(spec)
            pending = (ops.ACT_NONE, 0.0)
            continue
        return None
    return specs


# ----------------------------------------------------------------------------------------------
# weights
# ----------------------------------------------------------------------------------------------

def _layer_params(spec: LayerSpec):
    m = spec.module
    if hasattr(m, "weight_v"):
        return m.weight_v, m.weight_g, m.bias
    return m.weight, None, m.bias


def _phase_taps(K: int, stride: int, pad: int, p: int):
    """Taps of output phase p of a transposed map t = l*stride + k - pad: returns (k list in the
    order of increasing source row, pad'') such that source row = q + i - pad'' for tap i."""
    k0 = (p + pad) % stride
    ks = list(range(k0, K, stride))          # k = k0 + stride*m, m = 0..n-1 ; source row = q + c0 - m
    c0 = (p + pad - k0) // stride
    n = len(ks)
    # tap i (increasing source row) has m = n-1-i  ->  row = q + c0 - (n-1) + i
    order = [ks[n - 1 - i] for i in range(n)]
    return order, (n - 1) - c0


def _fused_phase_taps(K: int, stride: int, pad: int):
    """All `stride` output phases of a transposed map as ONE stride-1 conv whose output row q holds the `stride`
    positions q*stride + p side by side: returns (taps, J, pad_l) with taps[j*stride + p] = the parameter tap that
    phase p applies to source row q + j - pad_l (or -1: no tap, zero slab).  The weight [J][stride*C][C'] built from
    this list turns stride launches with strided output rows into one launch with stride-times wider rows
    (same bytes in memory), and the shared source rows are fetched once instead of once per phase."""
    phases = [_phase_taps(K, stride, pad, p) for p in range(stride)]
    omin = min(-padpp for _, padpp in phases)
    omax = max(len(order) - 1 - padpp for order, padpp in phases)
    J = omax - omin + 1
    taps = []
    for j in range(J):
        for order, padpp in phases:
            i = omin + j + padpp
            taps.append(order[i] if 0 <= i < len(order) else -1)
    return taps, J, -omin


def _wide_wgrad_taps(K: int, stride: int, pad: int):
    """Weight gradient of a strided layer on the operand viewed with `stride` positions per row: tap k reads source
    row l*stride + k - pad = (l + j)*stride + p, i.e. row l + j / channel block p of the view.  Returns (J, pad_l,
    slots) with slots[k] = (j - jmin)*stride + p: a J-tap stride-1 wgrad over stride-times wider rows (128-byte-plus
    contiguous TMA rows, the P tiles fetched J times instead of K times)."""
    js = [(k - pad) // stride for k in range(K)]
    jmin = min(js)
    slots = [(j - jmin) * stride + ((k - pad) - j * stride) for k, j in enumerate(js)]
    return max(js) - jmin + 1, -jmin, slots


class ConvLaunch(NamedTuple):
    """One ops.conv1d_tc launch of a prepared layer: the tap-major weight and the geometry it is read with.  phases > 1:
    the launch is the `phases` interleaved phases of a transposed map side by side, output row q holding positions
    q*phases .. q*phases + phases-1 (weight [J][phases*C][C'], see _fused_phase_taps)."""
    w: Optional[torch.Tensor]
    stride: int
    dil: int
    pad: Tuple[int, int]      # as conv1d_tc takes it: (left, right)
    phases: int = 1


class _PreparedWeights:
    """Effective weight of one layer in every tap-major bf16 layout the kernels need, and the launch (`fwd`, `dgrad`:
    ConvLaunch) each layout is read by.  `prepare_layers()` produces the layouts for a whole chain with ONE multi-tensor
    launch pair (row norms + re-layout): rave_weight_prep_tc_multi."""

    def __init__(self, spec: LayerSpec, need_dgrad: bool, need_fwd: bool):
        self.spec = spec
        K, s, dil, pad_l = spec.K, spec.stride, spec.dil, spec.pad[0]
        if spec.kind == "conv":
            self.C0p, self.C1p = spec.Cout + spec.cout_pad, spec.Cin + spec.cin_pad
        else:
            self.C0p, self.C1p = spec.Cin + spec.cin_pad, spec.Cout + spec.cout_pad
        self.norm = None
        self.raw = None           # (norm, outA, outB) as produced by the prep kernel (refresh_static_prep rewrites them)
        # tapsA feeds the launch without phases (conv forward, convT dgrad: [K][C0][C1]), tapsB the transposed one
        # (stride-1 conv dgrad: flipped taps [K][C1][C0]; strided conv dgrad, convT forward: all phases in one launch)
        self.fwd = self.dgrad = None
        if spec.kind == "conv":
            self.tapsA = list(range(K)) if need_fwd else []
            self.fwd = ConvLaunch(None, s, dil, spec.pad) if need_fwd else None
            if not need_dgrad:
                self.tapsB = []
            elif s == 1:
                self.tapsB = list(range(K - 1, -1, -1))
                self.dgrad = ConvLaunch(None, 1, dil, ((K - 1) * dil - pad_l, 0))
            else:
                self.tapsB, _, fused_pad = _fused_phase_taps(K, s, pad_l)
                self.dgrad = ConvLaunch(None, 1, 1, (fused_pad, 0), s)
        else:
            self.tapsB, _, fused_pad = _fused_phase_taps(K, s, pad_l)
            self.fwd = ConvLaunch(None, 1, 1, (fused_pad, 0), s)
            self.tapsA = list(range(K)) if need_dgrad else []
            if need_dgrad:
                self.dgrad = ConvLaunch(None, s, 1, (pad_l, 0))
        if len(self.tapsB) > 32:
            raise _lib.RaveB200Error(f"phase-fused layout of K={K}, stride={s} needs {len(self.tapsB)} > 32 slabs")

    def finalize(self, norm, outA, outB):
        """Attach the prep kernel's layouts to the launches (split-operand layouts, [all hi slabs | all lo slabs] along
        the leading axis, keep that order in the phase-wide view)."""
        self.norm = norm

        def attach(launch, w):
            if launch is None:
                return None
            if launch.phases > 1:       # [J*phases][C1p][C0p] -> [J][phases*C1p][C0p]
                w = w.view(-1, launch.phases * self.C1p, self.C0p)
            return launch._replace(w=w)
        fwd_w, dgrad_w = (outA, outB) if self.spec.kind == "conv" else (outB, outA)
        self.fwd, self.dgrad = attach(self.fwd, fwd_w), attach(self.dgrad, dgrad_w)
        return self


# ---- static prepared weights --------------------------------------------------------------------------------------
# A captured CUDA graph cannot use the version-keyed cache above (replays change parameters behind autograd's back), so
# every replay used to re-prepare every chain.  The discriminator's weights only change in D-steps (1 in 4): with
# `enable_static_prep(model.discriminator)` its prepared layouts live in persistent buffers that the chains read as they
# are, and that `refresh_static_prep` rewrites IN PLACE right after the discriminator's optimiser step (inside the
# D-step graph).  Whoever changes those parameters some other way (load_state_dict, an eager optimiser) must refresh.
# The records live in `module.__dict__["_tc_static"]`: a `_PreparedWeights` (refreshed with all the others by one batched
# prep call) or a `_StaticTensors` (refreshed on its own).

class _StaticTensors:
    """Static record of tensors the batched prep call does not make (the block-diagonal weights of a RawFirstLayer, the
    row norms of a layer that needs no layout): `refresh()` copies `build()`'s fresh values into `tensors` in place.
    `value` is what a chain gets on a hit: the tensors, unless another object carries them."""

    def __init__(self, tensors, build, value=None):
        self.tensors, self.build = tensors, build
        self.value = tensors if value is None else value

    def refresh(self):
        for old, new in zip(self.tensors, self.build()):
            if old is not None:
                old.copy_(new)


class ParamProxy:
    """Stands in for the conv module of a one-layer chain whose operand order is a permutation of its owner's
    parameters (discriminator.TimeStackedConv2d): `_layer_params` reads weight_v / weight_g / bias or weight / bias
    from it, `spec.module` is this object, and the prepared-weight cache and static records live in its __dict__.
    A permuted reshape is a copy, stale once the parameters move: `rebuild()` (the owner's) rewrites the attributes."""

    def __init__(self, owner: nn.Module, spec: LayerSpec, rebuild):
        self.spec, self.rebuild = spec, rebuild
        spec.module = self
        if "_tc_static" in owner.__dict__:       # enable_static_prep ran before the owner's first forward
            self.__dict__["_tc_static"] = {}
        owner.__dict__["_tc_proxy"] = self


def _proxy_of(m: nn.Module) -> Optional[ParamProxy]:
    proxy = m.__dict__.get("_tc_proxy")
    return proxy if isinstance(proxy, ParamProxy) else None


def _static_of(module):
    """The static records of `module` (a conv module or a ParamProxy), or None when it has none: they exist for the
    bf16 operand mode only."""
    return module.__dict__.get("_tc_static") if ACT_DTYPE == torch.bfloat16 else None


def _static_holders(root: nn.Module):
    """Modules under `root` that own prepared weights, plus the ParamProxy of every one-layer chain."""
    for m in root.modules():
        yield m
        proxy = _proxy_of(m)
        if proxy is not None:
            yield proxy


def enable_static_prep(root: nn.Module) -> None:
    for m in root.modules():
        if hasattr(m, "weight_v") or (hasattr(m, "weight") and isinstance(getattr(m, "weight"), nn.Parameter)):
            m.__dict__.setdefault("_tc_static", {})
            proxy = _proxy_of(m)                 # one created later marks itself (ParamProxy.__init__)
            if proxy is not None:
                proxy.__dict__.setdefault("_tc_static", {})


def disable_static_prep(root: nn.Module) -> None:
    for m in _static_holders(root):
        m.__dict__.pop("_tc_static", None)


@torch.no_grad()
def refresh_static_prep(root: nn.Module) -> int:
    """Recompute every static prepared layout under `root` into its existing buffers; returns how many."""
    items, into, single = {False: [], True: []}, {False: [], True: []}, []
    for m in root.modules():
        proxy = _proxy_of(m)
        if proxy is not None and proxy.__dict__.get("_tc_static"):
            proxy.rebuild()              # the proxy's permuted parameter copies are stale once the parameters moved
    for m in _static_holders(root):
        for key, rec in (m.__dict__.get("_tc_static") or {}).items():
            if isinstance(rec, _StaticTensors):
                single.append(rec)
                continue
            v, g, _ = _layer_params(rec.spec)
            x3 = bool(key[2])
            items[x3].append((v.detach(), g.detach() if g is not None else None, rec.tapsA, rec.tapsB, rec.C0p, rec.C1p))
            into[x3].append(rec.raw)
    for x3 in (False, True):
        if items[x3]:
            ops.weight_prep_tc_multi(items[x3], x3=x3, into=into[x3])
    for rec in single:
        rec.refresh()
    return len(items[False]) + len(items[True]) + len(single)


def _row_norms(spec: LayerSpec):
    v, g, _ = _layer_params(spec)
    return (ops.weight_norm_raw(v.detach(), g.detach())[1],)


def _capturing(t: torch.Tensor) -> bool:
    return t.is_cuda and torch.cuda.is_current_stream_capturing()


def prepare_layers(jobs, x3: bool = False):
    """jobs: list of (spec, v, g, need_dgrad, need_fwd).  Returns the list of _PreparedWeights, re-using the module's
    static records or its cache (keyed on parameter versions; bypassed while a CUDA graph is being captured) and
    preparing all misses with one multi-tensor launch pair.  x3: split-operand ([hi slabs | lo slabs]) layouts."""
    slot = "_tc_prep_x3" if x3 else "_tc_prep"
    out = [None] * len(jobs)
    misses = []
    for i, (spec, v, g, need_dgrad, need_fwd) in enumerate(jobs):
        capturing = _capturing(v)
        static = _static_of(spec.module)
        skey = (need_dgrad, need_fwd, x3)
        key = (v._version, g._version if g is not None else -1, need_dgrad, need_fwd, str(ACT_DTYPE), str(v.device),
               v.data_ptr(), _state["prep_epoch"], x3)
        if static is not None:
            hit = static.get(skey)
            if hit is not None:
                out[i] = hit.value if isinstance(hit, _StaticTensors) else hit
                continue
        elif not capturing:
            hit = spec.module.__dict__.get(slot)
            if hit is not None and hit[0] == key:
                out[i] = hit[1]
                continue
        misses.append((i, skey, key, capturing, _PreparedWeights(spec, need_dgrad, need_fwd), v, g))
    work = [(pw, v, g) for (_, _, _, _, pw, v, g) in misses if pw.tapsA or pw.tapsB]
    if work:
        res = ops.weight_prep_tc_multi([(v, g, pw.tapsA, pw.tapsB, pw.C0p, pw.C1p) for (pw, v, g) in work], x3=x3)
        for (pw, _, _), raw in zip(work, res):
            pw.finalize(*raw)
            pw.raw = raw
    for (i, skey, key, capturing, pw, v, g) in misses:
        out[i] = pw
        if pw.raw is None:            # nothing to re-layout (a raw first layer without dgrad): only the norm
            pw.norm = ops.weight_norm_raw(v, g)[1] if g is not None else None
        if capturing:                 # buffers of a capture belong to the graph's pool: only eager calls create a slot
            continue
        static = _static_of(pw.spec.module)
        if static is None:
            if pw.raw is not None:
                pw.spec.module.__dict__[slot] = (key, pw)
        elif pw.raw is not None:
            static[skey] = pw
        elif pw.norm is not None:
            static[skey] = _StaticTensors((pw.norm,), partial(_row_norms, pw.spec), value=pw)
    return out


# ----------------------------------------------------------------------------------------------
# the chain Function
# ----------------------------------------------------------------------------------------------

def _out_len(spec: LayerSpec, Lin: int) -> int:
    if spec.kind == "conv":
        return ops.conv_out_len(Lin, spec.K, spec.stride, spec.dil, spec.pad[0], spec.pad[1])
    return (Lin - 1) * spec.stride - 2 * spec.pad[0] + spec.K


def _pitch(Lout: int, nxt: Optional[LayerSpec]) -> int:
    """Rows allocated per batch for a stream of Lout positions: the consumer's 4-D tensor map needs a multiple of its
    stride."""
    s_next = nxt.stride if (nxt is not None and nxt.kind == "conv") else 1
    return (Lout + s_next - 1) // s_next * s_next


def _zero_rows(tensors, lo: int, hi: int) -> None:
    """Zero the slack rows [:, lo:hi] (positions past the true length) of every tensor given; None entries are skipped."""
    if hi > lo:
        for t in tensors:
            if t is not None:
                t[:, lo:hi].zero_()


def _conv(launch: ConvLaunch, x, Lin: int, Lout: int, pitch: int, act: int, slope: float, out_f32=None, out_act=None,
          bias=None, res=None, res_act=None, res_slope: float = 0.2, res_bf16=None, dact_src=None, fm_d=None,
          fm_partner=None, x3: bool = False) -> None:
    """ops.conv1d_tc of a prepared launch writing positions [0, Lout) of the [B][pitch][C] outputs.  A phase-fused launch
    sees every per-position tensor (outputs, residuals, dact_src, fm_partner) with `phases` positions per row -- the
    same bytes -- and computes every row: the caller zeroes the slack rows after it."""
    q = launch.phases
    act_cs = 0
    if q > 1:
        if pitch % q:
            raise _lib.RaveB200Error("phase-fused conv: the row pitch must be a multiple of the stride")
        pitch = Lout = pitch // q

        def wide(t):
            return t.view(t.shape[0], pitch, q * t.shape[2]) if t is not None else None
        out_f32, out_act, res, res_act, res_bf16, dact_src, fm_partner = (
            wide(t) for t in (out_f32, out_act, res, res_act, res_bf16, dact_src, fm_partner))
        if bias is not None:
            bias = bias.detach().repeat(q)
        if x3:                    # [hi | lo] pairs per position, not per row
            act_cs = launch.w.shape[1] // q
    ops.conv1d_tc(x, launch.w, bias, res, launch.stride, launch.dil, launch.pad, act, slope, want_f32=False,
                  want_act=False, out_f32=out_f32, out_act=out_act, out_rows=pitch, Lout=Lout, Lin=Lin,
                  res_bf16=res_bf16, dact_src=dact_src, res_act=res_act, res_slope=res_slope, fm_d=fm_d,
                  fm_partner=fm_partner, x3=x3, act_cs=act_cs)


def _fused_unit(specs: List[LayerSpec], flat, lens: List[int], i: int, in_pitch: int) -> bool:
    """True when layers i, i+1 are a Residual(DilatedUnit) -- act -> conv3(dil) -> act -> conv1x1 -> + x -- that one
    ops.dilated_unit_tc launch (csrc/unit_tc.cu) can run: LeakyReLU, no bias, equal widths it supports, a length the
    unit keeps and an operand pitch equal to the output's (`in_pitch`)."""
    if i + 1 >= len(specs):
        return False
    s, s1 = specs[i], specs[i + 1]
    s2 = specs[i + 2] if i + 2 < len(specs) else None
    return (s.kind == "conv" and s1.kind == "conv" and s.K == 3 and s1.K == 1 and s.stride == 1 and s1.stride == 1
            and s.pre_act == ops.ACT_LEAKY and s1.pre_act == ops.ACT_LEAKY and s1.res_opnd == i
            and s.res_src is None and s.res_opnd is None and flat[3 * i + 2] is None and flat[3 * i + 5] is None
            and s.Cin == s.Cout == s1.Cin == s1.Cout and not (s.cin_pad or s.cout_pad or s1.cin_pad or s1.cout_pad)
            and lens[i] == lens[i + 1] == lens[i + 2] and ops.dilated_unit_tc_supported(s.Cin, lens[i])
            and _pitch(lens[i + 1], s2) == in_pitch)


class RawFirstLayer:
    """First layer of a chain that reads the raw fp32 signal in place (raw_input_ok), one object per forward, kept for
    the backward.  The Cin*K taps become the W (16 or 32) "channels" of a tiny im2col X[r][l][c*K + k].  G = 64 / W
    consecutive positions are then read as ONE 64-channel row (X viewed as [R][L/G][64], 128-byte TMA rows instead of
    2W-byte ones) against the block-diagonal weight kron(I_G, w): the output row holds the G x Cout results of those
    positions, i.e. the same bytes as out[r][G*lg + p][co].  The geometry (W, G, the padded length Xp) is decided here
    and nowhere else: the output, its gradient and X are all viewed through `_rows`."""

    def __init__(self, spec: LayerSpec, cin: int, period: int, pool: int, src_shape, pitch: int, Lin: int, Lout: int):
        self.spec, self.period, self.pool, self.src_shape = spec, period, pool, tuple(src_shape)
        self.pitch, self.Lin, self.Lout = pitch, Lin, Lout
        self.W = ops.cin_width(cin, spec.K)
        G = max(1, C1_GROUP * 16 // self.W)
        self.G = G if pitch % G == 0 else 1      # the output (and so its gradient) must split into rows of G positions
        self.Xp = (Lout + self.G - 1) // self.G * self.G
        self.X = None             # im2col operand, [B][Xp][W]
        self.w_dgrad = None       # [1][G*W][G*Cout_p]

    def _rows(self, t):
        """[B][L][C] viewed with G positions per row; None passes through."""
        return t.view(t.shape[0], t.shape[1] // self.G, self.G * t.shape[2]) if t is not None else None

    @staticmethod
    def _build_weights(s: LayerSpec, G: int, W: int):
        """(forward weight [1][G*Cout_p][G*W], its transpose for the dgrad, bias repeated G times) from the parameters
        as they are now."""
        v, g, b = _layer_params(s)
        cout_p = s.Cout + s.cout_pad
        w_eff = ops.weight_norm_raw(v.detach(), g.detach())[0] if g is not None else v.detach()
        w_blk = nn.functional.pad(w_eff.reshape(s.Cout, s.Cin * s.K), (0, W - s.Cin * s.K, 0, s.cout_pad))  # [Cout_p, W]
        if G > 1:
            eye = torch.eye(G, dtype=w_blk.dtype, device=w_blk.device)
            w_blk = (eye[:, None, :, None] * w_blk[None, :, None, :]).reshape(G * cout_p, G * W)
        if b is not None:
            b = nn.functional.pad(b.detach(), (0, s.cout_pad)) if s.cout_pad else b.detach()
            if G > 1:
                b = b.repeat(G)
        return (w_blk.to(ACT_DTYPE).unsqueeze(0).contiguous(), w_blk.t().contiguous().to(ACT_DTYPE).unsqueeze(0), b)

    def weights(self):
        """The three tensors of _build_weights: the module's static record when it has one (made by the first eager
        call), else built from the current parameters."""
        build = partial(self._build_weights, self.spec, self.G, self.W)
        static = _static_of(self.spec.module)
        rec = static.get(("raw", self.G)) if static is not None else None
        if rec is not None:
            return rec.tensors
        tensors = build()
        if static is not None and not _capturing(self.X):
            static[("raw", self.G)] = _StaticTensors(tensors, build)
        return tensors

    def forward(self, a, out_f32, out_act, act_code, act_slope):
        s, rows = self.spec, self.Xp // self.G
        im2col = ops.im2col_c1 if a.dim() == 2 else ops.im2col_cin         # mono rows [Bs, T] / [Bs, Cin, T]
        self.X = im2col(a, self.Lin, self.Lout, self.Xp, s.K, s.stride, s.pad[0], self.period, self.pool)
        w_fwd, self.w_dgrad, bias_g = self.weights()
        # positions Lout .. Xp-1 of the last group see zero taps but get the bias: the caller zeroes them
        ops.conv1d_tc(self._rows(self.X), w_fwd, bias_g, None, 1, 1, (0, 0), act_code, act_slope, want_f32=False,
                      want_act=False, out_f32=self._rows(out_f32), out_act=self._rows(out_act), Lout=rows, Lin=rows,
                      out_rows=self.pitch // self.G)

    def wgrad(self, g, db):
        """Weight gradient partials [1][K][Cout][Cin] from the output gradient g [B][pitch][Cout_p]; the bias gradient
        goes to `db` (or nowhere: None)."""
        s, G, W = self.spec, self.G, self.W
        cout_p = s.Cout + s.cout_pad
        if G > 1:
            # the wanted [Cout][W] gradient is the sum of the G diagonal blocks of the [G*Cout][G*W] result
            rows = (self.Lout + G - 1) // G
            dbw = torch.zeros(G * cout_p, dtype=torch.float32, device=g.device) if db is not None else None
            d = ops.conv1d_tc_wgrad(self._rows(g), self._rows(self.X), 1, 1, 1, 0, Lp=rows, Lq=rows, dbias=dbw)
            dw_full = torch.diagonal(d.sum(0)[0].view(G, cout_p, G, W), dim1=0, dim2=2).sum(-1)   # [Cout_p][W]
            if db is not None:
                db.copy_(dbw.view(G, cout_p).sum(0))
        else:
            dw_full = ops.conv1d_tc_wgrad(g, self.X, 1, 1, 1, 0, Lp=self.Lout, Lq=self.Lout, dbias=db).sum(0)[0]
        dw_ck = dw_full[:s.Cout, :s.Cin * s.K].reshape(s.Cout, s.Cin, s.K)                     # [Cout][Cin][K]
        return dw_ck.permute(2, 0, 1).reshape(1, s.K, s.Cout, s.Cin).contiguous()              # [1][K][C0][C1]

    def dgrad(self, g, fake_only: bool):
        """Gradient of the source signal: P[r][l][c*K + k] = <g[r][l][:], w[:][c][k]> on the tensor cores (slack rows
        of g are zero), then a gather.  fake_only: g holds the second half of the source batches."""
        s = self.spec
        rows = g.shape[1] // self.G if self.G > 1 else self.Lout
        P, _ = ops.conv1d_tc(self._rows(g), self.w_dgrad, None, None, 1, 1, (0, 0), ops.ACT_NONE, 0.0, want_f32=True,
                             want_act=False, Lout=rows, Lin=rows)
        gather = ops.gather_c1 if len(self.src_shape) == 2 else ops.gather_cin
        return gather(P.view(g.shape[0], -1, self.W), self.src_shape, self.Lin, self.Lout, s.K, s.stride, s.pad[0],
                      self.period, self.pool, batch0=self.src_shape[0] // 2 if fake_only else 0)


class TcChainFn(torch.autograd.Function):
    """forward(x, specs, L0, fm, *flat_params).

    x   : [B, pitch, Cin(+pad)] operand stream (ACT_DTYPE), or -- when the first layer passes raw_input_ok --
          a raw fp32 signal tensor, [Bs, T] (mono) or [Bs, Cin, T] with `src` given, from which the chain rows are
          read in place: `src = (period, pool)` (L0 = positions per row; B = Bs*period rows; MPD fold / MSD pooling,
          ops.im2col_c1 / ops.im2col_cin); no padding to 16 channels, no bf16 rounding of the audio, no folded /
          pooled copy.
    fm  : False -> returns one fp32 channel-last tensor per `is_output` layer;
          True  -> discriminator feature-matching mode: the batch is [real; fake]; returns
                   (stats [n-1, 2] = per hidden layer (sum|h_r-h_f|, sum|h_r|),
                    score_stats [3, 2] = ((sum|s_r-s_f|, sum|s_r|), (sum relu(1-s_r), sum relu(1+s_f)),
                                          (sum s_r, sum s_f)) of channel 0 of the last layer -- zeros unless that
                                          layer has one output channel,
                    last layer fp32 output).
                   Hidden features never reach HBM in fp32; the losses are assembled from the two small stats
                   tensors (RAVE._fused_feature_matching), whose gradients drive fm_grad / score_grad here."""

    @staticmethod
    def forward(ctx, x_in, specs, L0, fm, src, fake_grad_only, x3, *flat):
        n = len(specs)
        ctx.set_materialize_grads(False)
        need_dgrad = x_in.requires_grad or any(t is not None and t.requires_grad for t in flat)
        if any(s.adain is not None for s in specs):
            need_dgrad = False     # eval-mode AdaIN chains are forward only (run_chain refuses them under autograd)
        if x3:
            # split-operand mode: forward chains only (x_in rows are [hi | lo]); the caller keeps autograd away
            if fm or x_in.dim() == 2:
                raise _lib.RaveB200Error("bf16x3: discriminator chains are not run in the split-operand mode")
            need_dgrad = False
        AW = 2 if x3 else 1                    # operand row width multiplier
        # Snake layers (v3): their alpha parameters follow the 3n (v, g, bias) entries of `flat`
        alpha_idx: Dict[int, int] = {}
        for i, s in enumerate(specs):
            if s.pre_act == ops.ACT_SNAKE:
                alpha_idx[i] = 3 * n + len(alpha_idx)
        if alpha_idx and (x3 or fm):
            raise _lib.RaveB200Error("Snake chains run in the plain bf16 mode only (no split operands, no fused fm)")
        hraw: Dict[int, torch.Tensor] = {}     # raw (pre-Snake) bf16 input stream of layer i
        lens = [L0] + chain_lengths(specs, L0)
        raw: Optional[RawFirstLayer] = None
        period = 1
        if x_in.dim() == 2 or src is not None:         # raw fp32 signal, read in place by the first layer
            period, pool = src if src is not None else (1, 1)
            cin = x_in.shape[1] if x_in.dim() == 3 else 1
            if not raw_input_ok(specs[0], cin):
                raise _lib.RaveB200Error("raw fp32 rows are only accepted by a first conv with Cin = the signal's "
                                         "channels, Cin * K <= 32 and no dilation")
            raw = RawFirstLayer(specs[0], cin, period, pool, x_in.shape, _pitch(lens[1], specs[1] if n > 1 else None),
                                L0, lens[1])
        B = x_in.shape[0] * period
        ctx.B = B
        # backward on the fake half only (see backward): always available to the fused feature-matching chains, and to
        # plain conv stacks (no residuals, no Snake: the Descript discriminator) whose caller asked for it
        plain = all(s.kind == "conv" and s.res_src is None and s.res_opnd is None and s.res_raw is None
                    and s.pre_act != ops.ACT_SNAKE for s in specs)
        ctx.fake_grad_only = bool(fake_grad_only) and (fm or (plain and B % 2 == 0 and not x3))
        dev = x_in.device
        a = x_in
        f32: Dict[int, torch.Tensor] = {}
        acts: List[torch.Tensor] = []                 # operand consumed by layer i
        outputs = []
        stats = torch.zeros(max(n - 1, 1), 2, dtype=torch.float32, device=dev) if fm else None
        jobs = []
        for i, s in enumerate(specs):
            own = raw is not None and i == 0        # a RawFirstLayer makes its own layouts: only the row norms here
            jobs.append((s, flat[3 * i].detach(), flat[3 * i + 1].detach() if flat[3 * i + 1] is not None else None,
                         need_dgrad and not own, not own))
        prepared = prepare_layers(jobs, x3=x3)
        # one step per launch, (first layer, last layer): a Residual(DilatedUnit) runs as ONE kernel where it can (the
        # intermediate operand stays in shared memory, written to HBM only when a backward will need it)
        fuse = FUSE_UNITS and not x3 and not fm and ACT_DTYPE == torch.bfloat16
        steps, i = [], 0
        while i < n:
            in_pitch = x_in.shape[1] if i == 0 else _pitch(lens[i], specs[i])
            j = i + 1 if fuse and (raw is None or i > 0) and _fused_unit(specs, flat, lens, i, in_pitch) else i
            steps.append((i, j))
            i = j + 1
        for i, j in steps:
            s = specs[j]                # the layer whose output this step writes
            Lout = lens[j + 1]
            nxt = specs[j + 1] if j + 1 < n else None
            want_act = nxt is not None
            act_code = nxt.pre_act if nxt is not None else ops.ACT_NONE
            act_slope = nxt.pre_slope if nxt is not None else 0.0
            snake_next = act_code == ops.ACT_SNAKE
            if snake_next:              # the epilogue writes h as bf16; ops.snake_cl_fwd makes the operand (below)
                act_code = ops.ACT_NONE
            want_f32 = s.want_f32 and not (fm and nxt is not None)
            pitch = _pitch(Lout, nxt)
            cout_p = s.Cout + s.cout_pad
            out_f32 = torch.empty(B, pitch, cout_p, dtype=torch.float32, device=dev) if want_f32 else None
            out_act = torch.empty(B, pitch, AW * cout_p, dtype=ACT_DTYPE, device=dev) if want_act else None
            acts.append(a)
            if j > i:
                unit = prepared[i].fwd
                a1, _, _ = ops.dilated_unit_tc(a, unit.w, prepared[j].fwd.w, unit.dil, unit.pad[0], specs[i].pre_slope,
                                               s.pre_slope, act_code, act_slope, L=Lout, want_a1=need_dgrad,
                                               out_f32=out_f32, out_act=out_act)
                acts.append(a1)
            elif raw is not None and i == 0:
                raw.forward(a, out_f32, out_act, act_code, act_slope)
            else:
                bias = flat[3 * i + 2]
                if bias is not None and s.cout_pad:
                    bias = nn.functional.pad(bias.detach(), (0, s.cout_pad))
                res = res_act = res_b16 = None
                res_slope = 0.2
                if s.res_opnd is not None:
                    res_act, res_slope = acts[s.res_opnd], specs[s.res_opnd].pre_slope
                elif s.res_raw is not None:
                    res_b16 = hraw[s.res_raw]
                elif s.res_src is not None:
                    res = f32[s.res_src]
                _conv(prepared[i].fwd, a, lens[i], Lout, pitch, act_code, act_slope, out_f32=out_f32, out_act=out_act,
                      bias=bias, res=res, res_act=res_act, res_slope=res_slope, res_bf16=res_b16, x3=x3)
            # positions past the true length: rows a launch did not write, or computed from zero taps (phase-fused
            # launches, the last group of a raw first layer)
            _zero_rows((out_f32, out_act), Lout, pitch)
            if snake_next:
                hraw[j + 1] = out_act
                ad = nxt.adain
                if ad is None:
                    out_act = ops.snake_cl_fwd(out_act, flat[alpha_idx[j + 1]])
                else:
                    # AdaIN on the raw stream: statistics / running update, then h <- h scale + shift in place (the
                    # unit's skip reads hraw) and the Snake operand of the transformed stream
                    scale, shift = ops.adain_cl_stats(out_act, Lout, ad.mean_x, ad.std_x, ad.mean_y, ad.std_y,
                                                      ad.learn_x, ad.learn_y, ad.num_update_x, ad.num_update_y)
                    out_act = ops.adain_snake_cl_fwd(out_act, flat[alpha_idx[j + 1]], scale, shift, Lout)
            if fm and nxt is not None:
                if act_code != ops.ACT_LEAKY or s.cout_pad:
                    raise _lib.RaveB200Error("feature-matching mode needs LeakyReLU between the layers")
                ops.fm_stats(out_act, stats[j], Lout, act_slope)
            if want_f32:
                f32[j] = out_f32
            if (s.is_output and not fm) or (fm and nxt is None):
                outputs.append(out_f32)
            a = out_act
        score_stats = None
        if fm:
            score_stats = torch.zeros(3, 2, dtype=torch.float32, device=dev)
            ctx.score_f32 = None
            if specs[-1].Cout == 1:
                ops.score_stats(outputs[-1], score_stats, lens[-1])
                ctx.score_f32 = outputs[-1]
        ctx.specs = specs
        ctx.hraw = hraw
        ctx.alpha_idx = alpha_idx
        ctx.acts = acts
        ctx.prepared = prepared
        ctx.lens = lens
        ctx.params = flat
        ctx.fm = fm
        ctx.raw = raw
        ctx.x_requires_grad = x_in.requires_grad
        ctx.out_index = [i for i, s in enumerate(specs) if s.is_output]
        if fm:
            return (stats, score_stats) + tuple(outputs)
        return tuple(outputs)

    @staticmethod
    def backward(ctx, *gouts):
        specs = ctx.specs
        n = len(specs)
        flat = ctx.params
        B = ctx.B
        # Generator step through a discriminator chain ([real; fake] batch, frozen parameters): the gradient of the real
        # rows only ever reaches the real INPUT, which nobody asks for -- conv layers do not mix batch rows, the
        # feature-matching term of the fake rows needs the real activations only as constants.  Run the whole backward
        # on the fake half (half the dgrad FLOPs and bytes).
        fo = ctx.fake_grad_only and not any(t is not None and t.requires_grad for t in flat)
        Bh = B // 2
        if fo:
            B = Bh

        def half(t):
            return t[Bh:] if (fo and t is not None) else t
        ext: Dict[int, torch.Tensor] = {}      # external gradient of layer i's output (ACT_DTYPE, h-space)
        dstats = None
        if ctx.fm:
            dstats = gouts[0]
            if dstats is not None:
                dstats = dstats.contiguous()
            if gouts[2] is not None:
                ext[n - 1] = half(gouts[2].to(ACT_DTYPE).contiguous())
            if gouts[1] is not None and ctx.score_f32 is not None:
                e = half(ops.score_grad(ctx.score_f32, gouts[1].to(torch.float32).contiguous(), ctx.lens[-1]))
                ext[n - 1] = e if (n - 1) not in ext else ext[n - 1] + e
        else:
            for i, g in zip(ctx.out_index, gouts):
                if g is not None:
                    ext[i] = half(g).to(ACT_DTYPE).contiguous()
        skip: Dict[int, torch.Tensor] = {}     # residual pass-through gradient for layer idx (or -1)
        g_cur: Optional[torch.Tensor] = None   # gradient (h-space) of layer i's output
        grads = [None] * len(flat)
        gx = None
        wn_jobs = []       # (layer, dwt partials, v, g, norm): one multi-tensor launch at the end
        # bias gradients accumulated by the wgrad kernels: ONE zero-filled buffer for the whole chain
        db_off, db_total = {}, 0
        for i, s in enumerate(specs):
            bias_i, v_i = flat[3 * i + 2], flat[3 * i]
            if s.kind == "conv" and bias_i is not None and bias_i.requires_grad and v_i.requires_grad:
                db_off[i] = db_total
                db_total += (s.Cout + s.cout_pad + 7) // 8 * 8
        db_all = torch.zeros(db_total, dtype=torch.float32, device=ctx.acts[-1].device) if db_total else None
        for i in range(n - 1, -1, -1):
            s = specs[i]
            pw = ctx.prepared[i]
            raw = ctx.raw if i == 0 else None
            a_full = ctx.acts[i]
            a_in = a_full if raw is not None else half(a_full)
            Lin, Lout = ctx.lens[i], ctx.lens[i + 1]
            g = g_cur
            if g is None:
                g = ext.get(i)
                if g is None:
                    raise _lib.RaveB200Error("chain backward: no gradient reaches the last layer")
            if s.res_src is not None:
                skip[s.res_src] = g
            cin_p, cout_p = s.Cin + s.cin_pad, s.Cout + s.cout_pad
            v, gpar, bias = flat[3 * i], flat[3 * i + 1], flat[3 * i + 2]
            # ---- weight gradient (+ bias gradient: column sums of g, taken by the wgrad kernel from the tiles it
            #      streams when g is its P operand, i.e. for conv layers)
            want_db = bias is not None and bias.requires_grad
            db = None
            remap = None
            if v.requires_grad:
                if i in db_off:
                    db = db_all[db_off[i]:db_off[i] + cout_p]
                if raw is not None:
                    dwt = raw.wgrad(g, db)
                else:
                    P_op, Q_op = (g, a_in) if s.kind == "conv" else (a_in, g)
                    Lp_, Lq_ = (Lout, Lin) if s.kind == "conv" else (Lin, Lout)
                    st = s.stride
                    J, padw, slots = _wide_wgrad_taps(s.K, st, s.pad[0]) if st > 1 else (0, 0, None)
                    if st > 1 and s.dil == 1 and Q_op.shape[1] % st == 0 and s.K <= 32 and 4 * J * st <= 5 * s.K:
                        # strided layer with many taps (K = 15, stride 4: 16 slots for 15 taps): wgrad on the Q operand
                        # viewed with `stride` positions per row.  Short kernels (K = 5: 8 slots) would waste the MMAs.
                        Bq, qp, cq = Q_op.shape
                        dwt = ops.conv1d_tc_wgrad(P_op, Q_op.view(Bq, qp // st, st * cq), J, 1, 1, padw, Lp=Lp_,
                                                  Lq=(Lq_ + st - 1) // st, dbias=db)
                        remap = (st, slots)
                    else:
                        dwt = ops.conv1d_tc_wgrad(P_op, Q_op, s.K, st, s.dil if s.kind == "conv" else 1, s.pad[0],
                                                  Lp=Lp_, Lq=Lq_, dbias=db)
                # dwt is [S][K][C0p][C1p] (or the phase-wide form + remap) in the parameter's own (C0, C1) order
                wn_jobs.append((i, dwt, v, gpar, pw.norm, remap))
            if want_db:
                grads[3 * i + 2] = db[:s.Cout] if db is not None else ops.colsum_bf16(g, Lout, s.Cout)
            # ---- input gradient
            need_prev = i > 0 or ctx.x_requires_grad
            if not need_prev:
                break
            prev = i - 1
            add = None
            if prev in skip:
                add = skip.pop(prev)
            e = ext.get(prev) if prev >= 0 else None
            fm_d = None
            if ctx.fm and prev >= 0 and dstats is not None:
                # feature-matching gradient of hidden feature `prev`: computed inside this layer's dgrad epilogue from
                # the saved operand a_in (real and fake rows), no gradient tensor of its own
                fm_d = dstats[prev]
                if s.pre_act != ops.ACT_LEAKY or raw is not None:
                    raise _lib.RaveB200Error("fused feature-matching gradient needs a LeakyReLU operand")
            if e is not None:
                add = e if add is None else (add + e)
            dact = a_in if s.pre_act == ops.ACT_LEAKY else None
            snake_here = s.pre_act == ops.ACT_SNAKE
            add_conv = None if snake_here else add       # Snake: the skip / external gradient joins after dSnake
            fm_partner = a_full[:Bh] if (fo and fm_d is not None) else None
            in_pitch = a_in.shape[1]
            if raw is not None:
                gx = raw.dgrad(g, fo)
                break
            if fo and i == 0:
                # fake-rows-only backward: the chain's input gradient is [zeros; gx_fake] -- the last dgrad writes its
                # rows straight into the second half of the full buffer (no zeros + copy pass afterwards)
                gx = torch.empty(ctx.B, in_pitch, cin_p, dtype=ACT_DTYPE, device=g.device)
                gx[:Bh].zero_()
                gp = gx[Bh:]
            else:
                gp = torch.empty(B, in_pitch, cin_p, dtype=ACT_DTYPE, device=g.device)
            _conv(pw.dgrad, g, Lout, Lin, in_pitch, ops.ACT_NONE, s.pre_slope, out_act=gp, res_bf16=add_conv,
                  dact_src=dact, fm_d=fm_d, fm_partner=fm_partner)
            _zero_rows((gp,), Lin, in_pitch)
            if snake_here:
                al = flat[ctx.alpha_idx[i]]
                gp, dal = ops.snake_cl_bwd(gp, ctx.hraw[i], al, add, want_dalpha=bool(al.requires_grad))
                if dal is not None:
                    grads[ctx.alpha_idx[i]] = dal.reshape(al.shape)
            g_cur = gp
            if i == 0 and not fo:       # (fake rows only: no Snake, gp is the second half of gx)
                gx = gp
        if wn_jobs:
            res = ops.weight_norm_bwd_multi([job[1:] for job in wn_jobs])
            for job, (dv, dg) in zip(wn_jobs, res):
                i = job[0]
                grads[3 * i], grads[3 * i + 1] = dv, dg
        return (gx, None, None, None, None, None, None) + tuple(grads)


_FAKE_ROWS_ONLY = False


class fake_rows_only:
    """Context: chains run inside it hold [real; fake] rows and their caller only ever uses the gradient reaching the
    FAKE rows (generator step through a frozen discriminator, rave/model.py:348-379): their backward runs on that half.
    No effect on chains with trainable parameters, residuals or Snake."""

    def __init__(self, state: bool = True):
        self.state = bool(state)

    def __enter__(self):
        global _FAKE_ROWS_ONLY
        self.prev, _FAKE_ROWS_ONLY = _FAKE_ROWS_ONLY, self.state
        return self

    def __exit__(self, *exc):
        global _FAKE_ROWS_ONLY
        _FAKE_ROWS_ONLY = self.prev
        return False


def run_chain(x_cl_bf16: torch.Tensor, specs: List[LayerSpec], L0: Optional[int] = None, fm: bool = False,
              src: Optional[Tuple[int, int]] = None, fake_grad_only: bool = False, x3: bool = False):
    """x_cl_bf16: [B, pitch, Cin(+pad)] (rows beyond the true length L0 must be zero), or raw fp32 rows
    [B, pitch] for a Cin = 1 first layer, or [B, Cin, pitch] with `src` given (engine.raw_input_ok).  Returns one fp32 channel-last tensor [B, pitch_i, Cout_i(+pad)]
    per output layer (slice [:, :L_i, :Cout_i]); with fm=True: (stats [n-1, 2], score_stats [3, 2], last layer
    output)."""
    flat = []
    for s in specs:
        v, g, b = _layer_params(s)
        flat += [v, g, b]
    flat += [s.pre_mod.alpha for s in specs if s.pre_act == ops.ACT_SNAKE]      # after the 3n weight entries
    if any(s.adain is not None for s in specs) and torch.is_grad_enabled() and (
            x_cl_bf16.requires_grad or any(t is not None and t.requires_grad for t in flat)):
        raise _lib.RaveB200Error("a chain with eval-mode AdaIN runs without autograd only (no backward through the "
                                 "style statistics)")
    if L0 is None:
        L0 = x_cl_bf16.shape[1]
    return TcChainFn.apply(x_cl_bf16, specs, L0, fm, src, fake_grad_only or _FAKE_ROWS_ONLY, x3, *flat)


def chain_lengths(specs: List[LayerSpec], L0: int) -> List[int]:
    out, L = [], L0
    for s in specs:
        L = _out_len(s, L)
        out.append(L)
    return out


class _ToChannelLast(torch.autograd.Function):
    """[B,C,L] fp32 -> [B,L,C(+pad)] bf16; backward converts the bf16 channel-last gradient back."""

    @staticmethod
    def forward(ctx, x, cpad):
        yb, _ = ops.ncl_to_cl(x)
        ctx.C = x.shape[1]
        if cpad:
            yb = nn.functional.pad(yb, (0, cpad))
        return yb

    @staticmethod
    def backward(ctx, g):
        return g[..., :ctx.C].float().permute(0, 2, 1).contiguous(), None


class _FromChannelLast(torch.autograd.Function):
    """[B,L,C] fp32 channel-last -> [B,C,L] fp32 (kernel transpose both ways)."""

    @staticmethod
    def forward(ctx, x_cl):
        return ops.cl_to_ncl(x_cl)

    @staticmethod
    def backward(ctx, g):
        _, gf = ops.ncl_to_cl(g.contiguous(), want_bf16=False, want_f32=True)
        return gf


def to_channel_last(x, cpad=0, x3=False):
    if x3:                       # split operand rows [hi | lo]; forward-only path, no autograd node
        y = ops.ncl_to_cl_x3(x.detach())
        if cpad:
            B, L, C2 = y.shape
            y = nn.functional.pad(y.view(B, L, 2, C2 // 2), (0, cpad)).reshape(B, L, C2 + 2 * cpad)
        return y
    return _ToChannelLast.apply(x, cpad)


def from_channel_last(x_cl):
    return _FromChannelLast.apply(x_cl)

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
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from . import _lib, ops

_state = {"precision": "fp32", "prep_epoch": 0}
ACT_DTYPE = torch.bfloat16   # storage type of operand / gradient streams (tests may widen it)


import os as _os
# output positions per tensor-core row of a Cin = 1 first layer (see TcChainFn.forward); 1 = plain 16-channel rows
C1_GROUP = int(_os.environ.get("RAVE_C1_GROUP", "4"))
# Residual(DilatedUnit) blocks as ONE launch (csrc/unit_tc.cu) where the width allows it; 0 = two launches per unit
FUSE_UNITS = _os.environ.get("RAVE_FUSE_UNITS", "1") != "0"


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

def _act_of(m):
    from . import cc
    code = cc._act_code(m)
    return code


def plan_sequential(mods: List[nn.Module]) -> Optional[List[LayerSpec]]:
    """EncoderV2.net / GeneratorV2.net style sequences: activations (LeakyReLU or Snake), cc.Conv1d, cc.ConvTranspose1d,
    Residual(DilatedUnit), AdaIN (identity in training).  Returns None if something is unsupported.
    Snake (v3): the producer writes its pre-activation as bf16, a channel-last Snake kernel turns it into the next conv's
    operand (and keeps the raw stream for the backward and for the unit's skip)."""
    from . import blocks, cc
    specs: List[LayerSpec] = []
    NONE = (ops.ACT_NONE, 0.0, None)
    pending = NONE
    last_idx = -1            # index of the layer producing the current stream (-1 = chain input)

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
        if isinstance(m, blocks.AdaptiveInstanceNormalization):
            if not m.training:
                return None
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
            pending = acts[1]
            if not add_conv(c1, res_src=src):
                return None
            if acts[0][0] == ops.ACT_LEAKY:
                specs[-1].res_opnd = c3_idx       # h_src = unleaky(operand of conv3): no fp32 stream needed
            else:
                specs[-1].res_raw = c3_idx        # Snake is not invertible: the raw bf16 input of conv3 is the skip
            continue
        return None
    if pending[0] != ops.ACT_NONE or not specs:
        return None
    if specs[0].pre_act != ops.ACT_NONE:
        # a chain's operands are activated by their PRODUCER's epilogue; the chain input has no producer, so a
        # sequence that starts with an activation (DilatedUnit.net on its own) is not run here
        return None
    specs[-1].is_output = True
    specs[-1].want_f32 = True
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


class _PreparedWeights:
    """Effective weight of one layer in every tap-major bf16 layout the kernels need.  `plan()` decides
    which layouts / tap orders are required; `prepare_layers()` produces them for a whole chain with ONE
    multi-tensor launch pair (row norms + re-layout): rave_weight_prep_tc_multi."""

    def __init__(self, spec: LayerSpec, need_dgrad: bool, need_fwd: bool):
        self.spec = spec
        K, s = spec.K, spec.stride
        if spec.kind == "conv":
            self.C0p, self.C1p = spec.Cout + spec.cout_pad, spec.Cin + spec.cin_pad
        else:
            self.C0p, self.C1p = spec.Cin + spec.cin_pad, spec.Cout + spec.cout_pad
        self.norm = None
        self.fwd = None           # conv: [K][Cout][Cin]
        self.fwd_fused = None     # convT: all output phases as one conv, wt [J][stride*Cout][Cin] (see
        self.dgrad = None         #   _fused_phase_taps); stride-1 conv: flipped taps [K][Cin][Cout]; convT: [K][Cin][Cout]
        self.dgrad_fused = None   # strided conv: all input phases as one conv, wt [J][stride*Cin][Cout]
        self.fused_J = self.fused_pad = 0
        self.need_dgrad = need_dgrad
        self.need_fwd = need_fwd
        self.raw = None           # (norm, outA, outB) as produced by the prep kernel (refresh_static_prep rewrites them)
        if spec.kind == "conv":
            self.tapsA = list(range(K)) if need_fwd else []
            if not need_dgrad:
                self.tapsB = []
            elif s == 1:
                self.tapsB = list(range(K - 1, -1, -1))
            else:
                self.tapsB, self.fused_J, self.fused_pad = _fused_phase_taps(K, s, spec.pad[0])
        else:
            self.tapsB, self.fused_J, self.fused_pad = _fused_phase_taps(K, s, spec.pad[0])
            self.tapsA = list(range(K)) if need_dgrad else []
        if len(self.tapsB) > 32:
            raise _lib.RaveB200Error(f"phase-fused layout of K={K}, stride={s} needs {len(self.tapsB)} > 32 slabs")

    def finalize(self, norm, outA, outB, parts: int = 1):
        """parts = 2: split-operand layouts, [all hi slabs | all lo slabs] along the leading axis."""
        spec = self.spec
        self.norm = norm
        if spec.kind == "conv":
            self.fwd = outA
            if self.need_dgrad:
                if spec.stride == 1:
                    self.dgrad = outB
                else:       # [J*stride][Cin_p][Cout_p] -> [J][stride*Cin_p][Cout_p]
                    self.dgrad_fused = outB.view(parts * self.fused_J, spec.stride * self.C1p, self.C0p)
        else:               # [J*stride][Cout_p][Cin_p] -> [J][stride*Cout_p][Cin_p]
            self.fwd_fused = outB.view(parts * self.fused_J, spec.stride * self.C1p, self.C0p)
            self.dgrad = outA
        return self


# ---- static prepared weights --------------------------------------------------------------------------------------
# A captured CUDA graph cannot use the version-keyed cache above (replays change parameters behind autograd's back), so
# every replay used to re-prepare every chain.  The discriminator's weights only change in D-steps (1 in 4): with
# `enable_static_prep(model.discriminator)` its prepared layouts live in persistent buffers that the chains read as they
# are, and that `refresh_static_prep` rewrites IN PLACE right after the discriminator's optimiser step (inside the
# D-step graph).  Whoever changes those parameters some other way (load_state_dict, an eager optimiser) must refresh.

def _static_holders(root: nn.Module):
    """Modules under `root` that own prepared weights, plus the parameter-view proxies of one-layer chains (the MRD's
    DiscConv2d plans its conv on a `_ParamView` holding permuted views of its parameters: descript_discriminator.py)."""
    for m in root.modules():
        yield m
        proxy = m.__dict__.get("_tc_proxy")
        if proxy is not None:
            yield proxy


def enable_static_prep(root: nn.Module) -> None:
    for m in root.modules():
        if hasattr(m, "weight_v") or (hasattr(m, "weight") and isinstance(getattr(m, "weight"), nn.Parameter)):
            m.__dict__.setdefault("_tc_static", {})
            if hasattr(m, "_tc_chain_spec"):          # proxy of a one-layer chain: created lazily, marked here or there
                m.__dict__["_tc_proxy_static"] = True
                proxy = m.__dict__.get("_tc_proxy")
                if proxy is not None:
                    proxy.__dict__.setdefault("_tc_static", {})


def disable_static_prep(root: nn.Module) -> None:
    for m in _static_holders(root):
        m.__dict__.pop("_tc_static", None)
        m.__dict__.pop("_tc_proxy_static", None)


@torch.no_grad()
def refresh_static_prep(root: nn.Module) -> int:
    """Recompute every static prepared layout under `root` into its existing buffers; returns how many."""
    items, into, extra = {False: [], True: []}, {False: [], True: []}, []
    for m in root.modules():
        if "_tc_proxy" in m.__dict__ and m.__dict__["_tc_proxy"].__dict__.get("_tc_static"):
            m._tc_refresh_proxy()        # the proxy's permuted parameter copies are stale once the parameters moved
    for m in _static_holders(root):
        st = m.__dict__.get("_tc_static")
        if not st:
            continue
        for key, pw in st.items():
            if key[0] == "c1":
                extra.append(pw)
                continue
            if pw.raw is None:        # norm-only entry of a Cin = 1 first layer: refreshed through its ("c1", "norm") record
                continue
            v, g, _ = _layer_params(pw.spec)
            x3 = bool(key[2])
            items[x3].append((v.detach(), g.detach() if g is not None else None, pw.tapsA, pw.tapsB, pw.C0p, pw.C1p))
            into[x3].append(pw.raw)
    for x3 in (False, True):
        if items[x3]:
            ops.weight_prep_tc_multi(items[x3], x3=x3, into=into[x3])
    for rec in extra:
        rec["refresh"]()
    return len(items[False]) + len(items[True]) + len(extra)


def prepare_layers(jobs, x3: bool = False):
    """jobs: list of (spec, v, g, need_dgrad, need_fwd).  Returns the list of _PreparedWeights, re-using the
    per-module cache (keyed on parameter versions; bypassed while a CUDA graph is being captured) and
    preparing all misses with one multi-tensor launch pair.  x3: split-operand ([hi slabs | lo slabs]) layouts."""
    out = [None] * len(jobs)
    todo = []
    for i, (spec, v, g, need_dgrad, need_fwd) in enumerate(jobs):
        capturing = v.is_cuda and torch.cuda.is_current_stream_capturing()
        static = spec.module.__dict__.get("_tc_static") if ACT_DTYPE == torch.bfloat16 else None
        if static is not None:
            hit = static.get((need_dgrad, need_fwd, x3))
            if hit is not None:
                out[i] = hit
                continue
        key = (v._version, g._version if g is not None else -1, need_dgrad, need_fwd, str(ACT_DTYPE), str(v.device),
               v.data_ptr(), _state["prep_epoch"], x3)
        slot = "_tc_prep_x3" if x3 else "_tc_prep"
        if not capturing and static is None:
            hit = spec.module.__dict__.get(slot)
            if hit is not None and hit[0] == key:
                out[i] = hit[1]
                continue
        todo.append((i, key, capturing, _PreparedWeights(spec, need_dgrad, need_fwd), v, g))
    work = [(i, key, cap, pw, v, g) for (i, key, cap, pw, v, g) in todo if pw.tapsA or pw.tapsB]
    if work:
        res = ops.weight_prep_tc_multi([(v, g, pw.tapsA, pw.tapsB, pw.C0p, pw.C1p) for (_, _, _, pw, v, g) in work],
                                       x3=x3)
        for (i, key, cap, pw, v, g), (norm, outA, outB) in zip(work, res):
            out[i] = pw.finalize(norm, outA, outB, 2 if x3 else 1)
            pw.raw = (norm, outA, outB)
            static = pw.spec.module.__dict__.get("_tc_static") if ACT_DTYPE == torch.bfloat16 else None
            if static is not None:
                if not cap:          # buffers of a capture belong to the graph's pool: only eager calls create a slot
                    static[(pw.need_dgrad, pw.need_fwd, x3)] = out[i]
            elif not cap:
                pw.spec.module.__dict__["_tc_prep_x3" if x3 else "_tc_prep"] = (key, out[i])
    for (i, key, cap, pw, v, g) in todo:
        if out[i] is None:            # nothing to re-layout (a c1 layer without dgrad): only the norm
            pw.norm = ops.weight_norm_raw(v, g)[1] if g is not None else None
            out[i] = pw
            static = pw.spec.module.__dict__.get("_tc_static") if ACT_DTYPE == torch.bfloat16 else None
            if static is not None and not cap and pw.norm is not None:
                norm_t, spec_ = pw.norm, pw.spec

                def _refresh(norm_t=norm_t, spec_=spec_):
                    v_, g_, _ = _layer_params(spec_)
                    norm_t.copy_(ops.weight_norm_raw(v_.detach(), g_.detach())[1])
                static[(pw.need_dgrad, pw.need_fwd, x3)] = pw
                static[("c1", "norm")] = {"refresh": _refresh}
    return out


# ----------------------------------------------------------------------------------------------
# the chain Function
# ----------------------------------------------------------------------------------------------

def _out_len(spec: LayerSpec, Lin: int) -> int:
    if spec.kind == "conv":
        return ops.conv_out_len(Lin, spec.K, spec.stride, spec.dil, spec.pad[0], spec.pad[1])
    return (Lin - 1) * spec.stride - 2 * spec.pad[0] + spec.K


class TcChainFn(torch.autograd.Function):
    """forward(x, specs, L0, fm, *flat_params).

    x   : [B, pitch, Cin(+pad)] operand stream (ACT_DTYPE), or -- when the first layer has Cin == 1 --
          a raw fp32 signal tensor [Bs, T] from which the chain rows are read in place: `src = (period, pool)`
          (L0 = positions per row; B = Bs*period rows; MPD fold / MSD pooling, ops.im2col_c1); no padding to 16
          channels, no bf16 rounding of the audio, no folded / pooled copy.
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
        c1 = x_in.dim() == 2
        period, pool = src if (c1 and src is not None) else (1, 1)
        B = x_in.shape[0] * period
        ctx.c1_src = (period, pool, tuple(x_in.shape))
        ctx.B = B
        # backward on the fake half only (see backward): always available to the fused feature-matching chains, and to
        # plain conv stacks (no residuals, no Snake: the Descript discriminator) whose caller asked for it
        plain = all(s.kind == "conv" and s.res_src is None and s.res_opnd is None and s.res_raw is None
                    and s.pre_act != ops.ACT_SNAKE for s in specs)
        ctx.fake_grad_only = bool(fake_grad_only) and (fm or (plain and B % 2 == 0 and not x3))
        if c1 and not (specs[0].kind == "conv" and specs[0].Cin == 1 and specs[0].dil == 1):
            raise _lib.RaveB200Error("raw fp32 rows are only accepted by a Cin = 1 first conv")
        dev = x_in.device
        a = x_in
        f32: Dict[int, torch.Tensor] = {}
        acts: List[torch.Tensor] = []                 # operand consumed by layer i
        prepared: List[_PreparedWeights] = []
        lens = [L0]
        outputs = []
        stats = torch.zeros(max(n - 1, 1), 2, dtype=torch.float32, device=dev) if fm else None
        prepared = prepare_layers([(s, flat[3 * i].detach(), flat[3 * i + 1].detach() if flat[3 * i + 1] is not None
                                    else None, need_dgrad and not (c1 and i == 0), not (c1 and i == 0))
                                   for i, s in enumerate(specs)], x3=x3)
        fused_second = False
        for i, s in enumerate(specs):
            if fused_second:           # the 1x1 conv of a unit the previous iteration ran as one fused launch
                fused_second = False
                continue
            v, g, bias = flat[3 * i], flat[3 * i + 1], flat[3 * i + 2]
            use_c1 = c1 and i == 0
            pw = prepared[i]
            Lin = lens[-1]
            Lout = _out_len(s, Lin)
            s1 = specs[i + 1] if i + 1 < n else None
            if (FUSE_UNITS and not x3 and not fm and not use_c1 and s1 is not None and ACT_DTYPE == torch.bfloat16
                    and s.kind == "conv" and s1.kind == "conv" and s.K == 3 and s1.K == 1 and s.stride == 1
                    and s1.stride == 1 and s.pre_act == ops.ACT_LEAKY and s1.pre_act == ops.ACT_LEAKY
                    and s1.res_opnd == i and s.res_src is None and s.res_opnd is None and bias is None
                    and flat[3 * i + 5] is None and s.Cin == s.Cout == s1.Cin == s1.Cout
                    and not (s.cin_pad or s.cout_pad or s1.cin_pad or s1.cout_pad) and Lout == Lin
                    and ops.dilated_unit_tc_supported(s.Cin, Lin)):
                # Residual(DilatedUnit) = act -> conv3(dil) -> act -> conv1x1 -> + x in ONE kernel: the intermediate
                # operand stays in shared memory (written to HBM only when a backward will need it)
                s2 = specs[i + 2] if i + 2 < n else None
                s_next = s2.stride if (s2 is not None and s2.kind == "conv") else 1
                pitch = (Lout + s_next - 1) // s_next * s_next
                if pitch == a.shape[1]:
                    want_f32 = s1.want_f32
                    out_f32 = torch.empty(B, pitch, s.Cout, dtype=torch.float32, device=dev) if want_f32 else None
                    out_act = torch.empty(B, pitch, s.Cout, dtype=ACT_DTYPE, device=dev) if s2 is not None else None
                    if pitch > Lout:
                        for t in (out_f32, out_act):
                            if t is not None:
                                t[:, Lout:].zero_()
                    a1, _, _ = ops.dilated_unit_tc(a, pw.fwd, prepared[i + 1].fwd, s.dil, s.pad[0], s.pre_slope,
                                                   s1.pre_slope, s2.pre_act if s2 is not None else ops.ACT_NONE,
                                                   s2.pre_slope if s2 is not None else 0.0, L=Lout, want_a1=need_dgrad,
                                                   out_f32=out_f32, out_act=out_act)
                    acts.append(a)
                    acts.append(a1)
                    lens.append(Lout)
                    lens.append(Lout)
                    if want_f32:
                        f32[i + 1] = out_f32
                    if s1.is_output:
                        outputs.append(out_f32)
                    a = out_act
                    fused_second = True
                    continue
            lens.append(Lout)
            nxt = specs[i + 1] if i + 1 < n else None
            want_act = nxt is not None
            act_code = nxt.pre_act if nxt is not None else ops.ACT_NONE
            act_slope = nxt.pre_slope if nxt is not None else 0.0
            snake_next = act_code == ops.ACT_SNAKE
            if snake_next:              # the epilogue writes h as bf16; ops.snake_cl_fwd makes the operand (below)
                act_code = ops.ACT_NONE
            want_f32 = s.want_f32 and not (fm and nxt is not None)
            # rows allocated per batch: the consumer's 4-D tensor map needs a multiple of its stride
            s_next = nxt.stride if (nxt is not None and nxt.kind == "conv") else 1
            pitch = (Lout + s_next - 1) // s_next * s_next
            cout_p = s.Cout + s.cout_pad
            bias_p = bias
            if bias is not None and s.cout_pad:
                bias_p = nn.functional.pad(bias.detach(), (0, s.cout_pad))
            res = res_act = res_b16 = None
            res_slope = 0.2
            if s.res_opnd is not None:
                res_act, res_slope = acts[s.res_opnd], specs[s.res_opnd].pre_slope
            elif s.res_raw is not None:
                res_b16 = hraw[s.res_raw]
            elif s.res_src is not None:
                res = f32[s.res_src]
            out_f32 = torch.empty(B, pitch, cout_p, dtype=torch.float32, device=dev) if want_f32 else None
            out_act = torch.empty(B, pitch, AW * cout_p, dtype=ACT_DTYPE, device=dev) if want_act else None
            if pitch > Lout:
                for t in (out_f32, out_act):
                    if t is not None:
                        t[:, Lout:].zero_()
            acts.append(a)
            if use_c1:
                # Cin = 1: the K taps become the 16 "channels" of a tiny im2col X[r][l][k].  Four consecutive
                # positions are then read as ONE 64-channel row (X viewed as [R][L/4][64], 128-byte TMA rows
                # instead of 32-byte ones) against the block-diagonal weight kron(I4, w): the output row holds
                # the 4 x Cout results of those positions, i.e. the same bytes as out[r][4*l4 + p][co].
                G = C1_GROUP if (pitch % C1_GROUP == 0) else 1
                Xp = (Lout + G - 1) // G * G
                X = ops.im2col_c1(a, Lin, Lout, Xp, s.K, s.stride, s.pad[0], period, pool)
                ctx.c1_X = X
                ctx.c1_group = G

                def c1_weights(s=s, G=G, cout_p=cout_p):
                    v_, g_, b_ = _layer_params(s)
                    w_eff = ops.weight_norm_raw(v_.detach(), g_.detach())[0] if g_ is not None else v_.detach()
                    w_ck = nn.functional.pad(w_eff.reshape(s.Cout, s.K), (0, 16 - s.K, 0, s.cout_pad))   # [Cout_p, 16]
                    if G > 1:
                        eye = torch.eye(G, dtype=w_ck.dtype, device=w_ck.device)
                        w_blk = (eye[:, None, :, None] * w_ck[None, :, None, :]).reshape(G * cout_p, G * 16)
                    else:
                        w_blk = w_ck
                    bp = b_
                    if b_ is not None and s.cout_pad:
                        bp = nn.functional.pad(b_.detach(), (0, s.cout_pad))
                    bias_g_ = bp.detach().repeat(G) if (bp is not None and G > 1) else (bp.detach() if bp is not None
                                                                                         else None)
                    return (w_blk.to(ACT_DTYPE).unsqueeze(0).contiguous(),                     # [1][G*Cout_p][G*16]
                            w_blk.t().contiguous().to(ACT_DTYPE).unsqueeze(0), bias_g_)        # [1][G*16][G*Cout_p]

                static = s.module.__dict__.get("_tc_static") if ACT_DTYPE == torch.bfloat16 else None
                rec = static.get(("c1", G, cout_p)) if static is not None else None
                if rec is None:
                    w_fwd, w_dg, bias_g = c1_weights()
                    if static is not None and not torch.cuda.is_current_stream_capturing():
                        def _refresh(w_fwd=w_fwd, w_dg=w_dg, bias_g=bias_g, fn=c1_weights):
                            a_, b_, c_ = fn()
                            w_fwd.copy_(a_)
                            w_dg.copy_(b_)
                            if bias_g is not None:
                                bias_g.copy_(c_)
                        static[("c1", G, cout_p)] = {"t": (w_fwd, w_dg, bias_g), "refresh": _refresh}
                else:
                    w_fwd, w_dg, bias_g = rec["t"]
                ctx.c1_wt_dgrad = w_dg
                ops.conv1d_tc(X.view(B, Xp // G, G * 16), w_fwd, bias_g,
                              None, 1, 1, (0, 0), act_code, act_slope, want_f32=False, want_act=False,
                              out_f32=out_f32.view(B, pitch // G, G * cout_p) if out_f32 is not None else None,
                              out_act=out_act.view(B, pitch // G, G * cout_p) if out_act is not None else None,
                              Lout=Xp // G, Lin=Xp // G, out_rows=pitch // G)
                if Xp > Lout:            # positions Lout .. Xp-1 of the last group saw zero taps but got the bias
                    for t in (out_f32, out_act):
                        if t is not None:
                            t[:, Lout:Xp].zero_()
            elif s.kind == "conv":
                ops.conv1d_tc(a, pw.fwd, bias_p, res, s.stride, s.dil, s.pad, act_code, act_slope,
                              want_f32=False, want_act=False, out_f32=out_f32, out_act=out_act, Lout=Lout,
                              Lin=Lin, out_rows=pitch, res_act=res_act, res_slope=res_slope, x3=x3, res_bf16=res_b16)
            else:
                # transposed conv: the `stride` output phases side by side in one stride-1 conv (output row q =
                # positions q*stride .. q*stride + stride-1: the same bytes as the [B][pitch][Cout] tensor)
                st = s.stride
                if pitch % st:
                    raise _lib.RaveB200Error("transposed conv: the output pitch must be a multiple of the stride")
                rows_q = pitch // st
                bias_f = bias_p.detach().repeat(st) if bias_p is not None else None
                ops.conv1d_tc(a, pw.fwd_fused, bias_f, None, 1, 1, (pw.fused_pad, 0), act_code, act_slope,
                              want_f32=False, want_act=False,
                              out_f32=out_f32.view(B, rows_q, st * cout_p) if out_f32 is not None else None,
                              out_act=out_act.view(B, rows_q, st * AW * cout_p) if out_act is not None else None,
                              out_rows=rows_q, Lout=rows_q, Lin=Lin, x3=x3, act_cs=cout_p if x3 else 0)
                if pitch > Lout:         # positions beyond the true length were computed too: back to zero
                    for t in (out_f32, out_act):
                        if t is not None:
                            t[:, Lout:].zero_()
            if snake_next:
                hraw[i + 1] = out_act
                out_act = ops.snake_cl_fwd(out_act, flat[alpha_idx[i + 1]])
            if fm and nxt is not None:
                if act_code != ops.ACT_LEAKY or s.cout_pad:
                    raise _lib.RaveB200Error("feature-matching mode needs LeakyReLU between the layers")
                ops.fm_stats(out_act, stats[i], Lout, act_slope)
            if want_f32:
                f32[i] = out_f32
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
        ctx.c1 = c1
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
        gx_full = None
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
            use_c1 = ctx.c1 and i == 0
            a_full = ctx.acts[i]
            a_in = a_full if use_c1 else half(a_full)
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
                if use_c1:
                    G = ctx.c1_group
                    X = ctx.c1_X
                    if G > 1 and g.shape[1] % G == 0 and X.shape[1] % G == 0:
                        # same G-positions-per-row view as the forward: 64-channel rows for the TMA loads; the wanted
                        # [Cout][16] gradient is the sum of the G diagonal blocks of the [G*Cout][G*16] result
                        dbw = torch.zeros(G * cout_p, dtype=torch.float32, device=g.device) if db is not None else None
                        d = ops.conv1d_tc_wgrad(g.view(B, g.shape[1] // G, G * cout_p), X.view(B, X.shape[1] // G, G * 16),
                                                1, 1, 1, 0, Lp=(Lout + G - 1) // G, Lq=(Lout + G - 1) // G, dbias=dbw)
                        blk = d.sum(0)[0].view(G, cout_p, G, 16)
                        dw_full = torch.diagonal(blk, dim1=0, dim2=2).sum(-1)                  # [Cout_p][16]
                        if db is not None:
                            db.copy_(dbw.view(G, cout_p).sum(0))
                    else:
                        dw_full = ops.conv1d_tc_wgrad(g, X, 1, 1, 1, 0, Lp=Lout, Lq=Lout, dbias=db).sum(0)[0]
                    dw_ck = dw_full[:s.Cout, :s.K]                                             # [Cout][K]
                    dwt = dw_ck.t().reshape(1, s.K, s.Cout, 1).contiguous()                    # [1][K][C0][C1=1]
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
                if s.pre_act != ops.ACT_LEAKY or use_c1:
                    raise _lib.RaveB200Error("fused feature-matching gradient needs a LeakyReLU operand")
            if e is not None:
                add = e if add is None else (add + e)
            dact = a_in if s.pre_act == ops.ACT_LEAKY else None
            snake_here = s.pre_act == ops.ACT_SNAKE
            add_conv = None if snake_here else add       # Snake: the skip / external gradient joins after dSnake
            fm_partner = a_full[:Bh] if (fo and fm_d is not None) else None
            in_pitch = a_in.shape[1]
            if use_c1:                  # P[r][l][k] = <g[r][l][:], w[:][k]> on the tensor cores, then a gather
                G = ctx.c1_group
                gpitch = g.shape[1]
                if G > 1 and gpitch % G == 0:
                    # same 4-positions-per-row view as the forward (slack rows of g are zero)
                    P, _ = ops.conv1d_tc(g.view(B, gpitch // G, G * cout_p), ctx.c1_wt_dgrad, None, None, 1, 1, (0, 0),
                                         ops.ACT_NONE, 0.0, want_f32=True, want_act=False, Lout=gpitch // G,
                                         Lin=gpitch // G)
                    P = P.view(B, gpitch, 16)
                else:
                    wt_d = ctx.c1_wt_dgrad if G == 1 else ctx.c1_wt_dgrad[:, :16, :cout_p].contiguous()
                    P, _ = ops.conv1d_tc(g, wt_d, None, None, 1, 1, (0, 0), ops.ACT_NONE, 0.0, want_f32=True,
                                         want_act=False, Lout=Lout, Lin=Lout)
                period, pool, src_shape = ctx.c1_src
                gx = ops.gather_c1(P, src_shape, Lin, Lout, s.K, s.stride, s.pad[0], period, pool,
                                   batch0=src_shape[0] // 2 if fo else 0)
                break
            if fo and i == 0:
                # fake-rows-only backward: the chain's input gradient is [zeros; gx_fake] -- the last dgrad writes its
                # rows straight into the second half of the full buffer (no zeros + copy pass afterwards)
                gx_full = torch.empty(ctx.B, in_pitch, cin_p, dtype=ACT_DTYPE, device=g.device)
                gx_full[:Bh].zero_()
                gp = gx_full[Bh:]
            else:
                gp = torch.empty(B, in_pitch, cin_p, dtype=ACT_DTYPE, device=g.device)
            if in_pitch > Lin:
                gp[:, Lin:].zero_()
            if s.kind == "conv":
                if s.stride == 1:
                    padp = (s.K - 1) * s.dil - s.pad[0]
                    ops.conv1d_tc(g, pw.dgrad, None, None, 1, s.dil, (padp, 0), ops.ACT_NONE, s.pre_slope,
                                  want_f32=False, want_act=False, out_act=gp, Lout=Lin, Lin=Lout,
                                  out_rows=in_pitch, res_bf16=add_conv, dact_src=dact, fm_d=fm_d,
                                  fm_partner=fm_partner)
                else:
                    # strided conv: the `stride` input phases side by side in one stride-1 conv over g (row q of the
                    # result = input positions q*stride .. +stride-1); g rows are fetched once, not once per phase
                    st = s.stride
                    if in_pitch % st:
                        raise _lib.RaveB200Error("strided conv dgrad: the operand pitch must be a multiple of the stride")
                    rows_q = in_pitch // st
                    wide = st * cin_p

                    def v4(t):
                        return t.view(B, rows_q, wide) if t is not None else None
                    ops.conv1d_tc(g, pw.dgrad_fused, None, None, 1, 1, (pw.fused_pad, 0), ops.ACT_NONE, s.pre_slope,
                                  want_f32=False, want_act=False, out_act=v4(gp), out_rows=rows_q, Lout=rows_q,
                                  Lin=Lout, res_bf16=v4(add_conv), dact_src=v4(dact), fm_d=fm_d,
                                  fm_partner=v4(fm_partner))
                    if in_pitch > Lin:
                        gp[:, Lin:].zero_()
            else:
                ops.conv1d_tc(g, pw.dgrad, None, None, s.stride, 1, (s.pad[0], 0), ops.ACT_NONE, s.pre_slope,
                              want_f32=False, want_act=False, out_act=gp, Lout=Lin, Lin=Lout, out_rows=in_pitch,
                              res_bf16=add_conv, dact_src=dact, fm_d=fm_d, fm_partner=fm_partner)
            if snake_here:
                al = flat[ctx.alpha_idx[i]]
                gp, dal = ops.snake_cl_bwd(gp, ctx.hraw[i], al, add, want_dalpha=bool(al.requires_grad))
                if dal is not None:
                    grads[ctx.alpha_idx[i]] = dal.reshape(al.shape)
            g_cur = gp
            if i == 0:
                gx = gp
        if wn_jobs:
            res = ops.weight_norm_bwd_multi([job[1:] for job in wn_jobs])
            for job, (dv, dg) in zip(wn_jobs, res):
                i = job[0]
                grads[3 * i], grads[3 * i + 1] = dv, dg
        if fo and gx is not None and not ctx.c1 and gx.shape[0] == Bh:
            if gx_full is not None and gx.data_ptr() == gx_full[Bh:].data_ptr() and gx.shape == gx_full[Bh:].shape:
                gx = gx_full                 # the real rows' gradient is identically unused: zeros
            else:
                full = torch.zeros((ctx.B,) + tuple(gx.shape[1:]), dtype=gx.dtype, device=gx.device)
                full[Bh:] = gx
                gx = full
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
    [B, pitch] for a Cin = 1 first layer.  Returns one fp32 channel-last tensor [B, pitch_i, Cout_i(+pad)]
    per output layer (slice [:, :L_i, :Cout_i]); with fm=True: (stats [n-1, 2], score_stats [3, 2], last layer
    output)."""
    flat = []
    for s in specs:
        v, g, b = _layer_params(s)
        flat += [v, g, b]
    flat += [s.pre_mod.alpha for s in specs if s.pre_act == ops.ACT_SNAKE]      # after the 3n weight entries
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

"""torch.autograd.Function wrappers around the C ABI (include/rave_b200.h).

PyTorch is plumbing here: it owns the device memory, the stream and the autograd tape; every
arithmetic operation of the hot path is one of the library's sm_90a kernels.  There is no
fallback implementation: host tensors or a missing library raise (`_lib.RaveB200Error`).
"""
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import call, ptr, stream_ptr

ACT_NONE, ACT_LEAKY, ACT_SNAKE = 0, 1, 2


def _f32c(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    if t is None:
        return None
    if t.dtype != torch.float32:
        raise _lib.RaveB200Error(f"expected float32 tensor, got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


def conv_out_len(Lin: int, K: int, stride: int, dil: int, pad_l: int, pad_r: int) -> int:
    return (Lin + pad_l + pad_r - dil * (K - 1) - 1) // stride + 1


# ----------------------------------------------------------------------------------------------
# raw launches (no autograd)
# ----------------------------------------------------------------------------------------------

def _gather(src, w, bias, res, out, K, stride, dil, pad_l, ws_m, ws_c, act, slope, alpha,
            post_act=0, post_slope=0.0, post_x=None, post_alpha=None):
    B, Cs, Ls = src.shape
    _, Cm, Lo = out.shape
    call("rave_conv1d_gather_f32", ptr(src), ptr(w), ptr(bias), ptr(res), ptr(out), B, Cs, Ls, Cm, Lo,
         K, stride, dil, pad_l, ws_m, ws_c, act, float(slope), ptr(alpha), post_act, float(post_slope),
         ptr(post_x), ptr(post_alpha), stream_ptr())


def _scatter(src, w, bias, res, out, K, stride, dil, pad_l, ws_m, ws_c, act, slope, alpha,
             post_act=0, post_slope=0.0, post_x=None, post_alpha=None):
    B, Cs, Ls = src.shape
    _, Cm, Lo = out.shape
    call("rave_conv1d_scatter_f32", ptr(src), ptr(w), ptr(bias), ptr(res), ptr(out), B, Cs, Ls, Cm, Lo,
         K, stride, dil, pad_l, ws_m, ws_c, act, float(slope), ptr(alpha), post_act, float(post_slope),
         ptr(post_x), ptr(post_alpha), stream_ptr())


def _wgrad(P, Q, dw, K, stride, dil, pad_l, os_a, os_c, act_p, act_q, slope, alpha):
    B, Ca, Lp = P.shape
    _, Cc, Lq = Q.shape
    lib = _lib.load()
    nbytes = lib.rave_conv1d_wgrad_workspace_bytes(B, Ca, Cc, Lp, K)
    ws = torch.empty(nbytes // 4, dtype=torch.float32, device=P.device)
    call("rave_conv1d_wgrad_f32", ptr(P), ptr(Q), ptr(dw), B, Ca, Lp, Cc, Lq, K, stride, dil, pad_l,
         os_a, os_c, act_p, act_q, float(slope), ptr(alpha), ptr(ws), stream_ptr())


def _act_grad_input(g, x, act, slope, alpha):
    """dx = g * act'(x) (+ dalpha for Snake)."""
    dx = torch.empty_like(x)
    dalpha = torch.empty_like(alpha) if act == ACT_SNAKE else None
    B, C, L = x.shape
    call("rave_act_bwd", ptr(g), ptr(x), ptr(dx), ptr(dalpha), B, C, L, act, float(slope), ptr(alpha),
         stream_ptr())
    return dx, dalpha


# ----------------------------------------------------------------------------------------------
# conv1d: y = bias + res + conv(act(x))      (cc.Conv1d.forward preceded by its activation)
# ----------------------------------------------------------------------------------------------

class Conv1dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, bias, res, alpha, stride, dil, pad_l, pad_r, act, slope):
        x, w, bias, res, alpha = _f32c(x), _f32c(w), _f32c(bias), _f32c(res), _f32c(alpha)
        B, Cin, Lin = x.shape
        Cout, Cin_w, K = w.shape
        if Cin_w != Cin:
            raise _lib.RaveB200Error(f"conv1d: weight expects {Cin_w} input channels, got {Cin}")
        Lout = conv_out_len(Lin, K, stride, dil, pad_l, pad_r)
        if Lout <= 0:
            raise _lib.RaveB200Error("conv1d: empty output")
        y = torch.empty(B, Cout, Lout, dtype=torch.float32, device=x.device)
        if res is not None and res.shape != y.shape:
            raise _lib.RaveB200Error("conv1d: residual shape mismatch")
        _gather(x, w, bias, res, y, K, stride, dil, pad_l, Cin * K, K, act, slope, alpha)
        ctx.save_for_backward(x, w, alpha)
        ctx.cfg = (stride, dil, pad_l, act, slope, bias is not None, res is not None)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, alpha = ctx.saved_tensors
        stride, dil, pad_l, act, slope, has_bias, has_res = ctx.cfg
        dy = _f32c(dy)
        B, Cin, Lin = x.shape
        Cout, _, K = w.shape
        dx = dw = dbias = dres = dalpha = None
        if ctx.needs_input_grad[0] or (act == ACT_SNAKE and ctx.needs_input_grad[4]):
            g = torch.empty_like(x)
            if act == ACT_SNAKE:
                _scatter(dy, w, None, None, g, K, stride, dil, pad_l, K, Cin * K, 0, 0.0, None)
                dx, dalpha = _act_grad_input(g, x, act, slope, alpha)
            else:
                _scatter(dy, w, None, None, g, K, stride, dil, pad_l, K, Cin * K, 0, 0.0, None,
                         post_act=act, post_slope=slope, post_x=x if act else None)
                dx = g
        if ctx.needs_input_grad[1]:
            dw = torch.empty_like(w)
            _wgrad(dy, x, dw, K, stride, dil, pad_l, Cin * K, K, 0, act, slope, alpha)
        if has_bias and ctx.needs_input_grad[2]:
            dbias = dy.sum((0, 2))
        if has_res and ctx.needs_input_grad[3]:
            dres = dy
        return dx, dw, dbias, dres, dalpha, None, None, None, None, None, None


def conv1d(x, w, bias=None, res=None, stride=1, dilation=1, pad=(0, 0), act=ACT_NONE, slope=0.2,
           alpha=None):
    return Conv1dFn.apply(x, w, bias, res, alpha, stride, dilation, pad[0], pad[1], act, slope)


# ----------------------------------------------------------------------------------------------
# conv_transpose1d: y = bias + convT(act(x)),  w: [Cin, Cout, K]   (blocks.py:650-657)
# ----------------------------------------------------------------------------------------------

class ConvTranspose1dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, bias, alpha, stride, padding, act, slope):
        x, w, bias, alpha = _f32c(x), _f32c(w), _f32c(bias), _f32c(alpha)
        B, Cin, Lin = x.shape
        Cin_w, Cout, K = w.shape
        if Cin_w != Cin:
            raise _lib.RaveB200Error(f"conv_transpose1d: weight expects {Cin_w} input channels, got {Cin}")
        Lout = (Lin - 1) * stride - 2 * padding + K
        y = torch.empty(B, Cout, Lout, dtype=torch.float32, device=x.device)
        _scatter(x, w, bias, None, y, K, stride, 1, padding, K, Cout * K, act, slope, alpha)
        ctx.save_for_backward(x, w, alpha)
        ctx.cfg = (stride, padding, act, slope, bias is not None)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, alpha = ctx.saved_tensors
        stride, padding, act, slope, has_bias = ctx.cfg
        dy = _f32c(dy)
        Cin, Cout, K = w.shape
        dx = dw = dbias = dalpha = None
        if ctx.needs_input_grad[0] or (act == ACT_SNAKE and ctx.needs_input_grad[3]):
            g = torch.empty_like(x)
            if act == ACT_SNAKE:
                _gather(dy, w, None, None, g, K, stride, 1, padding, Cout * K, K, 0, 0.0, None)
                dx, dalpha = _act_grad_input(g, x, act, slope, alpha)
            else:
                _gather(dy, w, None, None, g, K, stride, 1, padding, Cout * K, K, 0, 0.0, None,
                        post_act=act, post_slope=slope, post_x=x if act else None)
                dx = g
        if ctx.needs_input_grad[1]:
            dw = torch.empty_like(w)
            _wgrad(x, dy, dw, K, stride, 1, padding, Cout * K, K, act, 0, slope, alpha)
        if has_bias and ctx.needs_input_grad[2]:
            dbias = dy.sum((0, 2))
        return dx, dw, dbias, dalpha, None, None, None, None


def conv_transpose1d(x, w, bias=None, stride=1, padding=0, act=ACT_NONE, slope=0.2, alpha=None):
    return ConvTranspose1dFn.apply(x, w, bias, alpha, stride, padding, act, slope)


# ----------------------------------------------------------------------------------------------
# weight norm (blocks.normalization -> torch.nn.utils.weight_norm, rave/blocks.py:15-22)
# ----------------------------------------------------------------------------------------------

class WeightNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, v, g):
        v, g = _f32c(v), _f32c(g)
        C0 = v.shape[0]
        R = v.numel() // C0
        w = torch.empty_like(v)
        norm = torch.empty(C0, dtype=torch.float32, device=v.device)
        call("rave_weight_norm_fwd", ptr(v), ptr(g), ptr(w), ptr(norm), C0, R, stream_ptr())
        ctx.save_for_backward(v, g, norm)
        return w

    @staticmethod
    def backward(ctx, dw):
        v, g, norm = ctx.saved_tensors
        dw = _f32c(dw)
        C0 = v.shape[0]
        R = v.numel() // C0
        dv = torch.empty_like(v)
        dg = torch.empty_like(g)
        call("rave_weight_norm_bwd", ptr(dw), ptr(v), ptr(g), ptr(norm), ptr(dv), ptr(dg), C0, R,
             stream_ptr())
        return dv, dg


def weight_norm(v, g):
    return WeightNormFn.apply(v, g)


# ----------------------------------------------------------------------------------------------
# stand-alone activation (LeakyReLU / Snake) and generator tail
# ----------------------------------------------------------------------------------------------

class ActFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, alpha, act, slope):
        x, alpha = _f32c(x), _f32c(alpha)
        B, C, L = x.shape
        y = torch.empty_like(x)
        call("rave_act_fwd", ptr(x), ptr(y), B, C, L, act, float(slope), ptr(alpha), stream_ptr())
        ctx.save_for_backward(x, alpha)
        ctx.cfg = (act, slope)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, alpha = ctx.saved_tensors
        act, slope = ctx.cfg
        dx, dalpha = _act_grad_input(_f32c(dy), x, act, slope, alpha)
        return dx, dalpha, None, None


def activation(x, act, slope=0.2, alpha=None):
    if act == ACT_NONE:
        return x
    shape = x.shape
    if x.dim() != 3:
        x = x.reshape(shape[0], shape[1], -1)
    return ActFn.apply(x, alpha, act, slope).reshape(shape)


class AmTanhFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        x = _f32c(x)
        B, C2, L = x.shape
        C = C2 // 2
        y = torch.empty(B, C, L, dtype=torch.float32, device=x.device)
        call("rave_am_tanh_fwd", ptr(x), ptr(y), B, C, L, stream_ptr())
        ctx.save_for_backward(x)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        B, C2, L = x.shape
        dx = torch.empty_like(x)
        call("rave_am_tanh_bwd", ptr(_f32c(dy)), ptr(x), ptr(dx), B, C2 // 2, L, stream_ptr())
        return dx


class ReparamFn(torch.autograd.Function):
    """VariationalEncoder.reparametrize (rave/blocks.py:725-737) as one library pass: (zs, kl_sum) from z = (mean | scale)
    and eps; kl_sum = sum over every element of mean^2 + var - log var - 1.  The backward (phase 1 only: phase 2 detaches
    z) is the closed form on the saved inputs."""

    @staticmethod
    def forward(ctx, z, eps):
        z, eps = _f32c(z), _f32c(eps)
        B, C2, L = z.shape
        C = C2 // 2
        zs = torch.empty(B, C, L, dtype=torch.float32, device=z.device)
        kl_sum = torch.zeros((), dtype=torch.float32, device=z.device)
        call("rave_reparam_fwd", ptr(z), ptr(eps), ptr(zs), ptr(kl_sum), B, C, L, stream_ptr())
        ctx.save_for_backward(z, eps)
        return zs, kl_sum

    @staticmethod
    def backward(ctx, g_zs, g_kl):
        z, eps = ctx.saved_tensors
        mean, scale = z.chunk(2, 1)
        std = torch.nn.functional.softplus(scale) + 1e-4
        d_mean = torch.zeros_like(mean) if g_zs is None else g_zs.clone()
        d_std = torch.zeros_like(mean) if g_zs is None else g_zs * eps
        if g_kl is not None:
            d_mean = d_mean + g_kl * 2.0 * mean
            d_std = d_std + g_kl * (2.0 * std - 2.0 / std)
        return torch.cat([d_mean, d_std * torch.sigmoid(scale)], 1), None


def reparam(z, eps):
    return ReparamFn.apply(z, eps)


class MMDFn(torch.autograd.Function):
    """WasserteinEncoder's regulariser (rave/blocks.py:761-774) as one library pass: the MMD between the rows
    x_i = z[b, :, t] of z [B, D, L] and the prior sample [B·L, D], kernel exp(-|a - b|² / D²).  Returns (mmd, the three
    kernel means (xx, yy, xy)); only the MMD is differentiable, and only with respect to z.  The backward recomputes the
    kernel and reads the upstream gradient from device memory."""

    @staticmethod
    def forward(ctx, z, prior):
        z, prior = _f32c(z), _f32c(prior)
        B, D, L = z.shape
        if tuple(prior.shape) != (B * L, D):
            raise _lib.RaveB200Error(f"mmd: prior {tuple(prior.shape)} for z {tuple(z.shape)}, want {(B * L, D)}")
        means = torch.empty(3, dtype=torch.float32, device=z.device)
        mmd = torch.empty((), dtype=torch.float32, device=z.device)
        call("rave_mmd_fwd", ptr(z), ptr(prior), ptr(means), ptr(mmd), B, D, L, stream_ptr())
        ctx.save_for_backward(z, prior)
        ctx.mark_non_differentiable(means)
        return mmd, means

    @staticmethod
    def backward(ctx, g_mmd, g_means):
        z, prior = ctx.saved_tensors
        B, D, L = z.shape
        dz = torch.empty_like(z)
        call("rave_mmd_bwd", ptr(z), ptr(prior), ptr(_f32c(g_mmd)), ptr(dz), B, D, L, stream_ptr())
        return dz, None


def mmd(z, prior):
    return MMDFn.apply(z, prior)


class SphereNormFn(torch.autograd.Function):
    """SphericalEncoder.reparametrize (rave/blocks.py:839-842): z / |z|₂ over the channels of each (b, t) column."""

    @staticmethod
    def forward(ctx, z):
        z = _f32c(z)
        B, C, L = z.shape
        out = torch.empty_like(z)
        norm = torch.empty(B, L, dtype=torch.float32, device=z.device)
        call("rave_sphere_norm_fwd", ptr(z), ptr(out), ptr(norm), B, C, L, stream_ptr())
        ctx.save_for_backward(out, norm)
        return out

    @staticmethod
    def backward(ctx, g):
        out, norm = ctx.saved_tensors
        B, C, L = out.shape
        dz = torch.empty_like(out)
        call("rave_sphere_norm_bwd", ptr(_f32c(g)), ptr(out), ptr(norm), ptr(dz), B, C, L, stream_ptr())
        return dz


def sphere_norm(z):
    return SphereNormFn.apply(z)


def latent_moments(z, D, state):
    """Accumulates the rows z[b, :D, t] of z [B, C, L] (fp32, C >= D) into state = [n | mean[D] | M2[D*D]] (fp64, in
    place) with rave_latent_moments; the only allocation is the kernel's workspace."""
    B, C, L = z.shape
    if not (z.dtype == torch.float32 and z.stride(2) == 1 and z.stride(1) == L and (B == 1 or z.stride(0) >= C * L)
            and z.stride(0) % L == 0):
        z = _f32c(z)
    elif B > 1:
        C = z.stride(0) // L            # a channel slice of a [B, C', L] buffer (the mean half of the encoder output)
    if state.dtype != torch.float64 or state.numel() != 1 + D + D * D or not state.is_contiguous():
        raise _lib.RaveB200Error(f"latent_moments: state must be a contiguous fp64 tensor of 1 + D + D^2 = "
                                 f"{1 + D + D * D} elements")
    nbytes = int(_lib.load().rave_latent_moments_workspace_bytes(B, L, D))
    work = torch.empty(max(nbytes, 8) // 8, dtype=torch.float64, device=z.device)
    if not z.is_cuda:
        raise _lib.RaveB200Error("rave_b200 ops need CUDA tensors (there is no CPU path)")
    call("rave_latent_moments", z.data_ptr(), B, C, L, D, ptr(state), ptr(work), stream_ptr())
    return state


def am_tanh(x):
    """tanh(x[:, :C] * sigmoid(x[:, C:])) -- GeneratorV2 tail, rave/blocks.py:704-711."""
    return AmTanhFn.apply(x)


# ----------------------------------------------------------------------------------------------
# PQMF
# ----------------------------------------------------------------------------------------------

def _pqmf_analysis_raw(x, taps, Lout, pad_l, flip):
    """taps: dense table [16][ntaps], or the factorised form (Ct [32][16], Qt [17][32]) of pqmf._factorise."""
    B, T = x.shape
    y = torch.empty(B, 16, Lout, dtype=torch.float32, device=x.device)
    if isinstance(taps, tuple):
        call("rave_pqmf_analysis_fast", ptr(x), ptr(taps[0]), ptr(taps[1]), ptr(y), B, T, Lout, pad_l, int(flip),
             stream_ptr())
        return y
    call("rave_pqmf_analysis_fwd", ptr(x), ptr(taps), ptr(y), B, T, Lout, taps.shape[1], pad_l,
         int(flip), stream_ptr())
    return y


def _pqmf_synthesis_raw(x, w, pad_l, scale, flip):
    """w: dense weights [16][16][K], or the factorised form (Cc [16][32], Qt [17][32])."""
    B, M, L = x.shape
    out = torch.empty(B, 16 * L, dtype=torch.float32, device=x.device)
    if isinstance(w, tuple):
        call("rave_pqmf_synthesis_fast", ptr(x), ptr(w[0]), ptr(w[1]), ptr(out), B, L, pad_l, float(scale), int(flip),
             stream_ptr())
        return out
    call("rave_pqmf_synthesis_fwd", ptr(x), ptr(w), ptr(out), B, L, w.shape[2], pad_l, float(scale),
         int(flip), stream_ptr())
    return out


class PqmfAnalysisFn(torch.autograd.Function):
    """x[B,1,T] -> y[B,16,T/16]; `taps_bwd` = the same filter re-indexed as synthesis weights."""

    @staticmethod
    def forward(ctx, x, taps, taps_bwd, pad_l, pad_r, bwd_pad):
        x = _f32c(x)
        B, C, T = x.shape
        if C != 1:
            raise _lib.RaveB200Error("pqmf analysis expects [B,1,T]")
        ntaps = taps.shape[1] if torch.is_tensor(taps) else taps[2]
        Lout = (T + pad_l + pad_r - ntaps) // 16 + 1
        y = _pqmf_analysis_raw(x.view(B, T), taps, Lout, pad_l, True)
        ctx.taps_bwd = taps_bwd          # constant filter tables (never differentiated)
        ctx.cfg = (T, bwd_pad)
        return y

    @staticmethod
    def backward(ctx, dy):
        taps_bwd = ctx.taps_bwd
        T, bwd_pad = ctx.cfg
        dy = _f32c(dy)
        if dy.shape[2] * 16 != T:
            raise _lib.RaveB200Error("pqmf analysis backward needs T == 16 * Lout")
        dx = _pqmf_synthesis_raw(dy, taps_bwd, bwd_pad, 1.0, True)
        return dx.view(dy.shape[0], 1, T), None, None, None, None, None


class PqmfSynthesisFn(torch.autograd.Function):
    """y[B,16,L] -> x[B,1,16 L]; `w_bwd` = the same filter re-indexed as analysis taps."""

    @staticmethod
    def forward(ctx, y, w, w_bwd, pad_l, bwd_pad):
        y = _f32c(y)
        B, M, L = y.shape
        if M != 16:
            raise _lib.RaveB200Error("pqmf synthesis expects 16 bands")
        out = _pqmf_synthesis_raw(y, w, pad_l, 16.0, True)
        ctx.w_bwd = w_bwd
        ctx.cfg = (L, bwd_pad)
        return out.view(B, 1, 16 * L)

    @staticmethod
    def backward(ctx, dout):
        w_bwd = ctx.w_bwd
        L, bwd_pad = ctx.cfg
        dout = _f32c(dout)
        B = dout.shape[0]
        dy = _pqmf_analysis_raw(dout.view(B, 16 * L), w_bwd, L, bwd_pad, True)
        return dy, None, None, None, None


def act_to_bf16(x, act=ACT_NONE, slope=0.2, alpha=None):
    x = _f32c(x)
    B, C, L = x.shape
    y = torch.empty(B, C, L, dtype=torch.bfloat16, device=x.device)
    call("rave_act_to_bf16", ptr(x), ptr(y), B, C, L, act, float(slope), ptr(alpha), stream_ptr())
    return y


def weight_to_tapmajor_bf16(w, transpose=False, flip=False):
    w = _f32c(w)
    if transpose:
        Cin, Cout, K = w.shape
    else:
        Cout, Cin, K = w.shape
    wt = torch.empty(K, Cout, Cin, dtype=torch.bfloat16, device=w.device)
    call("rave_weight_to_tapmajor_bf16", ptr(w), ptr(wt), Cout, Cin, K, int(transpose), int(flip),
         stream_ptr())
    return wt


# ----------------------------------------------------------------------------------------------
# tensor-core engine (channel-last bf16 operands), raw launches
# ----------------------------------------------------------------------------------------------

def ncl_to_cl(x, act=ACT_NONE, slope=0.2, alpha=None, want_bf16=True, want_f32=False):
    """[B,C,L] fp32 -> channel-last ([B,L,C] bf16 = act(x), and/or [B,L,C] fp32 = x)."""
    x = _f32c(x)
    B, C, L = x.shape
    yb = torch.empty(B, L, C, dtype=torch.bfloat16, device=x.device) if want_bf16 else None
    yf = torch.empty(B, L, C, dtype=torch.float32, device=x.device) if want_f32 else None
    call("rave_ncl_to_cl", ptr(x), ptr(yb), ptr(yf), B, C, L, act, float(slope), ptr(alpha), stream_ptr())
    return yb, yf


def ncl_to_cl_x3(x):
    """[B,C,L] fp32 -> channel-last split operand [B,L,2C] bf16: [hi = bf16(x) | lo = bf16(x - hi)]."""
    x = _f32c(x)
    B, C, L = x.shape
    y = torch.empty(B, L, 2 * C, dtype=torch.bfloat16, device=x.device)
    call("rave_ncl_to_cl_x3", ptr(x), ptr(y), B, C, L, stream_ptr())
    return y


def cl_to_ncl(x_cl):
    """[B,L,C] fp32 -> [B,C,L] fp32."""
    x_cl = _f32c(x_cl)
    B, L, C = x_cl.shape
    y = torch.empty(B, C, L, dtype=torch.float32, device=x_cl.device)
    call("rave_cl_to_ncl", ptr(x_cl), ptr(y), B, C, L, stream_ptr())
    return y


def conv1d_tc_supported(Cin, Cout, K=1, stride=1, dil=1):
    return bool(_lib.load().rave_conv1d_tc_supported(Cin, Cout, K, stride, dil))


def conv1d_tc(xa_cl, wt, bias=None, res_cl=None, stride=1, dil=1, pad=(0, 0), act=ACT_NONE, slope=0.2,
              want_f32=True, want_act=False, out_f32=None, out_act=None, out_rows=0, out_row_stride=0,
              out_row_offset=0, Lout=None, res_bf16=None, dact_src=None, Lin=None, res_act=None, res_slope=0.2,
              fm_d=None, fm_partner=None, x3=False, act_cs=0):
    """xa_cl [B,Lin,Cin] bf16 (activated operand), wt [K,Cout,Cin] bf16 -> (out_f32 [B,Lout,Cout] fp32,
    out_act [B,Lout,Cout] bf16 = act(out)); either may be None.  fm_d (2 device floats): fused feature-matching
    gradient of a [real; fake] batch, see include/rave_b200.h; with fm_partner (the real rows, stored right before
    dact_src in the same allocation) the launch covers the fake half only."""
    B, in_pitch, Cin = xa_cl.shape          # allocated rows per batch; true length = Lin (slack rows zero)
    if Lin is None:
        Lin = in_pitch
    K, Cout, Cin_w = wt.shape
    if x3:                                   # split operands: rows [hi | lo] of 2*Cin, weights [2][K][Cout][Cin]
        if Cin % 2 or K % 2:
            raise _lib.RaveB200Error("conv1d_tc(x3): operands must be [hi | lo] pairs")
        Cin //= 2
        K //= 2
    if Cin_w != Cin or xa_cl.dtype != torch.bfloat16 or wt.dtype != torch.bfloat16:
        raise _lib.RaveB200Error("conv1d_tc: operand mismatch")
    if Lout is None:
        Lout = conv_out_len(Lin, K, stride, dil, pad[0], pad[1])
    rows = out_rows if out_rows else Lout
    if want_f32 and out_f32 is None:
        out_f32 = torch.empty(B, rows, Cout, dtype=torch.float32, device=xa_cl.device)
    if want_act and out_act is None:
        out_act = torch.empty(B, rows, Cout * (2 if x3 else 1), dtype=torch.bfloat16, device=xa_cl.device)
    if x3:
        if res_bf16 is not None or dact_src is not None or fm_d is not None:
            raise _lib.RaveB200Error("conv1d_tc(x3): forward path only")
        call("rave_conv1d_tc_fwd_x3", ptr(xa_cl), ptr(wt), ptr(bias), ptr(res_cl), ptr(res_act), float(res_slope),
             ptr(out_f32), ptr(out_act), B, Cin, Lin, in_pitch, Cout, Lout, K, stride, dil, pad[0], act, float(slope),
             out_rows, out_row_stride, out_row_offset, act_cs, stream_ptr())
        return out_f32, out_act
    fm_bh = 0
    if fm_d is not None:
        fm_bh = B // 2
        if fm_partner is not None:
            if (fm_partner.shape != dact_src.shape or not fm_partner.is_contiguous()
                    or fm_partner.data_ptr() + fm_partner.numel() * fm_partner.element_size() != dact_src.data_ptr()):
                raise _lib.RaveB200Error("conv1d_tc: fm_partner must be the half stored right before dact_src")
            fm_bh = -B
    call("rave_conv1d_tc_fwd", ptr(xa_cl), ptr(wt), ptr(bias), ptr(res_cl), ptr(res_bf16), ptr(dact_src),
         ptr(res_act), float(res_slope), ptr(out_f32), ptr(out_act), B, Cin, Lin, in_pitch, Cout, Lout, K, stride, dil, pad[0], act, float(slope),
         out_rows, out_row_stride, out_row_offset, fm_d.data_ptr() if fm_d is not None else None,
         fm_bh, stream_ptr())
    return out_f32, out_act


class TimeStackFn(torch.autograd.Function):
    """x [B, C, T, F] fp32 -> [(b t), Fp, Cp] bf16 rows holding the kt time-shifted copies of the channels side by side
    (rave_time_stack_cl); backward = the adjoint gather."""

    @staticmethod
    def forward(ctx, x, kt, pt, Cp, Fp):
        x = _f32c(x)
        B, C, T, F_ = x.shape
        out = torch.empty(B * T, Fp, Cp, dtype=torch.bfloat16, device=x.device)
        call("rave_time_stack_cl", ptr(x), ptr(out), B, C, T, F_, Fp, Cp, kt, pt, stream_ptr())
        ctx.cfg = (B, C, T, F_, Fp, Cp, kt, pt)
        return out

    @staticmethod
    def backward(ctx, g):
        B, C, T, F_, Fp, Cp, kt, pt = ctx.cfg
        g = g.contiguous()
        gx = torch.empty(B, C, T, F_, dtype=torch.float32, device=g.device)
        call("rave_time_stack_cl_bwd", ptr(g), ptr(gx), B, C, T, F_, Fp, Cp, kt, pt, stream_ptr())
        return gx, None, None, None, None


def time_stack_cl(x, kt, pt, Cp, Fp):
    return TimeStackFn.apply(x, kt, pt, Cp, Fp)


class TimeStackNhwcFn(torch.autograd.Function):
    """x [B, T, F, C] fp32 channel-last (any batch / time strides, channels and positions dense) -> the same
    [(b t), Fp, Cp] bf16 operand, tap dt reading time t + dt * dil - pt (rave_time_stack_nhwc_dil); backward = the
    adjoint into a contiguous [B, T, F, C]."""

    @staticmethod
    def forward(ctx, x, kt, pt, Cp, Fp, dil):
        if x.dtype != torch.float32:
            x = x.float()
        B, T, F_, C = x.shape
        if x.stride(3) != 1 or x.stride(2) != C:
            x = x.contiguous()
        out = torch.empty(B * T, Fp, Cp, dtype=torch.bfloat16, device=x.device)
        if not x.is_cuda:
            raise _lib.RaveB200Error("rave_b200 ops need CUDA tensors (there is no CPU path)")
        call("rave_time_stack_nhwc_dil", x.data_ptr(), ptr(out), B, C, T, F_, x.stride(0), x.stride(1), Fp, Cp, kt, pt,
             dil, stream_ptr())     # x: a strided view (band slice of the spectrogram / rows of the previous output)
        ctx.cfg = (B, C, T, F_, Fp, Cp, kt, pt, dil)
        return out

    @staticmethod
    def backward(ctx, g):
        B, C, T, F_, Fp, Cp, kt, pt, dil = ctx.cfg
        g = g.contiguous()
        gx = torch.empty(B, T, F_, C, dtype=torch.float32, device=g.device)
        call("rave_time_stack_nhwc_dil_bwd", ptr(g), ptr(gx), B, C, T, F_, Fp, Cp, kt, pt, dil, stream_ptr())
        return gx, None, None, None, None, None


def time_stack_nhwc(x, kt, pt, Cp, Fp, dil=1):
    return TimeStackNhwcFn.apply(x, kt, pt, Cp, Fp, dil)


class L1HalvesFn(torch.autograd.Function):
    """(sum |real - fake|, sum |real|) where real / fake are the first / second half (along dim 0) of ONE contiguous fp32
    buffer -- the discriminator ran on cat([real, fake]) -- and the gradient written into one buffer of the same layout
    (no split / cat passes).  Zero padding inside the buffer, identical in both halves, contributes nothing."""

    @staticmethod
    def forward(ctx, base):
        if base.dtype != torch.float32 or not base.is_contiguous() or base.shape[0] % 2:
            raise _lib.RaveB200Error("l1_halves: contiguous fp32 buffer with an even leading dimension expected")
        half = base.numel() // 2
        flat = base.view(-1)
        stats = torch.zeros(2, dtype=torch.float32, device=base.device)
        call("rave_l1_stats_f32", ptr(flat[:half]), ptr(flat[half:]), ptr(stats), half, stream_ptr())
        ctx.save_for_backward(base)
        return stats

    @staticmethod
    def backward(ctx, d):
        (base,) = ctx.saved_tensors
        d = _f32c(d)
        half = base.numel() // 2
        flat = base.view(-1)
        g = torch.empty_like(base)
        gf = g.view(-1)
        call("rave_l1_grad_f32", ptr(flat[:half]), ptr(flat[half:]), ptr(d), ptr(gf[:half]), ptr(gf[half:]), half,
             stream_ptr())
        return g


def l1_halves(base):
    return L1HalvesFn.apply(base)


class LeakyFmFn(torch.autograd.Function):
    """Feature tap of the Descript discriminator: x = a chain's fp32 output holding [real; fake] halves along dim 0 ->
    (a = LeakyReLU(x), stats = (sum |a_r - a_f|, sum |a_r|)) in one pass; one backward pass folds the gradient of the
    two sums, the gradient arriving at `a` and LeakyReLU' together (rave_leaky_fm_fwd / _bwd)."""

    @staticmethod
    def forward(ctx, x, slope):
        if x.dtype != torch.float32 or not x.is_contiguous() or x.shape[0] % 2:
            raise _lib.RaveB200Error("leaky_fm: contiguous fp32 buffer with an even leading dimension expected")
        ctx.set_materialize_grads(False)
        a = torch.empty_like(x)
        stats = torch.zeros(2, dtype=torch.float32, device=x.device)
        call("rave_leaky_fm_fwd", ptr(x), ptr(a), ptr(stats), x.numel() // 2, float(slope), stream_ptr())
        ctx.save_for_backward(a)
        ctx.slope = float(slope)
        return a, stats

    @staticmethod
    def backward(ctx, ga, dstats):
        (a,) = ctx.saved_tensors
        if ga is None and dstats is None:
            return None, None
        ga = _f32c(ga)
        dstats = _f32c(dstats)
        gx = torch.empty_like(a)
        call("rave_leaky_fm_bwd", ptr(a), ptr(ga), ptr(dstats), ptr(gx), a.numel() // 2, ctx.slope, stream_ptr())
        return gx, None


def leaky_fm(x, slope):
    return LeakyFmFn.apply(x, slope)


class LeakyFmStackFn(torch.autograd.Function):
    """LeakyFmFn that also writes the NEXT conv's operand in the same pass: x [(b t), F, C] fp32 with whole batch
    entries of T steps (first half of the rows real) -> (a, stats, xs) with xs [(b t), Fp, 3 C] bf16 =
    time_stack_nhwc(a.view(B, T, F, C), kt = 3, pt = dil, dil) (rave_leaky_fm_stack_dil_fwd; dil = 1 for the MRD, 1 / 2 / 4
    along the EncodecConvNet).  The backward is the composition of the two stand-alone backward kernels (adjoint of the
    time stack, then the tap's fused backward) in ONE kernel (rave_leaky_fm_stack_dil_bwd)."""

    @staticmethod
    def forward(ctx, x, slope, T, Fp, dil):
        if x.dtype != torch.float32 or not x.is_contiguous() or x.dim() != 3 or x.shape[0] % (2 * T) or x.shape[2] % 4:
            raise _lib.RaveB200Error("leaky_fm_stack: contiguous fp32 [(b t), F, C] rows, even batch, C % 4 == 0 expected")
        R2, F_, C = x.shape
        ctx.set_materialize_grads(False)
        a = torch.empty_like(x)
        stats = torch.zeros(2, dtype=torch.float32, device=x.device)
        xs = torch.empty(R2, Fp, 3 * C, dtype=torch.bfloat16, device=x.device)
        call("rave_leaky_fm_stack_dil_fwd", ptr(x), ptr(a), ptr(stats), ptr(xs), R2 // 2, T, F_, C, Fp, dil,
             float(slope), stream_ptr())
        ctx.save_for_backward(a)
        ctx.slope = float(slope)
        ctx.cfg = (C, T, F_, Fp, dil)
        return a, stats, xs

    @staticmethod
    def backward(ctx, ga, dstats, gxs):
        (a,) = ctx.saved_tensors
        if ga is None and dstats is None and gxs is None:
            return None, None, None, None, None
        C, T, F_, Fp, dil = ctx.cfg
        ga, dstats = _f32c(ga), _f32c(dstats)
        gx = torch.empty_like(a)
        if gxs is not None:
            # one pass: adjoint of the time stack + gradient at the feature + feature-matching terms + LeakyReLU'
            gxs = gxs.contiguous()
            call("rave_leaky_fm_stack_dil_bwd", ptr(a), ptr(gxs), ptr(ga), ptr(dstats), ptr(gx), a.shape[0] // 2, T, F_, C,
                 Fp, dil, ctx.slope, stream_ptr())
        else:
            call("rave_leaky_fm_bwd", ptr(a), ptr(ga), ptr(dstats), ptr(gx), a.numel() // 2, ctx.slope, stream_ptr())
        return gx, None, None, None, None


def leaky_fm_stack(x, slope, T, Fp, dil=1):
    return LeakyFmStackFn.apply(x, slope, T, Fp, dil)


class L1StatsFn(torch.autograd.Function):
    """(sum |t - v|, sum |t|) of two fp32 CUDA tensors in one pass, gradient in one pass (rave_l1_stats_f32 / _grad)."""

    @staticmethod
    def forward(ctx, t, v):
        t, v = _f32c(t), _f32c(v)
        stats = torch.zeros(2, dtype=torch.float32, device=t.device)
        call("rave_l1_stats_f32", ptr(t), ptr(v), ptr(stats), t.numel(), stream_ptr())
        ctx.save_for_backward(t, v)
        return stats

    @staticmethod
    def backward(ctx, d):
        t, v = ctx.saved_tensors
        d = _f32c(d)
        gt = torch.empty_like(t) if ctx.needs_input_grad[0] else None
        gv = torch.empty_like(v) if ctx.needs_input_grad[1] else None
        if gt is None and gv is None:
            return None, None
        call("rave_l1_grad_f32", ptr(t), ptr(v), ptr(d), ptr(gt), ptr(gv), t.numel(), stream_ptr())
        return gt, gv


def l1_stats(t, v):
    return L1StatsFn.apply(t, v)


def snake_cl_fwd(h_cl, alpha):
    """Channel-last Snake on an engine stream: h_cl [B, pitch, C] (ACT dtype) -> a = h + sin^2(alpha h) / (alpha + 1e-9)."""
    h_cl = h_cl.contiguous()
    C = h_cl.shape[-1]
    a = torch.empty_like(h_cl)
    al = _f32c(alpha.detach().reshape(-1))
    call("rave_snake_cl_fwd", ptr(h_cl), ptr(al), ptr(a), h_cl.numel() // C, C, stream_ptr())
    return a


def snake_cl_bwd(ga_cl, h_cl, alpha, add=None, want_dalpha=True):
    """g_h = g_a * dsnake/dh (+ add), dalpha [C] fp32 = sum over rows of g_a * dsnake/dalpha (None if not wanted)."""
    ga_cl, h_cl = ga_cl.contiguous(), h_cl.contiguous()
    C = h_cl.shape[-1]
    gh = torch.empty_like(ga_cl)
    al = _f32c(alpha.detach().reshape(-1))
    dal = torch.zeros(C, dtype=torch.float32, device=h_cl.device) if want_dalpha else None
    if add is not None:
        add = add.contiguous()
    call("rave_snake_cl_bwd", ptr(ga_cl), ptr(h_cl), ptr(al), ptr(add), ptr(gh), ptr(dal), h_cl.numel() // C, C,
         stream_ptr())
    return gh, dal


def _adain_buffer(t, C, rows=None):
    if t.dtype != torch.float32 or not t.is_contiguous() or t.shape[1:] != ((C, 1) if rows is None else ()) \
            or (rows is not None and t.numel() != rows):
        raise _lib.RaveB200Error(f"adain: statistics buffer of shape {tuple(t.shape)} / {t.dtype} does not fit C = {C}")
    return t


def adain_cl_stats(h_cl, L, mean_x, std_x, mean_y, std_y, learn_x, learn_y, num_update_x, num_update_y):
    """AdaptiveInstanceNormalization's eval-mode statistics on an engine stream h_cl [B, pitch, C] bf16 (first L rows
    valid), written into the module's own buffers (mean_* / std_* [N, C, 1], learn_* / num_update_* [1], fp32; B <= N):
    the learn_y / learn_x running update and counter step, all decided on the device.  Returns (scale, shift) [B, C]
    fp32 of the transfer (exactly 1 / 0 where it does not apply).  Forward only: the buffers are not autograd inputs."""
    B, pitch, C = h_cl.shape
    stats = [_adain_buffer(t, C) for t in (mean_x, std_x, mean_y, std_y)]
    flags = [_adain_buffer(t, C, rows=1) for t in (learn_x, learn_y, num_update_x, num_update_y)]
    if h_cl.dtype != torch.bfloat16 or not (0 < L <= pitch):
        raise _lib.RaveB200Error("adain_cl_stats: h must be a bf16 [B, pitch, C] stream with 0 < L <= pitch")
    scale = torch.empty(B, C, dtype=torch.float32, device=h_cl.device)
    shift = torch.empty_like(scale)
    call("rave_adain_cl_stats", ptr(h_cl), B, int(L), pitch, C, *(ptr(t) for t in stats), *(ptr(t) for t in flags),
         mean_x.shape[0], ptr(scale), ptr(shift), stream_ptr())
    return scale, shift


def adain_snake_cl_fwd(h_cl, alpha, scale, shift, L):
    """h_cl [B, pitch, C] bf16 <- h scale + shift on rows < L (in place: the residual's skip stream); returns the Snake
    operand a = Snake(h) [B, pitch, C] with zero rows [L, pitch)."""
    B, pitch, C = h_cl.shape
    if h_cl.dtype != torch.bfloat16 or scale.shape != (B, C) or shift.shape != (B, C) or not (0 < L <= pitch):
        raise _lib.RaveB200Error("adain_snake_cl_fwd: h [B, pitch, C] bf16, scale / shift [B, C], 0 < L <= pitch")
    a = torch.empty_like(h_cl)
    al = _f32c(alpha.detach().reshape(-1))
    call("rave_adain_snake_cl_fwd", ptr(h_cl), ptr(al), ptr(_f32c(scale)), ptr(_f32c(shift)), ptr(a), B, int(L), pitch,
         C, stream_ptr())
    return a


def dilated_unit_tc_supported(C, L):
    return bool(_lib.load().rave_dilated_unit_tc_supported(C, L))


def dilated_unit_tc(xa_cl, w3t, w1t, dil, pad_l, slope_in, slope_mid, act_out, slope_out, L=None, want_a1=False,
                    out_f32=None, out_act=None):
    """Fused Residual(DilatedUnit) forward (rave_dilated_unit_tc_fwd): xa_cl [B, pitch, C] bf16 = LeakyReLU(x),
    w3t [3, C, C], w1t [1, C, C] bf16 -> (a1 [B, pitch, C] bf16 | None, out_f32, out_act)."""
    B, pitch, C = xa_cl.shape
    L = pitch if L is None else L
    if w3t.shape != (3, C, C) or w1t.shape != (1, C, C):
        raise _lib.RaveB200Error("dilated_unit_tc: weight shapes")
    a1 = torch.empty(B, pitch, C, dtype=torch.bfloat16, device=xa_cl.device) if want_a1 else None
    if a1 is not None and pitch > L:
        a1[:, L:].zero_()
    call("rave_dilated_unit_tc_fwd", ptr(xa_cl), ptr(w3t), ptr(w1t), ptr(a1), ptr(out_f32), ptr(out_act), B, C, L,
         pitch, dil, pad_l, float(slope_in), float(slope_mid), act_out, float(slope_out), stream_ptr())
    return a1, out_f32, out_act


def conv1d_tc_wgrad(P_cl, Q_cl, K, stride=1, dil=1, pad_l=0, Lp=None, Lq=None, dbias=None):
    """dwt[k][m][n] = sum_{b,l} P[b,l,m] * Q[b, l*stride + k*dil - pad_l, n]  (bf16 operands, fp32 result).
    Tensors may be allocated with a row pitch larger than their true length (Lp / Lq).
    dbias [Cm] fp32 (pre-zeroed): += column sums of P over its Lp valid rows (conv bias gradient)."""
    B, p_pitch, Cm = P_cl.shape
    _, q_pitch, Cn = Q_cl.shape
    Lp = p_pitch if Lp is None else Lp
    Lq = q_pitch if Lq is None else Lq
    if P_cl.dtype != torch.bfloat16 or Q_cl.dtype != torch.bfloat16:
        raise _lib.RaveB200Error("conv1d_tc_wgrad: operands must be bf16")
    splits = _lib.load().rave_conv1d_tc_wgrad_splits(B, Cm, Lp, Cn, K)
    dwt = torch.empty(splits, K, Cm, Cn, dtype=torch.float32, device=P_cl.device)   # per-slice partial sums
    call("rave_conv1d_tc_wgrad", ptr(P_cl), ptr(Q_cl), ptr(dwt), dbias.data_ptr() if dbias is not None else None,
         B, Cm, Lp, p_pitch, Cn, Lq, q_pitch, K, stride, dil, pad_l, stream_ptr())
    return dwt


def tapmajor_to_weight(dwt, transpose=False):
    """sum over the leading split axis of dwt [S][K][Cm][Cn] and re-layout to the parameter's [.,.,K]."""
    S, K, Cm, Cn = dwt.shape
    dw = torch.empty((Cn, Cm, K) if transpose else (Cm, Cn, K), dtype=torch.float32, device=dwt.device)
    call("rave_tapmajor_to_weight_f32", ptr(dwt), ptr(dw), Cm, Cn, K, int(transpose), S, stream_ptr())
    return dw


def weight_prep_tc(v, g, tapsA, tapsB, C0p, C1p):
    """v [C0][C1][K(,1)] fp32 (+ weight-norm g) -> (norm [C0] | None, outA [nA][C0p][C1p] bf16 | None,
    outB [nB][C1p][C0p] bf16 | None) with out?[t] = bf16(w[..][..][taps?[t]]), w = g v/||v|| (or v)."""
    import ctypes
    v = _f32c(v)
    g = _f32c(g)
    C0, C1 = v.shape[0], v.shape[1]
    K = v.numel() // (C0 * C1)
    dev = v.device
    norm = torch.empty(C0, dtype=torch.float32, device=dev) if g is not None else None
    outA = torch.empty(len(tapsA), C0p, C1p, dtype=torch.bfloat16, device=dev) if tapsA else None
    outB = torch.empty(len(tapsB), C1p, C0p, dtype=torch.bfloat16, device=dev) if tapsB else None
    arrA = (ctypes.c_int * max(1, len(tapsA)))(*tapsA)
    arrB = (ctypes.c_int * max(1, len(tapsB)))(*tapsB)
    call("rave_weight_prep_tc", ptr(v), ptr(g), ptr(norm), ptr(outA), arrA, len(tapsA), ptr(outB), arrB,
         len(tapsB), C0, C1, K, C0p, C1p, stream_ptr())
    return norm, outA, outB


def weight_norm_bwd_tapmajor(dwt, v, g, norm):
    """dwt [S][K][C0p][C1p] fp32 partial sums -> (dv like v, dg like g | None)."""
    v = _f32c(v)
    dv = torch.empty_like(v)
    dg = torch.empty_like(g) if g is not None else None
    C0, C1 = v.shape[0], v.shape[1]
    K = v.numel() // (C0 * C1)
    call("rave_weight_norm_bwd_tapmajor", ptr(dwt), ptr(v), ptr(g), ptr(norm), ptr(dv), ptr(dg), C0, C1, K,
         dwt.shape[2], dwt.shape[3], dwt.shape[0], stream_ptr())
    return dv, dg


# ----------------------------------------------------------------------------------------------
# small-channel discriminator kernels (csrc/conv_small.cu)
# ----------------------------------------------------------------------------------------------

def conv1d_c1(x_rows, w, bias, Lin, stride, pad, act, slope, out_f32=None, out_act=None, Lout=None):
    """First conv of a ConvNet (Cin = 1): x_rows [R, x_pitch] fp32, w [Cout, 1, K(,1)] fp32 ->
    channel-last outputs [R, out_pitch, Cout] written in place (fp32 stream and/or bf16 act(out))."""
    x_rows = _f32c(x_rows)
    w = _f32c(w)
    R, x_pitch = x_rows.shape
    Cout = w.shape[0]
    K = w.numel() // Cout
    ref = out_f32 if out_f32 is not None else out_act
    call("rave_conv1d_c1_fwd", ptr(x_rows), ptr(w), ptr(bias), ptr(out_f32), ptr(out_act), R, x_pitch, Lin, Cout,
         Lout, ref.shape[1], K, stride, pad[0], act, float(slope), stream_ptr())
    return out_f32, out_act


def conv1d_c1_wgrad(g_cl, x_rows, Cout, K, Lin, Lout, stride, pad_l):
    """dwt [S, K, Cout, 1] fp32 partial sums: sum_rows g[r,l,co] * x[r, l*stride + k - pad_l]."""
    R, g_pitch, Cg = g_cl.shape
    x_rows = _f32c(x_rows)
    splits = _lib.load().rave_conv1d_c1_wgrad_splits(R, Lout)
    dwt = torch.empty(splits, K, Cout, 1, dtype=torch.float32, device=g_cl.device)
    call("rave_conv1d_c1_wgrad", ptr(g_cl), ptr(x_rows), ptr(dwt), R, x_rows.shape[1], Lin, Cout, Cg, Lout, g_pitch,
         K, stride, pad_l, stream_ptr())
    return dwt


def fm_stats(a_cl, stats_row, L, slope):
    """stats_row[0:2] += (sum |h_r - h_f|, sum |h_r|) over the real/fake batch halves of a = leaky(h)."""
    B2, pitch, C = a_cl.shape
    call("rave_fm_stats", ptr(a_cl), stats_row.data_ptr(), B2 // 2, L, pitch, C, float(slope), stream_ptr())


def fm_grad(a_cl, dstats_row, L, slope):
    """bf16 gradient stream of dstats_row[0]*S_diff + dstats_row[1]*S_abs with respect to h."""
    B2, pitch, C = a_cl.shape
    g = torch.empty_like(a_cl)
    call("rave_fm_grad", ptr(a_cl), dstats_row.data_ptr(), ptr(g), B2 // 2, L, pitch, C, float(slope), stream_ptr())
    return g


def score_stats(score_cl, stats6, L):
    """stats6[0:6] += the six sums of the discriminator score tail (channel 0 of the fp32 channel-last score
    tensor [2*Bh, pitch, C], real half first): |s_r-s_f|, |s_r|, relu(1-s_r), relu(1+s_f), s_r, s_f."""
    B2, pitch, C = score_cl.shape
    call("rave_score_stats", ptr(score_cl), stats6.data_ptr(), B2 // 2, L, pitch, C, stream_ptr())


def score_grad(score_cl, dstats6, L):
    """bf16 gradient stream [2*Bh, pitch, C] of sum_i dstats6[i] * stats6[i] with respect to the score."""
    B2, pitch, C = score_cl.shape
    g = torch.empty(B2, pitch, C, dtype=torch.bfloat16, device=score_cl.device)
    call("rave_score_grad", ptr(score_cl), dstats6.data_ptr(), ptr(g), B2 // 2, L, pitch, C, stream_ptr())
    return g


def weight_norm_raw(v, g):
    """(w, norm) = (g v/||v||, ||v||) without autograd (engine-internal)."""
    v, g = _f32c(v), _f32c(g)
    C0 = v.shape[0]
    w = torch.empty_like(v)
    norm = torch.empty(C0, dtype=torch.float32, device=v.device)
    call("rave_weight_norm_fwd", ptr(v), ptr(g), ptr(w), ptr(norm), C0, v.numel() // C0, stream_ptr())
    return w, norm


def conv1d_c1_dgrad(g_cl, w, x_pitch, Lin, Lout, stride, pad_l):
    """dx rows [R, x_pitch] fp32 of the Cin = 1 first conv (w: effective weight [Cout, 1, K(,1)])."""
    R, g_pitch, Cg = g_cl.shape
    w = _f32c(w)
    Cout = w.shape[0]
    K = w.numel() // Cout
    dx = torch.zeros(R, x_pitch, dtype=torch.float32, device=g_cl.device) if x_pitch > Lin else \
        torch.empty(R, x_pitch, dtype=torch.float32, device=g_cl.device)
    call("rave_conv1d_c1_dgrad", ptr(g_cl), ptr(w), ptr(dx), R, x_pitch, Lin, Cout, Cg, Lout, g_pitch, K, stride,
         pad_l, stream_ptr())
    return dx


def colsum_bf16(g_cl, L, C):
    """sum over batch and the first L rows of a channel-last gradient stream -> [C] fp32 (bias gradient)."""
    R, pitch, Cg = g_cl.shape
    if g_cl.dtype != torch.bfloat16:
        return g_cl[:, :L, :C].float().sum((0, 1))
    out = torch.empty(C, dtype=torch.float32, device=g_cl.device)
    call("rave_colsum_bf16", ptr(g_cl), ptr(out), R, L, pitch, Cg, C, stream_ptr())
    return out


def im2col_c1(src, Lin, Lout, out_pitch, K, stride, pad_l, period=1, pool=1):
    """X [R, out_pitch, 16] bf16 with X[r,l,k] = row_r[l*stride + k - pad_l] (zero outside / beyond K, Lout), the
    R = Bs*period rows read straight from src [Bs, T]: row b*period + w, position i ->
    mean_j src[b, (i*pool + j)*period + w] (MPD fold / MSD average pooling, see include/rave_b200.h)."""
    src = _f32c(src)
    Bs, T = src.shape
    R = Bs * period
    X = torch.empty(R, out_pitch, 16, dtype=torch.bfloat16, device=src.device)
    call("rave_im2col_c1", ptr(src), ptr(X), R, T, T, Lin, Lout, out_pitch, K, stride, pad_l, period, pool,
         stream_ptr())
    return X


def gather_c1(P_cl, src_shape, Lin, Lout, K, stride, pad_l, period=1, pool=1, batch0=0):
    """dsrc [Bs, T] fp32: the adjoint of im2col_c1 applied to P [R, p_pitch, 16] fp32 (taps, pooling, fold).  With
    batch0 > 0, P holds only the rows of source batches batch0 .. Bs-1 (the other gradients stay zero)."""
    P_cl = _f32c(P_cl)
    R, p_pitch, _ = P_cl.shape
    Bs, T = src_shape
    dsrc = torch.zeros(Bs, T, dtype=torch.float32, device=P_cl.device)
    if R != (Bs - batch0) * period:
        raise _lib.RaveB200Error("gather_c1: row count does not match the source batches")
    call("rave_gather_c1", ptr(P_cl), dsrc.data_ptr() + batch0 * T * 4, R, T, T, Lin, Lout, p_pitch, K, stride, pad_l,
         period, pool, stream_ptr())
    return dsrc


def cin_width(cin, K):
    """Row width W (bf16 columns) of the multichannel first-layer operand: 16 or 32 >= cin*K."""
    return 16 if cin * K <= 16 else 32


def im2col_cin(src, Lin, Lout, out_pitch, K, stride, pad_l, period=1, pool=1):
    """im2col_c1 for a first layer with Cin = src.shape[1] channels: X [R, out_pitch, W] bf16 (W = cin_width(cin, K))
    with X[r, l, c*K + k] = row_{r,c}[l*stride + k - pad_l], the rows read from src [Bs, cin, T] through the fold /
    pooling of each channel (R = Bs*period)."""
    src = _f32c(src)
    Bs, cin, T = src.shape
    W = cin_width(cin, K)
    R = Bs * period
    X = torch.empty(R, out_pitch, W, dtype=torch.bfloat16, device=src.device)
    call("rave_im2col_cin", ptr(src), ptr(X), R, cin, T, T, Lin, Lout, out_pitch, W, K, stride, pad_l, period, pool,
         stream_ptr())
    return X


def gather_cin(P_cl, src_shape, Lin, Lout, K, stride, pad_l, period=1, pool=1, batch0=0):
    """dsrc [Bs, cin, T] fp32: the adjoint of im2col_cin applied to P [R, p_pitch, W] fp32.  With batch0 > 0, P holds
    only the rows of source batches batch0 .. Bs-1 (the other gradients stay zero)."""
    P_cl = _f32c(P_cl)
    R, p_pitch, W = P_cl.shape
    Bs, cin, T = src_shape
    dsrc = torch.zeros(Bs, cin, T, dtype=torch.float32, device=P_cl.device)
    if R != (Bs - batch0) * period or W != cin_width(cin, K):
        raise _lib.RaveB200Error("gather_cin: P does not match the source batches or the row width")
    call("rave_gather_cin", ptr(P_cl), dsrc.data_ptr() + batch0 * cin * T * 4, R, cin, T, T, Lin, Lout, p_pitch, W, K,
         stride, pad_l, period, pool, stream_ptr())
    return dsrc


# ----------------------------------------------------------------------------------------------
# fused spectral distance of one STFT scale (csrc/spectral.cu)
# ----------------------------------------------------------------------------------------------

class SpectralDistanceFn(torch.autograd.Function):
    """lin + log distance between complex spectrograms X (target, no gradient) and Y (reconstruction)."""

    @staticmethod
    def forward(ctx, X, Y, eps):
        if X.dtype != torch.complex64 or Y.dtype != torch.complex64 or X.shape != Y.shape:
            raise _lib.RaveB200Error("spectral distance expects two complex64 spectrograms of equal shape")
        # the kernels are elementwise: any COMMON dense layout will do (torch.stft returns a transposed
        # view of a [N, frames, bins] buffer) -- avoid materialising contiguous copies
        if X.stride() == Y.stride() and X.transpose(-1, -2).is_contiguous():
            X, Y = X.transpose(-1, -2), Y.transpose(-1, -2)
            ctx.transposed = True
        else:
            X, Y = X.contiguous(), Y.contiguous()
            ctx.transposed = False
        n = X.numel()
        stats = torch.zeros(5, dtype=torch.float32, device=X.device)     # 3 sums, block ticket, distance
        call("rave_spectral_stats", ptr(torch.view_as_real(X)), ptr(torch.view_as_real(Y)), ptr(stats), n,
             float(eps), stream_ptr())
        ctx.save_for_backward(X, Y)
        ctx.stats = stats
        ctx.eps = float(eps)
        return stats[4]

    @staticmethod
    def backward(ctx, g):
        X, Y = ctx.saved_tensors
        stats = ctx.stats
        n = X.numel()
        g = g.to(torch.float32)
        if g.dim() != 0 or not g.is_cuda:
            raise _lib.RaveB200Error("spectral distance: the upstream gradient must be a CUDA scalar")
        dY = torch.empty_like(Y, memory_format=torch.contiguous_format)
        call("rave_spectral_grad", ptr(torch.view_as_real(X)), ptr(torch.view_as_real(Y)),
             ptr(torch.view_as_real(dY)), stats.data_ptr(), g.data_ptr(), n, ctx.eps, stream_ptr())
        return None, (dY.transpose(-1, -2) if ctx.transposed else dY), None


def spectral_distance(X, Y, eps):
    return SpectralDistanceFn.apply(X, Y, eps)


class StftFramesFn(torch.autograd.Function):
    """Windowed, reflect-padded frames [N, F, n_fft] of x [N, T] (torch.stft's framing, center=True)."""

    @staticmethod
    def forward(ctx, x, window, n_fft, hop):
        x = _f32c(x)
        N, T = x.shape
        F = 1 + T // hop
        frames = torch.empty(N, F, n_fft, dtype=torch.float32, device=x.device)
        call("rave_stft_frames", ptr(x), ptr(window), ptr(frames), N, T, n_fft, hop, stream_ptr())
        ctx.save_for_backward(window)
        ctx.dims = (N, T, n_fft, hop)
        return frames

    @staticmethod
    def backward(ctx, g):
        (window,) = ctx.saved_tensors
        N, T, n_fft, hop = ctx.dims
        g = _f32c(g)
        dx = torch.empty(N, T, dtype=torch.float32, device=g.device)
        call("rave_stft_frames_bwd", ptr(g), ptr(window), ptr(dx), N, T, n_fft, hop, stream_ptr())
        return dx, None, None, None


def stft_frames(x, window, n_fft, hop):
    return StftFramesFn.apply(x, window, n_fft, hop)


class StftFramesValidFn(torch.autograd.Function):
    """Uncentred frames [N, F, n_fft] = scale * window * x[f*hop : f*hop + n_fft], F = 1 + (T - n_fft) // hop (torch.stft's
    framing with center=False; scale = 1 / ||window||_2 gives torchaudio's normalized=True)."""

    @staticmethod
    def forward(ctx, x, window, n_fft, hop, scale):
        x = _f32c(x)
        N, T = x.shape
        F = 1 + (T - n_fft) // hop
        frames = torch.empty(N, F, n_fft, dtype=torch.float32, device=x.device)
        call("rave_stft_frames_valid", ptr(x), ptr(window), ptr(frames), N, T, n_fft, hop, float(scale), stream_ptr())
        ctx.save_for_backward(window)
        ctx.dims = (N, T, n_fft, hop, float(scale))
        return frames

    @staticmethod
    def backward(ctx, g):
        (window,) = ctx.saved_tensors
        N, T, n_fft, hop, scale = ctx.dims
        g = _f32c(g)
        dx = torch.empty(N, T, dtype=torch.float32, device=g.device)
        call("rave_stft_frames_valid_bwd", ptr(g), ptr(window), ptr(dx), N, T, n_fft, hop, scale, stream_ptr())
        return dx, None, None, None, None


def stft_frames_valid(x, window, n_fft, hop, scale):
    return StftFramesValidFn.apply(x, window, n_fft, hop, scale)


class RfftFn(torch.autograd.Function):
    """torch.fft.rfft on the last axis of a [N, F, n] tensor with the backward written as ONE c2r transform: for
    y = rfft(x) and a gradient G of y, dx = irfft(Z, n) with Z = G * n * (1, 1/2, ..., 1/2, 1) and the imaginary parts of
    the DC / Nyquist bins dropped (checked against autograd in float64).  PyTorch's own backward zero-pads G to full
    length, runs a complex-to-complex transform of twice the size and copies the real part (4-5 launches on 33 MB
    tensors per STFT scale)."""

    @staticmethod
    def forward(ctx, x, w):
        ctx.n = x.shape[-1]
        ctx.save_for_backward(w)
        return torch.fft.rfft(x)

    @staticmethod
    def backward(ctx, g):
        (w,) = ctx.saved_tensors
        if g.is_cuda and g.dim() == 3 and g.dtype == torch.complex64:
            g = g.resolve_conj()
            N, F, bins = g.shape
            z = torch.empty(N, F, bins, dtype=torch.complex64, device=g.device)
            sN, sF, sB = g.stride()
            call("rave_rfft_bwd_scale", torch.view_as_real(g).data_ptr(), ptr(torch.view_as_real(z)), N, F, bins, sN,
                 sF, sB, stream_ptr())
        else:
            z = g * w
            z = torch.complex(z.real, torch.cat([torch.zeros_like(z.imag[..., :1]), z.imag[..., 1:-1],
                                                 torch.zeros_like(z.imag[..., :1])], -1))
        return torch.fft.irfft(z, n=ctx.n), None


def rfft(x, w):
    return RfftFn.apply(x, w)


class NoiseFirFn(torch.autograd.Function):
    """h [B, C*NB, T] (conv output), M [TS, NB], noise [B, T, C, TS] -> filtered noise [B, C, T*TS]
    (rave_noise_fir_fwd / _bwd: the whole tail of NoiseGeneratorV2.forward)."""

    @staticmethod
    def forward(ctx, h, M, noise, C):
        h = _f32c(h)
        noise = _f32c(noise)
        B, CN, T = h.shape
        NB = CN // C
        TS = M.shape[0]
        out = torch.empty(B, C, T * TS, dtype=torch.float32, device=h.device)
        call("rave_noise_fir_fwd", ptr(h), ptr(M), ptr(noise), ptr(out), B, C, NB, T, TS, stream_ptr())
        ctx.save_for_backward(h, M, noise)
        ctx.dims = (B, C, NB, T, TS)
        return out

    @staticmethod
    def backward(ctx, dout):
        h, M, noise = ctx.saved_tensors
        B, C, NB, T, TS = ctx.dims
        dh = torch.empty_like(h)
        call("rave_noise_fir_bwd", ptr(h), ptr(M), ptr(noise), ptr(_f32c(dout)), ptr(dh), B, C, NB, T, TS,
             stream_ptr())
        return dh, None, None, None


def noise_fir(h, M, noise, C):
    return NoiseFirFn.apply(h, M, noise, C)


# ----------------------------------------------------------------------------------------------
# multi-tensor weight preparation / weight-norm backward (one launch pair per chain)
# ----------------------------------------------------------------------------------------------

def weight_prep_tc_multi(items, x3=False, into=None):
    """items: list of (v, g, tapsA, tapsB, C0p, C1p).  Returns a list of (norm, outA, outB) exactly like
    weight_prep_tc, using ONE row-norm launch and ONE re-layout launch for (up to 64 of) the layers.
    x3: split-operand layouts, outA [2 * nA][C0p][C1p] / outB [2 * nB][C1p][C0p] = all hi slabs, then all lo slabs.
    into: list of (norm, outA, outB) tensors of an earlier call to overwrite in place (same shapes)."""
    P = 2 if x3 else 1
    outs = []
    recs = []
    for idx, (v, g, tapsA, tapsB, C0p, C1p) in enumerate(items):
        v = _f32c(v)
        g = _f32c(g)
        C0, C1 = v.shape[0], v.shape[1]
        K = v.numel() // (C0 * C1)
        dev = v.device
        if into is not None:
            norm, outA, outB = into[idx]
        else:
            norm = torch.empty(C0, dtype=torch.float32, device=dev) if g is not None else None
            outA = torch.empty(P * len(tapsA), C0p, C1p, dtype=torch.bfloat16, device=dev) if tapsA else None
            outB = torch.empty(P * len(tapsB), C1p, C0p, dtype=torch.bfloat16, device=dev) if tapsB else None
        outs.append((norm, outA, outB))
        recs.append((v, g, norm, outA, outB, tapsA, tapsB, C0, C1, K, C0p, C1p))
    for i0 in range(0, len(recs), 64):
        chunk = recs[i0:i0 + 64]
        arr = (_lib.WPrepLayer * len(chunk))()
        for L, (v, g, norm, outA, outB, tapsA, tapsB, C0, C1, K, C0p, C1p) in zip(arr, chunk):
            L.v, L.g, L.norm, L.outA, L.outB = ptr(v), ptr(g), ptr(norm), ptr(outA), ptr(outB)
            L.C0, L.C1, L.K, L.C0p, L.C1p, L.nA, L.nB, L.splits = C0, C1, K, C0p, C1p, len(tapsA), len(tapsB), 1
            for j, t in enumerate(tapsA):
                L.tapsA[j] = t
            for j, t in enumerate(tapsB):
                L.tapsB[j] = t
        call("rave_weight_prep_tc_multi_x3" if x3 else "rave_weight_prep_tc_multi", len(chunk), arr, stream_ptr())
    return outs


def weight_norm_bwd_multi(items):
    """items: list of (dwt [S][K][C0p][C1p], v, g | None, norm | None[, remap]).  remap = (wide, slots): the
    gradient buffer is phase-wide, [S][J][C0p][wide*C1p], with parameter tap k in slot slots[k] = j*wide + p.
    Returns a list of (dv, dg | None)."""
    outs = []
    recs = []
    for item in items:
        dwt, v, g, norm = item[:4]
        remap = item[4] if len(item) > 4 else None
        v = _f32c(v)
        dv = torch.empty_like(v)
        dg = torch.empty_like(g) if g is not None else None
        outs.append((dv, dg))
        recs.append((dwt, v, g, norm, dv, dg, remap))
    for i0 in range(0, len(recs), 64):
        chunk = recs[i0:i0 + 64]
        arr = (_lib.WPrepLayer * len(chunk))()
        for L, (dwt, v, g, norm, dv, dg, remap) in zip(arr, chunk):
            C0, C1 = v.shape[0], v.shape[1]
            L.v, L.g, L.norm, L.dwt, L.dv, L.dg = ptr(v), ptr(g), ptr(norm), ptr(dwt), ptr(dv), ptr(dg)
            L.C0, L.C1, L.K = C0, C1, v.numel() // (C0 * C1)
            L.C0p, L.C1p, L.splits = dwt.shape[2], dwt.shape[3], dwt.shape[0]
            if remap is not None:
                wide, slots = remap
                L.C1p = dwt.shape[3] // wide
                L.nA, L.nB = wide, dwt.shape[1]
                for k, sl in enumerate(slots):
                    L.tapsA[k] = sl
        call("rave_weight_norm_bwd_multi", len(chunk), arr, stream_ptr())
    return outs


# ----------------------------------------------------------------------------------------------
# hybrid configuration: mel front end, GRU
# ----------------------------------------------------------------------------------------------

def mel_log1p(X, band, weights, n_mels, scale, batch, channels):
    """log1p(scale * |X|^2 @ fb) of the complex STFT X [B*C, F, bins], last frame dropped -> [B, C*n_mels, F-1]
    (rave_mel_log1p_fwd; forward only).  `band` [n_mels, 3] int32 (lo, hi, offset into `weights`)."""
    N, F, bins = X.shape
    X = X.contiguous()
    out = torch.empty(batch, channels * n_mels, F - 1, dtype=torch.float32, device=X.device)
    call("rave_mel_log1p_fwd", ptr(torch.view_as_real(X)), ptr(band), ptr(weights), ptr(out), N, F, bins, n_mels,
         weights.numel(), float(scale), stream_ptr())
    return out


class MelLog1pFn(torch.autograd.Function):
    """mel_log1p with a gradient with respect to X (rave_mel_log1p_bwd): the receptive-field probe of a mel-input model
    differentiates through the front end."""

    @staticmethod
    def forward(ctx, X, band, weights, n_mels, scale, batch, channels):
        X = X.contiguous()
        ctx.save_for_backward(X, band, weights)
        ctx.dims = (n_mels, float(scale))
        return mel_log1p(X, band, weights, n_mels, scale, batch, channels)

    @staticmethod
    def backward(ctx, dy):
        X, band, weights = ctx.saved_tensors
        n_mels, scale = ctx.dims
        N, F, bins = X.shape
        dX = torch.empty_like(X)
        call("rave_mel_log1p_bwd", ptr(torch.view_as_real(X)), ptr(band), ptr(weights), ptr(_f32c(dy)),
             ptr(torch.view_as_real(dX)), N, F, bins, n_mels, weights.numel(), scale, stream_ptr())
        return dX, None, None, None, None, None, None


def _dptr(t, offset=0):
    """Device pointer of contiguous fp32 `t` plus `offset` elements."""
    return ptr(t) + 4 * offset


def gemm_f32(A, sam, sak, Bm, sbk, sbn, M, N, K, out, ldc, bias=None, rowsum=None, a_off=0, b_off=0):
    """out[m][n] = sum_k A(m, k) B(k, n) (+ bias[n]) over element strides (rave_gemm_f32); rowsum[m] = sum_k A(m, k)."""
    S = int(_lib.load().rave_gemm_f32_splits(M, N, K))
    ws = torch.empty(S * (M * N + M), dtype=torch.float32, device=out.device) if S > 1 else None
    call("rave_gemm_f32", _dptr(A, a_off), sam, sak, _dptr(Bm, b_off), sbk, sbn, ptr(bias), ptr(out), ldc, ptr(rowsum),
         M, N, K, ptr(ws), S, stream_ptr())


class GruLayerFn(torch.autograd.Function):
    """One nn.GRU layer (batch_first, h0 = 0) on x [B, T, I]: the input projection for all t as one GEMM, the recurrence
    as one persistent launch (rave_gru_fwd); backward = the reverse-time recurrence (rave_gru_bwd) producing the gate
    gradients, then dx, dW_ih, dW_hh and both bias gradients as GEMMs over the B*T rows."""

    @staticmethod
    def forward(ctx, x, w_ih, w_hh, b_ih, b_hh):
        x, w_ih, w_hh, b_ih, b_hh = (_f32c(t) for t in (x, w_ih, w_hh, b_ih, b_hh))
        B, T, I = x.shape
        G, H = w_hh.shape
        gi = torch.empty(B, T, G, dtype=torch.float32, device=x.device)
        gemm_f32(x, I, 1, w_ih, 1, I, B * T, G, I, gi, G, bias=b_ih)
        h = torch.empty(B, T, H, dtype=torch.float32, device=x.device)
        need = any(ctx.needs_input_grad)
        save = torch.empty(B, T, 5, H, dtype=torch.float32, device=x.device) if need else None
        call("rave_gru_fwd", ptr(gi), ptr(w_hh), ptr(b_hh), ptr(h), ptr(save), B, T, H, stream_ptr())
        if need:
            ctx.save_for_backward(x, w_ih, w_hh, save)
        return h

    @staticmethod
    def backward(ctx, dh):
        x, w_ih, w_hh, save = ctx.saved_tensors
        B, T, I = x.shape
        G, H = w_hh.shape
        dh = _f32c(dh)
        dgi = torch.empty(B, T, G, dtype=torch.float32, device=x.device)
        dgh = torch.empty(B, T, G, dtype=torch.float32, device=x.device)
        call("rave_gru_bwd", ptr(dh), ptr(save), ptr(w_hh), ptr(dgi), ptr(dgh), B, T, H, stream_ptr())
        dx = dw_ih = dw_hh = db_ih = db_hh = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty(B, T, I, dtype=torch.float32, device=x.device)
            gemm_f32(dgi, G, 1, w_ih, I, 1, B * T, I, G, dx, I)
        if any(ctx.needs_input_grad[1:]):
            dw_ih = torch.empty(G, I, dtype=torch.float32, device=x.device)
            dw_hh = torch.empty(G, H, dtype=torch.float32, device=x.device)
            db_ih = torch.empty(G, dtype=torch.float32, device=x.device)
            db_hh = torch.empty(G, dtype=torch.float32, device=x.device)
            gemm_f32(dgi, 1, G, x, I, 1, G, I, B * T, dw_ih, I, rowsum=db_ih)
            gemm_f32(dgh, 1, G, save, 5 * H, 1, G, H, B * T, dw_hh, H, rowsum=db_hh, b_off=4 * H)   # h_prev slot
        return dx, dw_ih, dw_hh, db_ih, db_hh


def gru(x, rnn):
    """nn.GRU(batch_first=True) `rnn` applied to channel-first x [B, C, T] -> [B, H, T] (rave/blocks.py:308-313), one
    GruLayerFn per layer.  fp32 in every precision mode: the recurrence compounds rounding."""
    if (not rnn.batch_first or rnn.bidirectional or not rnn.bias or rnn.proj_size or
            (rnn.dropout and rnn.training and rnn.num_layers > 1)):
        raise _lib.RaveB200Error("gru: only unidirectional, biased, batch-first nn.GRU without dropout is on the hot path")
    h = x.transpose(1, 2).contiguous()
    for l in range(rnn.num_layers):
        h = GruLayerFn.apply(h, getattr(rnn, f"weight_ih_l{l}"), getattr(rnn, f"weight_hh_l{l}"),
                             getattr(rnn, f"bias_ih_l{l}"), getattr(rnn, f"bias_hh_l{l}"))
    return h.transpose(1, 2)


# ----------------------------------------------------------------------------------------------
# latent prior (csrc/prior.cu).  `cl` = True: channel-last streams with bf16 operands (wgmma engine); False: [B, C, T]
# fp32 (parity path).
# ----------------------------------------------------------------------------------------------

def prior_latent_classes(z, eps, latent_mean, latent_pca, D, R):
    """Encoder output z [B, 2L, T] and eps [B, L, T] -> int32 classes [B, T - D + 1, D] (include/rave_b200.h)."""
    z, eps, latent_mean, latent_pca = _f32c(z), _f32c(eps), _f32c(latent_mean), _f32c(latent_pca)
    B, L2, T = z.shape
    cls = torch.empty(B, T - D + 1, D, dtype=torch.int32, device=z.device)
    call("rave_prior_latent_classes", ptr(z), ptr(eps), ptr(latent_mean), ptr(latent_pca), ptr(cls), B, L2 // 2, T, D,
         R, stream_ptr())
    return cls


def _stream_shape(B, T, C, cl):
    return (B, T, C) if cl else (B, C, T)


def prior_embed_fwd(cls, w, bias, cl, slope=0.2):
    """pre_net + LeakyReLU on class indices: (fp32 stream, bf16 channel-last operand if cl else None)."""
    B, Tp, D = cls.shape
    Cout, R, K = w.shape
    out = torch.empty(_stream_shape(B, Tp, Cout, cl), dtype=torch.float32, device=w.device)
    op = torch.empty(B, Tp, Cout, dtype=torch.bfloat16, device=w.device) if cl else None
    call("rave_prior_embed_fwd", ptr(cls), ptr(_f32c(w)), ptr(_f32c(bias)), ptr(out), ptr(op), B, Tp, D, R, Cout, K,
         int(cl), float(slope), stream_ptr())
    return out, op


def prior_embed_wgrad(cls, dout, x, w_shape, cl, slope=0.2):
    """(dw [Cout, R, K], dbias [Cout]) of prior_embed_fwd from the fp32 gradient of its output; x = its operand
    (cl) or fp32 stream (LeakyReLU')."""
    B, Tp, D = cls.shape
    Cout, R, K = w_shape
    dw = torch.empty(w_shape, dtype=torch.float32, device=dout.device)
    db = torch.empty(Cout, dtype=torch.float32, device=dout.device)
    call("rave_prior_embed_wgrad", ptr(cls), ptr(_f32c(dout)), ptr(x), ptr(dw), ptr(db), B, Tp, D, R, Cout, K, int(cl),
         float(slope), stream_ptr())
    return dw, db


def _gate_dims(h, cl):
    if cl:
        B, T, C2 = h.shape
    else:
        B, C2, T = h.shape
    return B, C2 // 2, T


def gate_fwd(h, cl):
    """sigmoid(h[:, :C]) * tanh(h[:, C:]) over the channel axis of h (bf16 channel-last if cl, else fp32 [B, 2C, T])."""
    B, C, T = _gate_dims(h, cl)
    g = torch.empty(_stream_shape(B, T, C, cl), dtype=h.dtype, device=h.device)
    call("rave_gate_fwd", ptr(h), ptr(g), B, C, T, int(cl), stream_ptr())
    return g


def gate_bwd(dg, h, cl):
    B, C, T = _gate_dims(h, cl)
    dh = torch.empty_like(h)
    call("rave_gate_bwd", ptr(_f32c(dg)), ptr(h), ptr(dh), B, C, T, int(cl), stream_ptr())
    return dh


class GateFn(torch.autograd.Function):
    """The gated unit of the prior's ResidualBlock on [B, 2C, T] fp32 (dense Prior.forward)."""

    @staticmethod
    def forward(ctx, h):
        h = _f32c(h)
        ctx.save_for_backward(h)
        return gate_fwd(h, False)

    @staticmethod
    def backward(ctx, dg):
        (h,) = ctx.saved_tensors
        return gate_bwd(dg, h, False)


def gate(h):
    return GateFn.apply(h)


def _head_dims(x, cls, cl):
    B, Tp, D = cls.shape
    Cin = x.shape[2] if cl else x.shape[1]
    return B, Tp, D, Cin


def prior_head_ce_fwd(x, w, bias, cls, cl, slope=0.2):
    """Mean cross-entropy of post_net.2 on LeakyReLU(x) against the next frame's classes (0-d fp32 tensor)."""
    B, Tp, D, Cin = _head_dims(x, cls, cl)
    R = w.shape[0] // D
    loss = torch.empty((), dtype=torch.float32, device=x.device)
    call("rave_prior_head_ce_fwd", ptr(x), ptr(_f32c(w)), ptr(_f32c(bias)), ptr(cls), ptr(loss), B, Tp, D, R, Cin,
         int(cl), float(slope), stream_ptr())
    return loss


def prior_head_ce_bwd(x, w, bias, cls, gloss, cl, slope=0.2):
    """(d loss / d x in x's dtype and layout, dw like w, dbias) times the device scalar gloss."""
    B, Tp, D, Cin = _head_dims(x, cls, cl)
    R = w.shape[0] // D
    dx = torch.empty_like(x)
    dw = torch.empty_like(w)
    db = torch.empty(w.shape[0], dtype=torch.float32, device=x.device)
    call("rave_prior_head_ce_bwd", ptr(x), ptr(_f32c(w)), ptr(_f32c(bias)), ptr(cls), ptr(_f32c(gloss)), ptr(dx),
         ptr(dw), ptr(db), B, Tp, D, R, Cin, int(cl), float(slope), stream_ptr())
    return dx, dw, db


def prior_sample(params, dilation_cycle, prefix, uniform, n_frames, R, argmax, return_logits):
    """Cached sampling of the prior (csrc/prior_sample.cu) from its trained parameters (Prior._trained_parameters order):
    int32 prefix [B, P, D], fp32 uniform [B, n_frames, D] (None with argmax) -> (classes [B, n_frames, D] int32,
    logits [B, n_frames - 1, D, R] or None)."""
    import ctypes
    n_layers = (len(params) - 6) // 6
    C, _, K = params[0].shape
    Sk = params[-4].shape[0]
    B, P, D = prefix.shape
    prefix = prefix.contiguous()
    if prefix.dtype != torch.int32:
        raise _lib.RaveB200Error(f"prior_sample: prefix must be int32, got {prefix.dtype}")
    ps = [_f32c(p) for p in params]
    arr = (ctypes.c_void_p * len(ps))(*[ptr(p) for p in ps])
    nbytes = int(_lib.load().rave_prior_sample_workspace_bytes(B, n_layers, dilation_cycle, C, Sk, K, D))
    if nbytes < 0:
        raise _lib.RaveB200Error(f"prior_sample: bad shape (B {B}, {n_layers} layers, C {C}, Sk {Sk}, K {K}, D {D})")
    work = torch.empty(nbytes, dtype=torch.uint8, device=prefix.device)
    cls = torch.empty(B, n_frames, D, dtype=torch.int32, device=prefix.device)
    logits = (torch.empty(B, max(n_frames - 1, 0), D, R, dtype=torch.float32, device=prefix.device)
              if return_logits else None)
    call("rave_prior_sample", arr, n_layers, dilation_cycle, C, Sk, K, R, D, ptr(prefix), P,
         ptr(None if uniform is None else _f32c(uniform)), n_frames, B, int(argmax), ptr(cls), ptr(logits), ptr(work),
         nbytes, stream_ptr())
    return cls, logits


def prior_classes_to_latent(classes, dither, noise, latent_pca, latent_mean, R):
    """int32 classes [B, T, D], dither [B, T, D], noise [B, L - D, T - D + 1] -> RAVE latent z [B, L, T - D + 1]
    (QuantizedNormal.decode, DiagonalShift.inverse and VariationalPrior.pre_process_latent in one kernel)."""
    B, T, D = classes.shape
    L = latent_pca.shape[0]
    if classes.dtype != torch.int32:
        raise _lib.RaveB200Error(f"prior_classes_to_latent: classes must be int32, got {classes.dtype}")
    z = torch.empty(B, L, T - D + 1, dtype=torch.float32, device=classes.device)
    call("rave_prior_classes_to_latent", ptr(classes.contiguous()), ptr(_f32c(dither)),
         ptr(None if noise is None or L == D else _f32c(noise)), ptr(_f32c(latent_pca)), ptr(_f32c(latent_mean)),
         ptr(z), B, T, D, L, R, stream_ptr())
    return z


# ----------------------------------------------------------------------------------------------
# Training-batch transforms (rave_b200/transforms.py)
# ----------------------------------------------------------------------------------------------

def augment(raw, draws, key, out, noise=None, normalize=False, derivative=False):
    """raw [B, C, L] int16 / fp32 -> out [B, C, N] fp32 with rave_augment (include/rave_b200.h): draws [B, 4] fp64,
    key [2] int64, noise [B, C, N] fp64 or None.  Shapes and dtypes are the caller's to check."""
    B, C, L = raw.shape
    call("rave_augment", ptr(raw), int(raw.dtype == torch.int16), B, C, L, out.shape[-1], ptr(draws), ptr(key),
         ptr(noise), ptr(out), int(normalize), int(derivative), stream_ptr())
    return out


# ----------------------------------------------------------------------------------------------
# Exponential moving average of parameters (rave_b200/ema.py)
# ----------------------------------------------------------------------------------------------

def ema_chunk_elems() -> int:
    """Elements per chunk of the EMA table's chunk prefix (include/rave_b200.h)."""
    return int(_lib.load().rave_ema_chunk_elems())


def ema_update(table, n_tensors, n_chunks, state, factor):
    """rave_ema_update over the tensors of `table` [4T + 1] int64: ema = ema * factor + p * (1 - factor) in float32,
    1 - factor in double as Python computes it; a tensor whose state flag is 0 is copied instead."""
    call("rave_ema_update", ptr(table), int(n_tensors), int(n_chunks), ptr(state), float(factor), 1.0 - float(factor),
         stream_ptr())


def ema_swap(table, n_tensors, n_chunks):
    """rave_ema_swap: exchange the parameters and the averages of `table` in place."""
    call("rave_ema_swap", ptr(table), int(n_tensors), int(n_chunks), stream_ptr())

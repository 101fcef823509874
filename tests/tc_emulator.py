"""TEST DOUBLE: torch emulation of the tensor-core entry points' documented semantics (include/rave_b200.h).  Not part
of the product.  Two users:

- tests/test_engine_cpu.py installs it in place of rave_b200.ops to exercise the host-side engine logic (planning, phase
  decomposition, pitches, the explicit backward) without a GPU.  Default: fp32 arithmetic on the inputs' device.
- tests/launch_checker.py evaluates it under `compute(torch.float64)` on the snapshotted operands of every launch the
  engine issues on the GPU (tests/test_gpu_launch_replay.py), as the high-precision reference of each kernel.

OPERAND_DTYPE is the type operands / bf16 outputs are rounded to; COMPUTE_DTYPE the type every sum is formed in.  Every
entry point computes on its inputs' device."""
import contextlib

import torch
import torch.nn.functional as F


OPERAND_DTYPE = torch.bfloat16
COMPUTE_DTYPE = torch.float32


@contextlib.contextmanager
def compute(dtype=torch.float64):
    """Evaluate every entry point in `dtype` inside the block."""
    global COMPUTE_DTYPE
    saved = COMPUTE_DTYPE
    COMPUTE_DTYPE = dtype
    try:
        yield
    finally:
        COMPUTE_DTYPE = saved


def _c(t):
    return t.to(COMPUTE_DTYPE)


def _dev(t):
    return t.device


def _zeros(like, *shape):
    return torch.zeros(*shape, dtype=COMPUTE_DTYPE, device=like.device)


def _bf16(t):
    return t.to(OPERAND_DTYPE)


def conv1d_tc(xa_cl, wt, bias=None, res_cl=None, stride=1, dil=1, pad=(0, 0), act=0, slope=0.2,
              want_f32=True, want_act=False, out_f32=None, out_act=None, out_rows=0, out_row_stride=0,
              out_row_offset=0, Lout=None, res_bf16=None, dact_src=None, Lin=None, res_act=None, res_slope=0.2,
              fm_d=None, fm_partner=None, x3=False, act_cs=0):
    if x3:
        return _conv1d_tc_x3(xa_cl, wt, bias, res_cl, stride, dil, pad, act, slope, out_f32, out_act, out_rows, Lout,
                             Lin, res_act, res_slope, act_cs, out_row_stride, out_row_offset)
    B, in_pitch, Cin = xa_cl.shape
    Lin = in_pitch if Lin is None else Lin
    K, Cout, _ = wt.shape
    assert in_pitch >= -(-Lin // stride) * stride
    if in_pitch > Lin:
        assert float(xa_cl[:, Lin:].float().abs().max()) == 0.0, "slack rows must be zero"
    x = _c(xa_cl[:, :Lin]).permute(0, 2, 1)                         # [B, Cin, Lin]
    w = _c(wt).permute(1, 2, 0)                                      # [Cout, Cin, K]
    if Lout is None:
        Lout = (Lin + pad[0] + pad[1] - dil * (K - 1) - 1) // stride + 1
    # rows l*stride + k*dil - pad_l, zero outside [0, Lin)
    need = (Lout - 1) * stride + (K - 1) * dil + 1
    pl = pad[0]
    if pl >= 0:
        xp = F.pad(x, (pl, max(0, need - pl - Lin)))
    else:
        xp = F.pad(x[..., -pl:], (0, max(0, need - (Lin + pl))))
    xp = xp[..., :max(need, 1)]
    if xp.shape[-1] < need:
        xp = F.pad(xp, (0, need - xp.shape[-1]))
    y = F.conv1d(xp, w, None, stride, 0, dil)[..., :Lout]            # [B, Cout, Lout]
    v = y.permute(0, 2, 1)                                           # [B, Lout, Cout]
    if bias is not None:
        v = v + _c(bias)
    rows = out_rows if out_rows else Lout
    idx = out_row_index(Lout, out_row_stride, out_row_offset, _dev(xa_cl))
    if dact_src is not None:
        sgn = torch.signbit(_c(dact_src[:, idx]))
        v = torch.where(sgn, v * slope, v)
    if fm_d is not None and fm_partner is not None:      # fake half only: partner = the real rows
        fd = _c(fm_d)
        a = _c(dact_src[:, idx])
        ar = _c(fm_partner[:, idx])
        hf, hr = torch.where(a > 0, a, a / slope), torch.where(ar > 0, ar, ar / slope)
        v = v - fd[0] * torch.sign(hr - hf)
    elif fm_d is not None:
        fd = _c(fm_d)
        a = _c(dact_src[:, idx])
        h = torch.where(a > 0, a, a / slope)
        hr, hf = h[:B // 2], h[B // 2:]
        sd = torch.sign(hr - hf)
        v = v + torch.cat([fd[0] * sd + fd[1] * torch.sign(hr), -fd[0] * sd], 0)
    if res_bf16 is not None:
        v = v + _c(res_bf16[:, idx])
    if res_act is not None:
        ra = _c(res_act[:, idx])
        v = v + torch.where(ra > 0, ra, ra / res_slope)
    if res_cl is not None:
        v = v + _c(res_cl[:, idx])
    if want_f32 and out_f32 is None:
        out_f32 = _zeros(xa_cl, B, rows, Cout)
    if want_act and out_act is None:
        out_act = torch.zeros(B, rows, Cout, dtype=OPERAND_DTYPE, device=_dev(xa_cl))
    if out_f32 is not None:
        out_f32[:, idx] = v.to(out_f32.dtype)
    if out_act is not None:
        a = F.leaky_relu(v, slope) if act == 1 else v
        out_act[:, idx] = _bf16(a).to(out_act.dtype)
    return out_f32, out_act


def out_row_index(Lout, out_row_stride=0, out_row_offset=0, device=None):
    """Rows of a [B][out_rows][C] output that positions 0 .. Lout-1 land in: l * out_row_stride + out_row_offset."""
    return torch.arange(Lout, device=device) * (out_row_stride if out_row_stride else 1) + out_row_offset


def _split(v):
    hi = v.to(torch.bfloat16)
    lo = (v - hi.to(v.dtype)).to(torch.bfloat16)
    return hi, lo


def _conv1d_tc_x3(xa_cl, wt, bias, res_cl, stride, dil, pad, act, slope, out_f32, out_act, out_rows, Lout, Lin, res_act,
                  res_slope, act_cs, out_row_stride=0, out_row_offset=0):
    """Split-operand semantics of rave_conv1d_tc_fwd_x3 (include/rave_b200.h): rows [hi | lo], weights [2][K][Cout][Cin],
    hi*hi + lo*hi + hi*lo accumulated in fp32; out_act positions are [hi | lo] pairs of act_cs channels."""
    B, in_pitch, C2 = xa_cl.shape
    Cin = C2 // 2
    K = wt.shape[0] // 2
    Cout = wt.shape[1]
    a_hi, a_lo = xa_cl[..., :Cin], xa_cl[..., Cin:]
    w_hi, w_lo = wt[:K], wt[K:]

    def run(a, w):
        o, _ = conv1d_tc(a.contiguous(), w, None, None, stride, dil, pad, 0, slope, want_f32=True, want_act=False,
                         Lout=Lout, Lin=Lin)
        return o
    v = run(a_hi, w_hi) + run(a_lo, w_hi) + run(a_hi, w_lo)          # [B, Lout, Cout]
    LoutE = v.shape[1]
    rows = out_rows if out_rows else LoutE
    idx = out_row_index(LoutE, out_row_stride, out_row_offset, _dev(xa_cl))
    if bias is not None:
        v = v + _c(bias)
    if res_act is not None:
        ra = _c(res_act[:, idx, :Cout]) + _c(res_act[:, idx, Cout:])
        v = v + torch.where(ra > 0, ra, ra / res_slope)
    if res_cl is not None:
        v = v + _c(res_cl[:, idx])
    if out_f32 is not None:
        out_f32[:, idx] = v.to(out_f32.dtype)
    if out_act is not None:
        a = F.leaky_relu(v, slope) if act == 1 else v
        cs = act_cs if act_cs else Cout
        hi, lo = _split(a)
        q = Cout // cs
        pair = torch.stack([hi.reshape(B, LoutE, q, cs), lo.reshape(B, LoutE, q, cs)], 3)    # [B, Lout, q, 2, cs]
        out_act[:, idx] = pair.reshape(B, LoutE, 2 * Cout).to(out_act.dtype)
    return out_f32, out_act


def dilated_unit_tc_supported(C, L):
    return C in (96, 192, 384) and L >= 8


def dilated_unit_tc(xa_cl, w3t, w1t, dil, pad_l, slope_in, slope_mid, act_out, slope_out, L=None, want_a1=False,
                    out_f32=None, out_act=None):
    """Semantics of rave_dilated_unit_tc_fwd: the two per-layer launches back to back, the intermediate rounded to the
    operand type exactly as the kernel rounds it before the second GEMM."""
    L = xa_cl.shape[1] if L is None else L
    a1 = unit_stage1(xa_cl, w3t, dil, pad_l, slope_mid, L)
    unit_stage2(a1, xa_cl, w1t, slope_in, act_out, slope_out, L, out_f32, out_act)
    return (a1 if want_a1 else None), out_f32, out_act


def unit_stage1(xa_cl, w3t, dil, pad_l, slope_mid, L, out_act=None):
    """a1 [B, pitch, C] = operand-type LeakyReLU(conv3(xa, dil)) over rows [0, L), zero slack rows."""
    B, pitch, C = xa_cl.shape
    if out_act is None:
        out_act = torch.zeros(B, pitch, C, dtype=OPERAND_DTYPE, device=_dev(xa_cl))
    _, a1 = conv1d_tc(xa_cl, w3t, None, None, 1, dil, (pad_l, 2 * dil - pad_l), 1, slope_mid, want_f32=False,
                      want_act=True, out_act=out_act, out_rows=pitch, Lout=L, Lin=L)
    if pitch > L:
        a1[:, L:] = 0
    return a1


def unit_stage2(a1, xa_cl, w1t, slope_in, act_out, slope_out, L, out_f32=None, out_act=None):
    """The unit's outputs from its intermediate a1: conv1x1(a1) + unleaky(xa) (the residual), rows [0, L)."""
    return conv1d_tc(a1, w1t, None, None, 1, 1, (0, 0), act_out, slope_out, want_f32=False, want_act=False,
                     out_f32=out_f32, out_act=out_act, out_rows=xa_cl.shape[1], Lout=L, Lin=L, res_act=xa_cl,
                     res_slope=slope_in)


def ncl_to_cl_x3(x):
    xt = x.permute(0, 2, 1).contiguous()
    hi, lo = _split(xt)
    return torch.cat([hi, lo], -1)


def conv1d_tc_wgrad(P_cl, Q_cl, K, stride=1, dil=1, pad_l=0, Lp=None, Lq=None, dbias=None):
    B, p_pitch, Cm = P_cl.shape
    _, q_pitch, Cn = Q_cl.shape
    Lp = p_pitch if Lp is None else Lp
    Lq = q_pitch if Lq is None else Lq
    P = P_cl[:, :Lp].to(COMPUTE_DTYPE)
    if dbias is not None:
        dbias += P.sum((0, 1))
    Q = Q_cl[:, :q_pitch].to(COMPUTE_DTYPE)
    if q_pitch > Lq:
        assert float(Q[:, Lq:].abs().max()) == 0.0
    S = 2                                  # two "row slices": the batch halves
    dwt = _zeros(P, S, K, Cm, Cn)
    l = torch.arange(Lp, device=P.device)
    half = (B + 1) // 2
    for k in range(K):
        r = l * stride + k * dil - pad_l
        ok = (r >= 0) & (r < Lq)
        if ok.any():
            dwt[0, k] = torch.einsum("blm,bln->mn", P[:half, l[ok]], Q[:half, r[ok]])
            if B > half:
                dwt[1, k] = torch.einsum("blm,bln->mn", P[half:, l[ok]], Q[half:, r[ok]])
    return dwt


def weight_prep_tc(v, g, tapsA, tapsB, C0p, C1p):
    C0, C1 = v.shape[0], v.shape[1]
    v3 = v.reshape(C0, C1, -1)
    norm = None
    w = v3
    if g is not None:
        norm = v3.reshape(C0, -1).norm(2, 1)
        w = v3 * (g.reshape(C0, 1, 1) / norm.reshape(C0, 1, 1))
    wp = F.pad(w, (0, 1, 0, C1p - C1, 0, C0p - C0))          # extra all-zero tap: index -1
    outA = _bf16(wp[:, :, tapsA].permute(2, 0, 1).contiguous()) if tapsA else None
    outB = _bf16(wp[:, :, tapsB].permute(2, 1, 0).contiguous()) if tapsB else None
    return norm, outA, outB


def weight_norm_bwd_tapmajor(dwt, v, g, norm):
    C0, C1 = v.shape[0], v.shape[1]
    dw = dwt.sum(0)[:, :C0, :C1].permute(1, 2, 0).reshape(v.shape)
    if g is None:
        return dw.contiguous(), None
    v2 = v.reshape(C0, -1)
    dw2 = dw.reshape(C0, -1)
    dot = (dw2 * v2).sum(1)
    n = norm
    gg = g.reshape(C0)
    dv = (gg / n).unsqueeze(1) * (dw2 - v2 * (dot / (n * n)).unsqueeze(1))
    dg = (dot / n).reshape(g.shape)
    return dv.reshape(v.shape), dg


def ncl_to_cl(x, act=0, slope=0.2, alpha=None, want_bf16=True, want_f32=False):
    xt = x.permute(0, 2, 1).contiguous()
    a = F.leaky_relu(xt, slope) if act == 1 else xt
    return (_bf16(a) if want_bf16 else None), (xt if want_f32 else None)


def cl_to_ncl(x_cl):
    return x_cl.permute(0, 2, 1).contiguous()


def weight_norm_raw(v, g):
    C0 = v.shape[0]
    norm = v.reshape(C0, -1).norm(2, 1)
    shape = (C0,) + (1,) * (v.dim() - 1)
    return v * (g.reshape(shape) / norm.reshape(shape)), norm


def conv1d_c1(x_rows, w, bias, Lin, stride, pad, act, slope, out_f32=None, out_act=None, Lout=None):
    R, x_pitch = x_rows.shape
    Cout = w.shape[0]
    K = w.numel() // Cout
    x = x_rows[:, :Lin].unsqueeze(1)
    need = (Lout - 1) * stride + K
    xp = F.pad(x, (pad[0], max(0, need - pad[0] - Lin)))
    y = F.conv1d(xp, w.reshape(Cout, 1, K), bias, stride)[..., :Lout].permute(0, 2, 1)
    if out_f32 is not None:
        out_f32[:, :Lout] = y
    if out_act is not None:
        out_act[:, :Lout] = _bf16(F.leaky_relu(y, slope) if act == 1 else y)
    return out_f32, out_act


def conv1d_c1_wgrad(g_cl, x_rows, Cout, K, Lin, Lout, stride, pad_l):
    R = g_cl.shape[0]
    g = g_cl[:, :Lout, :Cout].to(COMPUTE_DTYPE)
    dwt = _zeros(g, 3, K, Cout, 1)                         # 3 "slices": rows split arbitrarily
    l = torch.arange(Lout, device=g.device)
    for k in range(K):
        pos = l * stride + k - pad_l
        ok = (pos >= 0) & (pos < Lin)
        if ok.any():
            xv = x_rows[:, pos[ok]]                          # [R, n]
            full = torch.einsum("rlc,rl->c", g[:, l[ok]], xv)
            dwt[0, k, :, 0] = 0.25 * full
            dwt[1, k, :, 0] = 0.5 * full
            dwt[2, k, :, 0] = 0.25 * full
    return dwt


def conv1d_c1_dgrad(g_cl, w, x_pitch, Lin, Lout, stride, pad_l):
    R = g_cl.shape[0]
    Cout = w.shape[0]
    K = w.numel() // Cout
    g = g_cl[:, :Lout, :Cout].to(COMPUTE_DTYPE).permute(0, 2, 1)               # [R, Cout, Lout]
    full = F.conv_transpose1d(g, w.reshape(Cout, 1, K), None, stride)  # [R, 1, (Lout-1)*s + K]
    dx = _zeros(g, R, x_pitch)
    seg = full[:, 0, pad_l:pad_l + Lin]
    dx[:, :seg.shape[1]] = seg
    return dx


def colsum_bf16(g_cl, L, C):
    return g_cl[:, :L, :C].to(COMPUTE_DTYPE).sum((0, 1))


def _c1_rows(src, Lin, period, pool):
    """rows [Bs*period, Lin] derived from src [Bs, T] exactly like the reference: fold (zero pad to a multiple of the
    period) or repeated average pooling."""
    Bs, T = src.shape
    if period > 1:
        xp = F.pad(src, (0, Lin * period - T))
        return xp.reshape(Bs, Lin, period).permute(0, 2, 1).reshape(Bs * period, Lin)
    if pool > 1:
        return src[:, :Lin * pool].reshape(Bs, Lin, pool).mean(-1)
    return src[:, :Lin]


def im2col_c1(src, Lin, Lout, out_pitch, K, stride, pad_l, period=1, pool=1):
    x_rows = _c1_rows(src.to(COMPUTE_DTYPE), Lin, period, pool)
    R = x_rows.shape[0]
    X = _zeros(x_rows, R, out_pitch, 16)
    l = torch.arange(Lout, device=src.device)
    for k in range(K):
        pos = l * stride + k - pad_l
        ok = (pos >= 0) & (pos < Lin)
        X[:, l[ok], k] = x_rows[:, pos[ok]]
    return _bf16(X)


def gather_c1(P_cl, src_shape, Lin, Lout, K, stride, pad_l, period=1, pool=1, batch0=0):
    if batch0:
        part = gather_c1(P_cl, (src_shape[0] - batch0, src_shape[1]), Lin, Lout, K, stride, pad_l, period, pool)
        return torch.cat([_zeros(part, batch0, src_shape[1]), part], 0)
    R = P_cl.shape[0]
    Bs, T = src_shape
    P = _c(P_cl)
    dx = _zeros(P, R, Lin)
    t = torch.arange(Lin, device=P.device)
    for k in range(K):
        q = t + pad_l - k
        ok = (q >= 0) & (q % stride == 0) & (q // stride < Lout)
        dx[:, t[ok]] += P[:, (q[ok] // stride), k]
    # adjoint of _c1_rows
    with torch.enable_grad():
        src = _zeros(P, Bs, T).requires_grad_(True)
        rows = _c1_rows(src, Lin, period, pool)
        (g,) = torch.autograd.grad(rows, src, dx)
    return g.detach()


def im2col_cin(src, Lin, Lout, out_pitch, K, stride, pad_l, period=1, pool=1):
    """im2col_c1 of each of the src [Bs, cin, T] channels side by side: X[r, l, c*K + k], zero up to W = 16 or 32."""
    Bs, cin, T = src.shape
    W = 16 if cin * K <= 16 else 32
    X = torch.cat([im2col_c1(src[:, c], Lin, Lout, out_pitch, K, stride, pad_l, period, pool)[..., :K]
                   for c in range(cin)], -1)
    return F.pad(X, (0, W - cin * K))


def gather_cin(P_cl, src_shape, Lin, Lout, K, stride, pad_l, period=1, pool=1, batch0=0):
    """The adjoint of im2col_cin: dsrc [Bs, cin, T]."""
    Bs, cin, T = src_shape
    return torch.stack([gather_c1(P_cl[..., c * K:(c + 1) * K], (Bs, T), Lin, Lout, K, stride, pad_l, period, pool,
                                  batch0) for c in range(cin)], 1)


def _unleaky(a, slope):
    return torch.where(a > 0, a, a / slope)


def fm_stats(a_cl, stats_row, L, slope):
    B2 = a_cl.shape[0]
    h = _unleaky(a_cl[:, :L].to(COMPUTE_DTYPE), slope)
    hr, hf = h[:B2 // 2], h[B2 // 2:]
    stats_row[0] += (hr - hf).abs().sum()
    stats_row[1] += hr.abs().sum()


def fm_grad(a_cl, dstats_row, L, slope):
    B2 = a_cl.shape[0]
    h = _unleaky(a_cl.to(COMPUTE_DTYPE), slope)
    hr, hf = h[:B2 // 2], h[B2 // 2:]
    sd = torch.sign(hr - hf)
    g = torch.cat([dstats_row[0] * sd + dstats_row[1] * torch.sign(hr), -dstats_row[0] * sd], 0)
    g[:, L:] = 0
    return _bf16(g)


def score_stats(score_cl, stats6, L):
    B2 = score_cl.shape[0]
    s = score_cl[:, :L, 0].to(COMPUTE_DTYPE)
    sr, sf = s[:B2 // 2], s[B2 // 2:]
    stats6.view(-1).add_(torch.stack([(sr - sf).abs().sum(), sr.abs().sum(), torch.relu(1 - sr).sum(),
                           torch.relu(1 + sf).sum(), sr.sum(), sf.sum()]))


def score_grad(score_cl, dstats6, L):
    B2, pitch, C = score_cl.shape
    s = score_cl[:, :L, 0].to(COMPUTE_DTYPE)
    sr, sf = s[:B2 // 2], s[B2 // 2:]
    d = dstats6.to(COMPUTE_DTYPE).reshape(-1)
    sd = torch.sign(sr - sf)
    gr = d[0] * sd + d[1] * torch.sign(sr) - d[2] * (sr < 1).to(COMPUTE_DTYPE) + d[4]
    gf = -d[0] * sd + d[3] * (sf > -1).to(COMPUTE_DTYPE) + d[5]
    g = torch.zeros(B2, pitch, C, dtype=torch.float32, device=score_cl.device)
    g[:B2 // 2, :L, 0] = gr
    g[B2 // 2:, :L, 0] = gf
    from rave_b200 import engine
    return g.to(engine.ACT_DTYPE)


def weight_prep_tc_multi(items, x3=False, into=None):
    """`into`: overwrite the (norm, outA, outB) tensors of an earlier call in place (engine.refresh_static_prep)."""
    if into is not None:
        fresh = weight_prep_tc_multi(items, x3=x3)
        for new, old in zip(fresh, into):
            for a, b in zip(new, old):
                if b is not None:
                    b.copy_(a)
        return into
    if not x3:
        return [weight_prep_tc(*it) for it in items]
    out = []
    saved = globals()["OPERAND_DTYPE"]
    globals()["OPERAND_DTYPE"] = torch.float32            # keep fp32, then split into [hi slabs | lo slabs]
    try:
        for it in items:
            norm, A, Bm = weight_prep_tc(*it)
            cat = lambda t: None if t is None else torch.cat(_split(t.to(COMPUTE_DTYPE)), 0)
            out.append((norm, cat(A), cat(Bm)))
    finally:
        globals()["OPERAND_DTYPE"] = saved
    return out


def weight_norm_bwd_multi(items):
    out = []
    for it in items:
        dwt, v, g, norm = it[:4]
        if len(it) > 4 and it[4] is not None:          # phase-wide buffer [S][J][C0p][wide*C1p] -> [S][K][C0p][C1p]
            wide, slots = it[4]
            S, J, C0p, W = dwt.shape
            C1p = W // wide
            d5 = dwt.reshape(S, J, C0p, wide, C1p)
            dwt = torch.stack([d5[:, sl // wide, :, sl % wide, :] for sl in slots], 1)
        out.append(weight_norm_bwd_tapmajor(dwt, v, g, norm))
    return out


def snake_cl_fwd(h_cl, alpha):
    al = alpha.detach().reshape(-1).to(COMPUTE_DTYPE)
    x = h_cl.to(COMPUTE_DTYPE)
    return _bf16(x + torch.sin(al * x) ** 2 / (al + 1e-9))


def snake_cl_bwd(ga_cl, h_cl, alpha, add=None, want_dalpha=True):
    al = alpha.detach().reshape(-1).to(COMPUTE_DTYPE)
    ae = al + 1e-9
    x, g = h_cl.to(COMPUTE_DTYPE), ga_cl.to(COMPUTE_DTYPE)
    s2 = torch.sin(2 * al * x)
    gh = g * (1 + al * s2 / ae)
    if add is not None:
        gh = gh + add.to(COMPUTE_DTYPE)
    dal = (g * (x * s2 / ae - torch.sin(al * x) ** 2 / (ae * ae))).reshape(-1, x.shape[-1]).sum(0) if want_dalpha else None
    return _bf16(gh), dal


def activation(x, act, slope=0.2, alpha=None):
    """ops.activation (fp32 elementwise kernel with its own autograd): plain torch here."""
    if act == 1:
        return F.leaky_relu(x, slope)
    if act == 2:
        al = alpha.reshape(1, -1, *([1] * (x.dim() - 2)))
        return x + torch.sin(al * x) ** 2 / (al + 1e-9)
    return x


def leaky_fm(x, slope):
    """ops.leaky_fm: LeakyReLU + the L1 feature-matching sums of the [real; fake] halves, plain torch autograd here."""
    a = F.leaky_relu(x, slope)
    h = a.shape[0] // 2
    return a, torch.stack([(a[:h] - a[h:]).abs().sum(), a[:h].abs().sum()])


def time_stack_nhwc(x, kt, pt, Cp, Fp):
    """ops.time_stack_nhwc: x [B, T, F, C] fp32 channel-last -> [(b t), Fp, Cp] operand rows holding the kt time-shifted
    copies of the channels side by side (zero outside the T steps, in the pad columns / channels); torch autograd."""
    B, T, Fq, C = x.shape
    xp = F.pad(x, (0, 0, 0, 0, pt, kt - 1 - pt))                             # zero time steps on both sides
    st = torch.cat([xp[:, dt:dt + T] for dt in range(kt)], dim=-1)          # [B, T, F, kt*C], channel = dt*C + c
    st = F.pad(st, (0, Cp - kt * C, 0, Fp - Fq))
    return _bf16(st.reshape(B * T, Fp, Cp))


def leaky_fm_stack(x, slope, T, Fp):
    """ops.leaky_fm_stack = leaky_fm + the next conv's time-stacked operand (kt = 3, pt = 1) from its output."""
    a, st = leaky_fm(x, slope)
    R2, Fq, C = x.shape
    return a, st, time_stack_nhwc(a.view(R2 // T, T, Fq, C), 3, 1, 3 * C, Fp)


def stft_frames(x, window, n_fft, hop):
    """ops.stft_frames: reflect pad (centred STFT) + frame + window, [N, T] -> [N, frames, n_fft]; torch autograd."""
    p = n_fft // 2
    xp = F.pad(x[:, None], (p, p), mode="reflect")[:, 0]
    return xp.unfold(-1, n_fft, hop) * window


def install(monkeypatch):
    from rave_b200 import ops
    for name in ("conv1d_tc", "conv1d_tc_wgrad", "weight_prep_tc", "weight_norm_bwd_tapmajor", "ncl_to_cl",
                 "cl_to_ncl", "weight_norm_raw", "conv1d_c1", "conv1d_c1_wgrad", "fm_stats", "fm_grad", "conv1d_c1_dgrad", "colsum_bf16", "im2col_c1", "gather_c1", "im2col_cin", "gather_cin",
                 "weight_prep_tc_multi",
                 "weight_norm_bwd_multi", "score_stats", "score_grad", "ncl_to_cl_x3", "dilated_unit_tc",
                 "dilated_unit_tc_supported", "snake_cl_fwd", "snake_cl_bwd", "activation", "leaky_fm", "time_stack_nhwc",
                 "leaky_fm_stack", "stft_frames"):
        monkeypatch.setattr(ops, name, globals()[name])

"""GPU: the wgmma conv engine against the CPU oracle evaluated on the SAME bf16-rounded operands
(so the only difference is fp32 accumulation order: tolerance 2e-5), and against the un-rounded fp32
oracle with the stated bf16-mode tolerance (1e-2 rel-L2 per conv)."""
import pytest
import torch

from oracle import rave_oracle as O
from tests.conftest import rel_l2

pytestmark = pytest.mark.gpu

TC_CASES = [
    # B, Cin, Cout, L, K, stride, dil, pad, bias, res
    (2, 64, 64, 256, 3, 1, 1, (1, 1), False, False),
    (2, 96, 96, 512, 3, 1, 3, (3, 3), False, True),
    (3, 96, 96, 384, 1, 1, 1, (0, 0), False, True),
    (2, 16, 96, 512, 7, 1, 1, (3, 3), False, False),
    (2, 96, 192, 512, 8, 4, 1, (3, 4), False, False),
    (4, 768, 1536, 64, 4, 2, 1, (1, 2), False, False),
    (5, 1536, 256, 32, 3, 1, 1, (1, 1), False, False),
    (2, 128, 1536, 32, 3, 1, 1, (1, 1), False, False),
    (2, 192, 192, 1000, 3, 1, 9, (9, 9), True, True),       # ragged length (not a multiple of 128)
    (2, 96, 32, 300, 7, 1, 1, (6, 0), True, False),          # causal padding
    (1, 32, 48, 40, 15, 4, 1, (7, 7), True, False),          # discriminator-like
    (3, 192, 384, 2048, 15, 4, 1, (7, 7), True, False),      # MSD layer
    (6, 128, 256, 700, 5, 4, 1, (2, 2), True, False),        # MPD layer, ragged
    (2, 64, 128, 640, 7, 1, 1, (3, 3), False, True),         # k7, one group of 7 taps
    (3, 96, 192, 1032, 15, 4, 1, (7, 7), False, False),      # Cin = 96: 64-byte swizzle spans
]


@pytest.mark.parametrize("case", TC_CASES)
def test_conv1d_tc_vs_oracle(case):
    from rave_b200 import ops
    B, Cin, Cout, L, K, stride, dil, pad, use_bias, use_res = case
    assert ops.conv1d_tc_supported(Cin, Cout, K, stride, dil)
    g = torch.Generator().manual_seed(hash(case) % (2 ** 31))
    x = torch.randn(B, Cin, L, generator=g)
    w = torch.randn(Cout, Cin, K, generator=g) / (Cin * K) ** 0.5
    bias = torch.randn(Cout, generator=g) if use_bias else None
    # oracle on bf16-rounded operands
    xa = O.leaky_relu(x, 0.2).bfloat16().float()
    wr = w.bfloat16().float()
    y_exact = O.conv1d(xa, wr, bias, stride, dil, pad)
    y_fp32 = O.conv1d(O.leaky_relu(x, 0.2), w, bias, stride, dil, pad)
    res = torch.randn(y_exact.shape, generator=g) if use_res else None
    if use_res:
        y_exact = y_exact + res
        y_fp32 = y_fp32 + res

    xa_cl, _ = ops.ncl_to_cl(x.cuda(), ops.ACT_LEAKY, 0.2)
    assert torch.equal(xa_cl.float().cpu(), xa.permute(0, 2, 1))
    wt = ops.weight_to_tapmajor_bf16(w.cuda())
    assert torch.equal(wt.float().cpu(), wr.permute(2, 0, 1))
    res_cl = res.permute(0, 2, 1).contiguous().cuda() if use_res else None
    out_f32, out_act = ops.conv1d_tc(xa_cl, wt, bias.cuda() if use_bias else None, res_cl, stride, dil, pad,
                                     ops.ACT_LEAKY, 0.2, want_f32=True, want_act=True)
    torch.cuda.synchronize()
    y = ops.cl_to_ncl(out_f32)
    assert y.shape == y_exact.shape
    assert rel_l2(y, y_exact) < 2e-5
    assert rel_l2(y, y_fp32) < 1e-2
    act_ref = O.leaky_relu(y_exact, 0.2).bfloat16().float().permute(0, 2, 1)
    assert rel_l2(out_act.float(), act_ref) < 5e-3


WG_CASES = [
    # B, Cm(=Cout), Cn(=Cin), L, K, stride, dil, pad_l, pad_r
    (2, 64, 64, 256, 3, 1, 1, 1, 1),
    (2, 96, 96, 512, 3, 1, 3, 3, 3),
    (3, 96, 16, 384, 7, 1, 1, 3, 3),
    (2, 192, 96, 512, 8, 4, 1, 3, 4),
    (4, 1536, 768, 64, 4, 2, 1, 1, 2),
    (5, 256, 1536, 32, 3, 1, 1, 1, 1),
    (2, 192, 192, 1000, 3, 1, 9, 9, 9),
    (2, 32, 96, 300, 7, 1, 1, 6, 0),
]


@pytest.mark.parametrize("case", WG_CASES)
def test_conv1d_tc_wgrad_vs_oracle(case):
    from rave_b200 import ops
    B, Cm, Cn, L, K, stride, dil, pad_l, pad_r = case
    g = torch.Generator().manual_seed(hash(case) % (2 ** 31))
    x = torch.randn(B, Cn, L, generator=g).bfloat16().float()
    Lout = (L + pad_l + pad_r - dil * (K - 1) - 1) // stride + 1
    dy = torch.randn(B, Cm, Lout, generator=g).bfloat16().float()
    w = torch.zeros(Cm, Cn, K, requires_grad=True)
    y = O.conv1d(x, w, None, stride, dil, (pad_l, pad_r))
    (dw_ref,) = torch.autograd.grad(y, w, dy)
    P = dy.permute(0, 2, 1).contiguous().bfloat16().cuda()
    Q = x.permute(0, 2, 1).contiguous().bfloat16().cuda()
    db = torch.zeros(Cm, device="cuda")
    dwt = ops.conv1d_tc_wgrad(P, Q, K, stride, dil, pad_l, dbias=db)
    dw = ops.tapmajor_to_weight(dwt)
    torch.cuda.synchronize()
    assert dw.shape == dw_ref.shape
    assert rel_l2(dw, dw_ref) < 2e-5
    assert rel_l2(db, dy.sum((0, 2))) < 1e-5          # fused bias gradient (column sums of P)


def test_small_channel_kernels_vs_emulator():
    """conv_c1 fwd/wgrad and the feature-matching stats/grad kernels against the torch emulation of
    their documented semantics (tests/tc_emulator.py), which test_engine_cpu.py ties to the oracle."""
    from rave_b200 import ops
    from tests import tc_emulator as E
    torch.manual_seed(0)
    for (R, L, Cout, K, stride, pad) in [(6, 1000, 96, 15, 4, 7), (10, 333, 48, 5, 4, 2), (3, 64, 32, 5, 3, 2)]:
        x = torch.randn(R, L + 3)
        w = torch.randn(Cout, 1, K) * 0.3
        b = torch.randn(Cout)
        Lout = (L + 2 * pad - K) // stride + 1
        pitch = Lout + 2
        of_e, oa_e = torch.zeros(R, pitch, Cout), torch.zeros(R, pitch, Cout, dtype=torch.bfloat16)
        E.conv1d_c1(x, w, b, L, stride, (pad, pad), 1, 0.2, out_f32=of_e, out_act=oa_e, Lout=Lout)
        of = torch.zeros(R, pitch, Cout, device="cuda")
        oa = torch.zeros(R, pitch, Cout, device="cuda", dtype=torch.bfloat16)
        ops.conv1d_c1(x.cuda(), w.cuda(), b.cuda(), L, stride, (pad, pad), 1, 0.2, out_f32=of, out_act=oa, Lout=Lout)
        assert rel_l2(of, of_e) < 1e-5 and rel_l2(oa.float(), oa_e.float()) < 4e-3
        g = torch.randn(R, pitch, Cout).bfloat16()
        dw_e = E.conv1d_c1_wgrad(g, x, Cout, K, L, Lout, stride, pad).sum(0)
        dw = ops.conv1d_c1_wgrad(g.cuda(), x.cuda(), Cout, K, L, Lout, stride, pad).sum(0)
        assert dw.shape == dw_e.shape and rel_l2(dw, dw_e) < 1e-4
        we = torch.randn(Cout, 1, K) * 0.3
        dx_e = E.conv1d_c1_dgrad(g, we, L + 3, L, Lout, stride, pad)
        dx = ops.conv1d_c1_dgrad(g.cuda(), we.cuda(), L + 3, L, Lout, stride, pad)
        assert dx.shape == dx_e.shape and rel_l2(dx, dx_e) < 1e-5
        xz = x.clone()
        xz[:, L:] = 0                         # rows handed over as a padded tensor: slack beyond L is zero
        X_e = E.im2col_c1(xz, L, Lout, pitch, K, stride, pad)
        X = ops.im2col_c1(xz.cuda(), L, Lout, pitch, K, stride, pad)
        assert torch.equal(X.float().cpu(), X_e.float())
        Pm = torch.randn(R, pitch, 16)
        assert rel_l2(ops.gather_c1(Pm.cuda(), (R, L + 3), L, Lout, K, stride, pad),
                      E.gather_c1(Pm, (R, L + 3), L, Lout, K, stride, pad)) < 1e-6
        # the same rows read in place from a signal tensor: fold by a period / average pooling
        # period 64: the staged tile exceeds 96 KB of shared memory and the per-thread im2col kernel runs
        for (period, pool) in [(3, 1), (7, 1), (1, 2), (1, 4), (64, 1)]:
            Bs, T = 4, L * period * pool - (2 if period > 1 else 0) + (1 if pool > 1 else 0)
            src = torch.randn(Bs, T)
            Ls = (T + period - 1) // period if period > 1 else T // pool
            Lo = (Ls + 2 * pad - K) // stride + 1
            Xs_e = E.im2col_c1(src, Ls, Lo, Lo + 1, K, stride, pad, period, pool)
            Xs = ops.im2col_c1(src.cuda(), Ls, Lo, Lo + 1, K, stride, pad, period, pool)
            assert rel_l2(Xs.float(), Xs_e.float()) < 4e-3          # bf16 rounding of pooled means may differ by 1 ulp
            Ps = torch.randn(Bs * period, Lo + 1, 16)
            assert rel_l2(ops.gather_c1(Ps.cuda(), (Bs, T), Ls, Lo, K, stride, pad, period, pool),
                          E.gather_c1(Ps, (Bs, T), Ls, Lo, K, stride, pad, period, pool)) < 1e-6
        cs = ops.colsum_bf16(g.cuda(), Lout, Cout)
        assert rel_l2(cs, E.colsum_bf16(g, Lout, Cout)) < 1e-5
    for (B2, L, pitch, C) in [(4, 100, 104, 96), (8, 17, 20, 192), (2, 5, 5, 16)]:
        a = torch.randn(B2, pitch, C).bfloat16()
        st_e = torch.zeros(2)
        E.fm_stats(a, st_e, L, 0.2)
        st = torch.zeros(2, device="cuda")
        ops.fm_stats(a.cuda(), st, L, 0.2)
        assert rel_l2(st, st_e) < 1e-4
        d = torch.tensor([0.37, -1.2])
        g_e = E.fm_grad(a, d, L, 0.2)
        g = ops.fm_grad(a.cuda(), d.cuda(), L, 0.2)
        assert torch.equal(g.float().cpu(), g_e.float())


def test_multi_tensor_weight_kernels_match_single():
    from rave_b200 import ops
    torch.manual_seed(1)
    items, singles = [], []
    for (C0, C1, K, wn, C0p, C1p) in [(96, 16, 7, True, 96, 16), (192, 96, 8, True, 192, 96), (96, 1, 15, True, 96, 16),
                                      (1, 768, 1, False, 16, 768), (1536, 768, 4, True, 1536, 768), (48, 48, 3, True, 48, 48),
                                      (8, 2048, 15, True, 16, 2048)]:
        v = torch.randn(C0, C1, K, device="cuda")
        g = (torch.rand(C0, 1, 1, device="cuda") + 0.5) if wn else None
        tapsA = list(range(K))
        tapsB = list(range(K - 1, -1, -1))
        items.append((v, g, tapsA, tapsB, C0p, C1p))
        singles.append(ops.weight_prep_tc(v, g, tapsA, tapsB, C0p, C1p))
    multi = ops.weight_prep_tc_multi(items)
    for (n1, a1, b1), (n2, a2, b2) in zip(singles, multi):
        assert (n1 is None) == (n2 is None)
        if n1 is not None:
            assert torch.equal(n1, n2)
        assert torch.equal(a1, a2) and torch.equal(b1, b2)
    jobs, ref = [], []
    for (v, g, tapsA, tapsB, C0p, C1p), (norm, _, _) in zip(items, multi):
        K = v.shape[2]
        dwt = torch.randn(3, K, C0p, C1p, device="cuda")
        jobs.append((dwt, v, g, norm))
        ref.append(ops.weight_norm_bwd_tapmajor(dwt, v, g, norm))
    # one launch takes the kernel its widest row allows: the last row (C1 K > 24 k weights) does not fit the shared-memory
    # tile, so on its own it runs the global-memory kernel
    out = ops.weight_norm_bwd_multi(jobs[:-1]) + ops.weight_norm_bwd_multi(jobs[-1:])
    for (dv1, dg1), (dv2, dg2) in zip(ref, out):
        assert torch.allclose(dv1, dv2, rtol=1e-5, atol=1e-6)
        assert (dg1 is None) == (dg2 is None)
        if dg1 is not None:
            assert torch.allclose(dg1, dg2, rtol=1e-5, atol=1e-6)


def test_score_tail_kernels_vs_emulator():
    """rave_score_stats / rave_score_grad (discriminator score tail) against the torch emulation."""
    from rave_b200 import ops
    from tests import tc_emulator as E
    g = torch.Generator().manual_seed(11)
    for (B2, pitch, L, C) in [(8, 24, 24, 16), (64, 260, 257, 16), (6, 96, 94, 16)]:
        s = torch.randn(B2, pitch, C, generator=g) * 1.5
        st_ref = torch.zeros(3, 2)
        E.score_stats(s, st_ref, L)
        st = torch.zeros(3, 2, device="cuda")
        ops.score_stats(s.cuda(), st, L)
        torch.cuda.synchronize()
        assert rel_l2(st, st_ref) < 1e-5
        d = torch.randn(3, 2, generator=g)
        g_ref = E.score_grad(s, d, L).float()
        g_gpu = ops.score_grad(s.cuda(), d.cuda(), L)
        torch.cuda.synchronize()
        assert g_gpu.dtype == torch.bfloat16 and g_gpu.shape == (B2, pitch, C)
        assert torch.equal(g_gpu.float().cpu(), g_ref.bfloat16().float())


@pytest.mark.parametrize("shape", [(4, 64, 96, 300, 3, 1), (6, 192, 96, 515, 2, 4)])
def test_conv1d_tc_fused_fm_gradient_vs_emulator(shape):
    """dgrad-style launch with the feature-matching gradient fused into the epilogue (LeakyReLU' mask from the saved
    operand, then + d0 sgn(h_r - h_f) + d1 sgn(h_r) / - d0 sgn(h_r - h_f)), plain and phase-interleaved rows."""
    from rave_b200 import ops
    from tests import tc_emulator as E
    B, Cin, Cout, L, K, rs = shape
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, L, Cin, generator=g).bfloat16()
    wt = (torch.randn(K, Cout, Cin, generator=g) / (Cin * K) ** 0.5).bfloat16()
    rows = L * rs + 3
    a = torch.nn.functional.leaky_relu(torch.randn(B, rows, Cout, generator=g), 0.2).bfloat16()
    d = torch.tensor([0.37, -0.21])
    kw = dict(stride=1, dil=1, pad=(K - 1, 0), act=0, slope=0.2, want_f32=False, want_act=False, Lout=L, Lin=L,
              out_rows=rows, out_row_stride=rs, out_row_offset=rs - 1)
    ref = torch.zeros(B, rows, Cout, dtype=torch.bfloat16)
    E.conv1d_tc(x, wt, None, None, out_act=ref, dact_src=a, fm_d=d, **kw)
    out = torch.zeros(B, rows, Cout, dtype=torch.bfloat16, device="cuda")
    ops.conv1d_tc(x.cuda(), wt.cuda(), None, None, out_act=out, dact_src=a.cuda(), fm_d=d.cuda(), **kw)
    torch.cuda.synchronize()
    assert rel_l2(out.float(), ref.float()) < 4e-3          # bf16 rounding of the stored gradient
    idx = torch.arange(L) * rs + rs - 1
    mask = torch.ones(rows, dtype=torch.bool)
    mask[idx] = False
    assert float(out[:, mask].float().abs().max()) == 0.0   # rows of other phases untouched


UNIT_CASES = [
    # B, C, L, dil, pad_l (centered = dil, causal = 2 * dil), training (keep a1), fp32 output
    (2, 96, 512, 1, 1, True, False),
    (3, 96, 1000, 3, 3, False, True),        # ragged length
    (2, 96, 4096, 9, 9, True, False),
    (2, 192, 1024, 3, 3, True, True),
    (5, 192, 256, 9, 18, False, False),      # causal padding
    (2, 384, 256, 1, 1, True, False),        # two N chunks of 192
    (9, 384, 64, 9, 9, False, True),         # several batches per tile
    (32, 96, 4096, 3, 3, True, False),       # BASELINE config 3 shape: 1024 tiles over 132 persistent CTAs
]


@pytest.mark.parametrize("case", UNIT_CASES)
def test_fused_dilated_unit_vs_two_launches_and_oracle(case):
    """rave_dilated_unit_tc_fwd (one kernel, intermediate in shared memory) against the per-layer wgmma launches it
    replaces (same operands, same accumulation order: <= 1e-6) and against the fp32 oracle of Residual(DilatedUnit)
    (rave/blocks.py:31-45, 83-112) at the bf16-mode tolerance."""
    from rave_b200 import ops
    B, C, L, dil, pad_l, keep_a1, want_f32 = case
    g = torch.Generator().manual_seed(hash(case) % (2 ** 31))
    x = torch.randn(B, C, L, generator=g)
    w3 = torch.randn(C, C, 3, generator=g) / (3 * C) ** 0.5
    w1 = torch.randn(C, C, 1, generator=g) / C ** 0.5
    pad = (pad_l, 2 * dil - pad_l)
    y_ref = x + O.conv1d(O.leaky_relu(O.conv1d(O.leaky_relu(x, 0.2), w3, None, 1, dil, pad), 0.2), w1, None, 1, 1, (0, 0))
    xa, _ = ops.ncl_to_cl(x.cuda(), ops.ACT_LEAKY, 0.2)
    w3t = ops.weight_to_tapmajor_bf16(w3.cuda())
    w1t = ops.weight_to_tapmajor_bf16(w1.cuda())
    # two launches
    _, a1_ref = ops.conv1d_tc(xa, w3t, None, None, 1, dil, pad, ops.ACT_LEAKY, 0.2, want_f32=False, want_act=True)
    o_ref, oa_ref = ops.conv1d_tc(a1_ref, w1t, None, None, 1, 1, (0, 0), ops.ACT_LEAKY, 0.2, want_f32=True, want_act=True,
                                  res_act=xa, res_slope=0.2)
    # fused
    out_f32 = torch.full((B, L, C), float("nan"), device="cuda") if want_f32 else None
    out_act = torch.empty(B, L, C, device="cuda", dtype=torch.bfloat16)
    a1, _, _ = ops.dilated_unit_tc(xa, w3t, w1t, dil, pad_l, 0.2, 0.2, ops.ACT_LEAKY, 0.2, want_a1=keep_a1,
                                   out_f32=out_f32, out_act=out_act)
    torch.cuda.synchronize()
    if keep_a1:
        assert rel_l2(a1.float(), a1_ref.float()) < 1e-6
    assert rel_l2(out_act.float(), oa_ref.float()) < 1e-6
    if want_f32:
        assert rel_l2(out_f32, o_ref) < 1e-6
        assert rel_l2(ops.cl_to_ncl(out_f32), y_ref) < 1.5e-2
    y_act = O.leaky_relu(y_ref, 0.2).permute(0, 2, 1)
    assert rel_l2(out_act.float(), y_act) < 1.5e-2

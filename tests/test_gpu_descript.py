"""GPU: the v3 discriminator (rave/descript_discriminator.py) entirely on the library kernels -- MPD as conv1d over the
period-folded signal, MRD as framing kernel + rfft + (kt, kf) Conv2d stacks run as conv1d along frequency -- against the
oracle restatement (pinned against the live reference: tests/test_oracle_golden.py), forward features and gradients."""
import pytest
import torch

from oracle import rave_oracle as O
from tests.conftest import rel_l2

pytestmark = pytest.mark.gpu


def test_disc_conv2d_vs_torch_conv2d():
    """DiscConv2d (time taps folded into channels, conv1d along frequency) == F.conv2d, forward and gradients."""
    from rave_b200.descript_discriminator import DiscConv2d
    torch.manual_seed(0)
    for (cin, cout, k, s, p, shape) in [(2, 32, (3, 9), (1, 1), (1, 4), (2, 2, 17, 51)),
                                        (32, 32, (3, 9), (1, 2), (1, 4), (2, 32, 9, 77)),
                                        (32, 1, (3, 3), (1, 1), (1, 1), (3, 32, 5, 20))]:
        conv = DiscConv2d(cin, cout, k, s, padding=p)
        x = torch.randn(*shape)
        xo = x.clone().requires_grad_(True)
        y_o = torch.nn.functional.conv2d(xo, conv.weight, conv.bias, s, p)
        probe = torch.randn_like(y_o)
        g_o = torch.autograd.grad((y_o * probe).sum(), [xo, conv.weight, conv.bias])
        conv.cuda()
        xg = x.cuda().requires_grad_(True)
        y = conv(xg)
        assert y.shape == y_o.shape and rel_l2(y, y_o) < 2e-5
        g = torch.autograd.grad((y * probe.cuda()).sum(), [xg, conv.weight, conv.bias])
        for a, b in zip(g, g_o):
            assert rel_l2(a, b) < 1e-4


def test_descript_mrd_vs_oracle():
    from rave_b200.descript_discriminator import MRD
    torch.manual_seed(0)
    mrd = MRD(512)
    sd = {k: v.detach().clone() for k, v in mrd.state_dict().items()}
    assert "band_convs.0.0.0.weight_g" in sd and "conv_post.weight_v" in sd and "stft.window" in sd
    x = torch.randn(2, 1, 4000)
    po = {k: v.clone().requires_grad_(v.is_floating_point() and "window" not in k) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    want = O.descript_mrd(xo, po, "", 512)
    mrd.cuda()
    xg = x.cuda().requires_grad_(True)
    got = mrd(xg)
    assert len(got) == len(want) == 26
    for a, b in zip(got, want):
        assert a.shape == b.shape and rel_l2(a, b) < 5e-5, (a.shape, rel_l2(a, b))
    probes = [torch.randn_like(b) for b in want]
    names = sorted(k for k, v in po.items() if v.requires_grad)
    g_o = torch.autograd.grad(sum((b * p).sum() for b, p in zip(want, probes)), [xo] + [po[k] for k in names])
    pg = dict(mrd.named_parameters())
    g = torch.autograd.grad(sum((a * p.cuda()).sum() for a, p in zip(got, probes)), [xg] + [pg[k] for k in names])
    errs = sorted(((rel_l2(a, b), k) for k, a, b in zip(["x"] + names, g, g_o)), reverse=True)
    print("MRD gradient rel-L2, worst five:", [(k, f"{e:.2e}") for e, k in errs[:5]])
    # every tensor <= 2e-4 except band 3 / layer 1 (stride-2 (3, 9) conv over
    # the 64-bin band): weight_v 5.9e-4, bias 6.7e-4.  The CPU oracle's own fp32-vs-fp64 distance on these tensors is
    # ~1e-6, so this is kernel summation order on a cancelling sum, not conditioning of the problem; stated bound 1e-3.
    for e, k in errs:
        assert e < 1e-3, (k, e)


def test_descript_discriminator_full_vs_oracle():
    """DescriptDiscriminator.forward (preprocess, 5 MPD + 3 MRD): 8 feature lists (6 / 26 features), all on library
    kernels, against the oracle; then the training-step arithmetic (feature matching + hinge) on those features."""
    from rave_b200.descript_discriminator import DescriptDiscriminator
    torch.manual_seed(1)
    dd = DescriptDiscriminator()
    sd = {"discriminator." + k: v.detach().clone() for k, v in dd.state_dict().items()}
    x = (0.5 * torch.randn(2, 1, 8192 + 5)).clamp(-1, 1)
    want = O.descript_discriminator(x, sd)
    dd.cuda()
    got = dd(x.cuda())
    assert [len(f) for f in got] == [6] * 5 + [26] * 3
    for fa, fb in zip(got, want):
        for a, b in zip(fa, fb):
            assert a.shape == b.shape and rel_l2(a, b) < 1e-4, (a.shape, rel_l2(a, b))
    fm, ld, la = O.gan_losses([[f.cpu() for f in s] for s in got], 1, True)
    fm_o, ld_o, la_o = O.gan_losses(want, 1, True)
    assert rel_l2(fm, fm_o) < 1e-4 and rel_l2(ld, ld_o) < 1e-4


def test_descript_mpd_bf16_engine_vs_oracle():
    """Descript MPD (1024-channel (5,1) convs: 77 % of the v3 discriminator FLOPs) as ONE wgmma chain in bf16 mode
    against the fp32 oracle: features within the bf16-mode tolerance, gradient direction of every large tensor."""
    import rave_b200
    from rave_b200.descript_discriminator import MPD
    torch.manual_seed(5)
    period = 5
    mpd = MPD(period)
    sd = {k: v.detach().clone() for k, v in mpd.state_dict().items()}
    x = (0.5 * torch.randn(2, 1, 12000 + 3)).clamp(-1, 1)
    po = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    want = O.descript_mpd(xo, po, "", period)
    probes = [torch.randn_like(b) for b in want]
    names = sorted(po)
    g_o = torch.autograd.grad(sum((b * p).sum() for b, p in zip(want, probes)), [xo] + [po[k] for k in names])
    mpd.cuda()
    rave_b200.set_precision("bf16")
    try:
        assert mpd._tc_specs() is not None
        xg = x.cuda().requires_grad_(True)
        got = mpd(xg)
        assert len(got) == 6
        for a, b in zip(got, want):
            assert a.shape == b.shape and rel_l2(a, b) < 3e-2, (a.shape, rel_l2(a, b))
        pg = dict(mpd.named_parameters())
        g = torch.autograd.grad(sum((a * p.cuda()).sum() for a, p in zip(got, probes)), [xg] + [pg[k] for k in names])
    finally:
        rave_b200.set_precision("fp32")

    def cos(a, b):
        a, b = a.detach().double().cpu().reshape(-1), b.detach().double().reshape(-1)
        return float(a @ b / (a.norm() * b.norm()).clamp_min(1e-30))
    assert cos(g[0], g_o[0]) > 0.98, cos(g[0], g_o[0])
    for k, a, b in zip(names, g[1:], g_o[1:]):
        if a.numel() >= 64:
            assert cos(a, b) > 0.97, (k, cos(a, b))


def test_descript_mrd_bf16_engine_vs_oracle():
    """MRD in bf16 mode: every (kt, kf) Conv2d as a one-layer wgmma chain (conv along frequency, time taps folded into
    channels) against the fp32 oracle: features within the bf16-mode tolerance, gradient direction."""
    import rave_b200
    from rave_b200.descript_discriminator import MRD
    torch.manual_seed(6)
    mrd = MRD(512)
    sd = {k: v.detach().clone() for k, v in mrd.state_dict().items()}
    x = torch.randn(2, 1, 6000)
    po = {k: v.clone().requires_grad_(v.is_floating_point() and "window" not in k) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    want = O.descript_mrd(xo, po, "", 512)
    probes = [torch.randn_like(b) for b in want]
    names = sorted(k for k, v in po.items() if v.requires_grad)
    g_o = torch.autograd.grad(sum((b * p).sum() for b, p in zip(want, probes)), [xo] + [po[k] for k in names])
    mrd.cuda()
    rave_b200.set_precision("bf16")
    try:
        xg = x.cuda().requires_grad_(True)
        got = mrd(xg)
        assert len(got) == len(want) == 26
        for a, b in zip(got, want):
            assert a.shape == b.shape and rel_l2(a, b) < 3e-2, (a.shape, rel_l2(a, b))
        pg = dict(mrd.named_parameters())
        g = torch.autograd.grad(sum((a * p.cuda()).sum() for a, p in zip(got, probes)), [xg] + [pg[k] for k in names])
    finally:
        rave_b200.set_precision("fp32")

    def cos(a, b):
        a, b = a.detach().double().cpu().reshape(-1), b.detach().double().reshape(-1)
        return float(a @ b / (a.norm() * b.norm()).clamp_min(1e-30))
    assert cos(g[0], g_o[0]) > 0.98, cos(g[0], g_o[0])
    ga = torch.cat([a.detach().cpu().reshape(-1) for a in g[1:]])
    gb = torch.cat([b.reshape(-1) for b in g_o[1:]])
    assert cos(ga, gb) > 0.99, cos(ga, gb)
    for k, a, b in zip(names, g[1:], g_o[1:]):
        if a.numel() >= 64:
            assert cos(a, b) > 0.95, (k, cos(a, b))


def test_time_stack_nhwc_and_l1_halves_vs_torch():
    """The channel-last MRD plumbing: rave_time_stack_nhwc (+ adjoint) on a strided band slice and on dense rows, and
    the one-buffer L1 feature matching (rave_l1_* on the two halves of a buffer)."""
    from rave_b200 import ops
    torch.manual_seed(3)
    for (B, T, Ftot, C, lo, hi, kt, Cp, Fp) in [(3, 9, 40, 2, 5, 31, 3, 16, 26), (2, 7, 33, 32, 0, 33, 3, 96, 34),
                                                (2, 5, 20, 32, 3, 20, 3, 112, 17), (2, 4, 12, 8, 0, 12, 1, 16, 12)]:
        pt = (kt - 1) // 2
        base = torch.randn(B, T, Ftot, C, device="cuda")
        x = base[:, :, lo:hi, :].detach().requires_grad_(True)
        F_ = hi - lo
        out = ops.time_stack_nhwc(x, kt, pt, Cp, Fp)
        xp = torch.nn.functional.pad(x, (0, 0, 0, 0, pt, pt))
        want = torch.cat([xp[:, dt:dt + T] for dt in range(kt)], -1)                      # [B, T, F, kt C]
        want = torch.nn.functional.pad(want, (0, Cp - kt * C, 0, Fp - F_)).reshape(B * T, Fp, Cp)
        assert torch.equal(out, want.bfloat16())
        g = torch.randn_like(out)
        (gx,) = torch.autograd.grad(out, x, g)
        (gw,) = torch.autograd.grad(want, x, g.float())
        assert rel_l2(gx, gw) < 1e-6
    buf = torch.randn(6, 50, 32, device="cuda")
    buf[:, 45:] = 0.
    b1 = buf.clone().requires_grad_(True)
    b2 = buf.clone().requires_grad_(True)
    st = ops.l1_halves(b1)
    want = torch.stack([(b2[:3] - b2[3:]).abs().sum(), b2[:3].abs().sum()])
    assert rel_l2(st, want) < 1e-6
    d = torch.tensor([0.7, -0.3], device="cuda")
    (g1,) = torch.autograd.grad((st * d).sum(), b1)
    (g2,) = torch.autograd.grad((want * d).sum(), b2)
    assert torch.allclose(g1, g2, atol=1e-6)


def test_descript_feature_matching_on_dense_buffers_matches_generic():
    """model.compute_losses' feature matching from the feature taps' own sums (`_fm_stats`, ops.leaky_fm) and on the
    `_cl_base` buffers == core.mean_difference on the split feature views (values and the gradient reaching the
    discriminator input); engine.fake_rows_only (generator step, frozen discriminator) leaves the fake half's
    gradient unchanged."""
    import rave_b200
    from rave_b200 import core, engine
    from rave_b200.descript_discriminator import DescriptDiscriminator
    torch.manual_seed(2)
    dd = DescriptDiscriminator().cuda()
    x = (0.5 * torch.randn(4, 1, 16384, device="cuda")).clamp(-1, 1)
    rave_b200.set_precision("bf16")
    try:
        res = {}
        for mode in ("stats", "bases", "generic", "stats_fake_only"):
            frozen = mode == "stats_fake_only"
            for p in dd.parameters():
                p.requires_grad_(not frozen)
            xg = x.clone().requires_grad_(True)
            with engine.fake_rows_only(frozen):
                feats = dd(xg)
            total = 0.
            n_bases = 0
            for scale in feats:
                for f in scale[:-1]:
                    assert f.shape[0] == 4
                    base, st = getattr(f, "_cl_base", None), getattr(f, "_fm_stats", None)
                    n_bases += base is not None and st is not None
                    if mode.startswith("stats"):
                        total = total + st[0] / (f.numel() // 2)
                    elif mode == "bases":
                        total = total + core.mean_difference_halves(base, f.numel() // 2, False)
                    else:
                        total = total + core.mean_difference(f[:2], f[2:], "L1", False)
                total = total - scale[-1][2:].mean()      # the score: every chain's last layer needs a gradient
            assert n_bases == 5 * 5 + 3 * 25
            (gx,) = torch.autograd.grad(total, xg)
            res[mode] = (total.detach(), gx)
    finally:
        rave_b200.set_precision("fp32")
        for p in dd.parameters():
            p.requires_grad_(True)
    for mode in ("stats", "bases", "stats_fake_only"):
        assert rel_l2(res[mode][0], res["generic"][0]) < 1e-5, mode
    # bf16 gradient streams, different accumulation order between the fused and the generic backward
    assert rel_l2(res["stats"][1], res["generic"][1]) < 2e-3
    assert rel_l2(res["bases"][1], res["generic"][1]) < 2e-3
    assert rel_l2(res["stats_fake_only"][1][2:], res["stats"][1][2:]) < 1e-4
    assert torch.count_nonzero(res["stats_fake_only"][1][:2]) == 0


def test_leaky_fm_stack_equals_tap_plus_time_stack():
    """ops.leaky_fm_stack (the feature tap that also writes the next MRD conv's time-stacked operand) == ops.leaky_fm
    followed by ops.time_stack_nhwc, bit for bit in the forward (borders, pad columns, both halves) and through the
    backward (with and without a gradient arriving at the feature itself)."""
    from rave_b200 import ops
    torch.manual_seed(6)
    for (B, T, F_, C, stride) in [(4, 5, 9, 32, 2), (2, 3, 8, 32, 1), (2, 1, 5, 16, 2), (6, 7, 33, 32, 2), (2, 2, 1, 8, 2)]:
        Fp = F_ + (-F_) % stride
        x = torch.randn(B * T, F_, C, device="cuda")
        x1 = x.clone().requires_grad_(True)
        x2 = x.clone().requires_grad_(True)
        a1, st1, xs1 = ops.leaky_fm_stack(x1, 0.1, T, Fp)
        a2, st2 = ops.leaky_fm(x2, 0.1)
        xs2 = ops.time_stack_nhwc(a2.view(B, T, F_, C), 3, 1, 3 * C, Fp)
        assert xs1.shape == xs2.shape == (B * T, Fp, 3 * C)
        assert torch.equal(a1, a2) and torch.equal(xs1, xs2) and rel_l2(st1, st2) < 1e-6
        pa = torch.randn_like(a1)
        px = torch.randn(xs1.shape, device="cuda")
        d = torch.tensor([0.7, -0.3], device="cuda")
        for with_a in (True, False):
            l1 = (st1 * d).sum() + (xs1.float() * px).sum() + ((a1 * pa).sum() if with_a else 0.)
            l2 = (st2 * d).sum() + (xs2.float() * px).sum() + ((a2 * pa).sum() if with_a else 0.)
            (g1,) = torch.autograd.grad(l1, x1, retain_graph=True)
            (g2,) = torch.autograd.grad(l2, x2, retain_graph=True)
            assert torch.allclose(g1, g2, rtol=1e-5, atol=1e-5), (B, T, F_, C, with_a)


def test_leaky_fm_tap_vs_torch():
    from rave_b200 import ops
    torch.manual_seed(4)
    for shape in [(6, 50, 32), (2, 7, 3), (4, 33, 16)]:
        x = torch.randn(*shape, device="cuda")
        x1 = x.clone().requires_grad_(True)
        x2 = x.clone().requires_grad_(True)
        a, st = ops.leaky_fm(x1, 0.1)
        h = shape[0] // 2
        a2 = torch.nn.functional.leaky_relu(x2, 0.1)
        st2 = torch.stack([(a2[:h] - a2[h:]).abs().sum(), a2[:h].abs().sum()])
        assert torch.equal(a, a2) and rel_l2(st, st2) < 1e-6
        probe = torch.randn_like(a)
        d = torch.tensor([0.7, -0.3], device="cuda")
        for use_a, use_d in [(True, True), (True, False), (False, True)]:
            l1 = (a * probe).sum() * use_a + (st * d).sum() * use_d
            l2 = (a2 * probe).sum() * use_a + (st2 * d).sum() * use_d
            (g1,) = torch.autograd.grad(l1, x1, retain_graph=True)
            (g2,) = torch.autograd.grad(l2, x2, retain_graph=True)
            assert torch.allclose(g1, g2, atol=1e-6), (shape, use_a, use_d)

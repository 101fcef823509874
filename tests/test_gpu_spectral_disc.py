"""GPU: the multi-scale spectral discriminator (rave/discriminator.py:12-74, 139-153) on the library kernels -- the
uncentred normalised framing kernel + rfft, the time-dilated stacking and feature-tap kernels, SpectralConv2d on the
fp32 conv1d kernels and as one-layer wgmma chains -- against torch, the oracle restatement and the reference's goldens."""
import copy
import math
import os
from functools import partial

import pytest
import torch

from oracle import rave_oracle as O
from oracle import spectral_oracle as S
from tests.conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu


def load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def cos(a, b):
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    return float(a @ b / (a.norm() * b.norm()).clamp_min(1e-30))


def test_valid_framing_and_rfft_vs_torch_stft():
    """rave_stft_frames_valid (+ cuFFT) == torch.stft(center=False) / ||w||_2, ragged lengths; adjoint == autograd."""
    from rave_b200 import ops
    torch.manual_seed(0)
    for n_fft, T in [(256, 4096 + 37), (1024, 8192), (4096, 4096 + 3), (512, 513 + 64 * 5)]:
        hop = n_fft // 4
        w = torch.hann_window(n_fft, device="cuda")
        s = float(1.0 / w.pow(2).sum().sqrt())
        bw = torch.full((n_fft // 2 + 1,), 0.5 * n_fft, device="cuda")
        bw[0] = bw[-1] = n_fft
        x = torch.randn(3, T, device="cuda")
        xg = x.clone().requires_grad_(True)
        fr = ops.stft_frames_valid(xg, w, n_fft, hop, s)
        z = ops.rfft(fr, bw)
        want = (torch.stft(x, n_fft, hop, n_fft, w, center=False, normalized=False, onesided=True, return_complex=True)
                / w.pow(2).sum().sqrt()).transpose(-1, -2)
        assert z.shape == want.shape and rel_l2(torch.view_as_real(z), torch.view_as_real(want)) <= 1e-6
        xr = x.clone().requires_grad_(True)
        fr_ref = xr.unfold(-1, n_fft, hop) * w * s
        assert rel_l2(fr, fr_ref) <= 1e-6
        probe = torch.randn_like(fr)
        (g1,) = torch.autograd.grad((fr * probe).sum(), xg)
        (g2,) = torch.autograd.grad((fr_ref * probe).sum(), xr)
        assert rel_l2(g1, g2) <= 1e-6, (n_fft, T, rel_l2(g1, g2))


def _gather_stack(x, kt, pt, dil, Cp, Fp):
    B, T, F_, C = x.shape
    xp = torch.nn.functional.pad(x, (0, 0, 0, 0, pt, pt))
    want = torch.cat([xp[:, j * dil:j * dil + T] for j in range(kt)], -1)
    return torch.nn.functional.pad(want, (0, Cp - kt * C, 0, Fp - F_)).reshape(B * T, Fp, Cp)


def test_dilated_time_stack_vs_torch_gather():
    """rave_time_stack_nhwc_dil (+ adjoint), dil in {1, 2, 4}, on strided band slices / odd F / dense rows: bit-exact
    against a torch gather; at dil = 1 bit-identical to rave_time_stack_nhwc (+ _bwd)."""
    from rave_b200 import ops
    from rave_b200._lib import call, ptr, stream_ptr
    torch.manual_seed(3)
    for (B, T, Ftot, C, lo, hi, kt, Cp, Fp) in [(3, 9, 40, 2, 5, 31, 3, 16, 26), (2, 7, 33, 32, 0, 33, 3, 96, 34),
                                                (2, 5, 21, 32, 3, 20, 3, 112, 17), (2, 4, 12, 8, 0, 12, 1, 16, 12),
                                                (2, 13, 9, 16, 0, 9, 3, 48, 10)]:
        for dil in (1, 2, 4):
            pt = dil * (kt - 1) // 2
            base = torch.randn(B, T, Ftot, C, device="cuda")
            x = base[:, :, lo:hi, :].detach().requires_grad_(True)
            F_ = hi - lo
            out = ops.time_stack_nhwc(x, kt, pt, Cp, Fp, dil)
            want = _gather_stack(x, kt, pt, dil, Cp, Fp)
            assert torch.equal(out, want.bfloat16()), (B, T, C, dil)
            g = torch.randn_like(out)
            (gx,) = torch.autograd.grad(out, x, g)
            (gw,) = torch.autograd.grad(want, x, g.float())
            assert rel_l2(gx, gw) <= 1e-6
            if dil == 1:
                old = torch.empty_like(out)
                xd = x.detach()
                call("rave_time_stack_nhwc", xd.data_ptr(), ptr(old), B, C, T, F_, xd.stride(0), xd.stride(1), Fp, Cp,
                     kt, pt, stream_ptr())
                assert torch.equal(old, out)
                gold = torch.empty(B, T, F_, C, device="cuda")
                call("rave_time_stack_nhwc_bwd", ptr(g), ptr(gold), B, C, T, F_, Fp, Cp, kt, pt, stream_ptr())
                assert torch.equal(gold, gx)


def test_dilated_leaky_fm_stack_equals_tap_plus_dilated_stack():
    """ops.leaky_fm_stack(dil) == ops.leaky_fm followed by ops.time_stack_nhwc(kt = 3, pt = dil, dil), bit for bit in
    the forward (borders, T <= dil, pad columns, both halves) and through the backward; at dil = 1 bit-identical to
    rave_leaky_fm_stack_fwd / _bwd."""
    from rave_b200 import ops
    from rave_b200._lib import call, ptr, stream_ptr
    torch.manual_seed(6)
    for (B, T, F_, C, stride) in [(4, 5, 9, 32, 2), (2, 3, 8, 32, 1), (2, 1, 5, 16, 2), (6, 7, 33, 32, 2),
                                  (2, 2, 1, 8, 2), (2, 11, 17, 32, 1)]:
        Fp = F_ + (-F_) % stride
        for dil in (1, 2, 4):
            x = torch.randn(B * T, F_, C, device="cuda")
            x1 = x.clone().requires_grad_(True)
            x2 = x.clone().requires_grad_(True)
            a1, st1, xs1 = ops.leaky_fm_stack(x1, 0.2, T, Fp, dil)
            a2, st2 = ops.leaky_fm(x2, 0.2)
            xs2 = ops.time_stack_nhwc(a2.view(B, T, F_, C), 3, dil, 3 * C, Fp, dil)
            assert xs1.shape == xs2.shape == (B * T, Fp, 3 * C)
            assert torch.equal(a1, a2) and torch.equal(xs1, xs2) and rel_l2(st1, st2) < 1e-6, (B, T, dil)
            pa = torch.randn_like(a1)
            px = torch.randn(xs1.shape, device="cuda")
            d = torch.tensor([0.7, -0.3], device="cuda")
            for with_a in (True, False):
                l1 = (st1 * d).sum() + (xs1.float() * px).sum() + ((a1 * pa).sum() if with_a else 0.)
                l2 = (st2 * d).sum() + (xs2.float() * px).sum() + ((a2 * pa).sum() if with_a else 0.)
                (g1,) = torch.autograd.grad(l1, x1, retain_graph=True)
                (g2,) = torch.autograd.grad(l2, x2, retain_graph=True)
                assert torch.allclose(g1, g2, rtol=1e-5, atol=1e-5), (B, T, F_, C, dil, with_a)
            if dil == 1:
                a3 = torch.empty_like(x)
                st3 = torch.zeros(2, device="cuda")
                xs3 = torch.empty_like(xs1)
                call("rave_leaky_fm_stack_fwd", ptr(x), ptr(a3), ptr(st3), ptr(xs3), B * T // 2, T, F_, C, Fp, 0.2,
                     stream_ptr())
                assert torch.equal(a3, a1) and torch.equal(xs3, xs1) and torch.equal(st3, st1)
                gxs = px.bfloat16()
                gn = torch.empty_like(x)
                gd = torch.empty_like(x)
                call("rave_leaky_fm_stack_bwd", ptr(a1.detach()), ptr(gxs), ptr(pa), ptr(d), ptr(gn), B * T // 2, T, F_,
                     C, Fp, 0.2, stream_ptr())
                call("rave_leaky_fm_stack_dil_bwd", ptr(a1.detach()), ptr(gxs), ptr(pa), ptr(d), ptr(gd), B * T // 2, T,
                     F_, C, Fp, 1, 0.2, stream_ptr())
                assert torch.equal(gn, gd)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_spectral_conv2d_vs_torch_conv2d(precision):
    """SpectralConv2d == F.conv2d on [B, C, F, T]: the EncodecConvNet geometries.  fp32 kernels: forward <= 2e-5,
    gradients <= 1e-4; the one-layer wgmma chain (bf16 operands): <= 2e-2 / gradient cosine > 0.99."""
    import rave_b200
    from rave_b200.discriminator import SpectralConv2d
    torch.manual_seed(0)
    cases = [(2, 32, (9, 3), (1, 1), (1, 1), (4, 1), (2, 2, 65, 19)),
             (32, 32, (9, 3), (2, 1), (1, 1), (4, 1), (2, 32, 33, 11)),
             (32, 32, (9, 3), (2, 1), (1, 2), (4, 2), (2, 32, 31, 13)),
             (32, 32, (9, 3), (2, 1), (1, 4), (4, 4), (2, 32, 17, 9)),
             (32, 32, (3, 3), (1, 1), (1, 1), (1, 1), (2, 32, 9, 7)),
             (32, 1, (3, 3), (1, 1), (1, 1), (1, 1), (3, 32, 9, 7))]
    for (cin, cout, k, s, d, p, shape) in cases:
        conv = SpectralConv2d(cin, cout, k, s, padding=p, dilation=d)
        x = torch.randn(*shape)
        xo = x.clone().requires_grad_(True)
        y_o = torch.nn.functional.conv2d(xo, conv.weight, conv.bias, s, p, d)
        probe = torch.randn_like(y_o)
        g_o = torch.autograd.grad((y_o * probe).sum(), [xo, conv.weight, conv.bias])
        conv.cuda()
        rave_b200.set_precision(precision)
        try:
            xg = x.cuda().requires_grad_(True)
            y = conv(xg)
            g = torch.autograd.grad((y * probe.cuda()).sum(), [xg, conv.weight, conv.bias])
        finally:
            rave_b200.set_precision("fp32")
        assert y.shape == y_o.shape
        if precision == "fp32":
            assert rel_l2(y, y_o) <= 2e-5
            for a, b in zip(g, g_o):
                assert rel_l2(a, b) <= 1e-4
        else:
            assert rel_l2(y, y_o) <= 2e-2, (k, d, rel_l2(y, y_o))
            for a, b in zip(g, g_o):
                assert cos(a, b) > 0.99, (k, d, cos(a, b))


def test_spectral_discriminator_fp32_vs_reference_golden():
    """MultiScaleSpectralDiscriminator on the fp32 kernels against tests/golden/discriminator_spectral.pt (written by the
    unmodified reference): features <= 5e-5, fm / loss_dis <= 1e-4, gradients of fm + loss_dis + loss_adv <= 1e-3."""
    from rave_b200.discriminator import EncodecConvNet, MultiScaleSpectralDiscriminator
    g = load("discriminator_spectral.pt")
    disc = MultiScaleSpectralDiscriminator(g["scales"], partial(EncodecConvNet, capacity=g["capacity"]))
    sd = disc.state_dict()
    params = {k[len("discriminator."):]: v for k, v in g["params"].items()}
    assert set(params) <= set(sd) and all(k.endswith(".window") for k in set(sd) - set(params))
    disc.load_state_dict(dict(sd, **params), strict=True)
    disc.cuda()
    xg = g["x"].cuda().requires_grad_(True)
    feats = disc(xg)
    assert [len(f) for f in feats] == [6] * 5
    for fa, fb in zip(feats, g["features"]):
        for a, (shape, idx, val) in zip(fa, fb):
            got = a.detach().cpu().reshape(-1)[idx]
            assert tuple(a.shape) == tuple(shape) and rel_l2(got, val) <= 5e-5, (shape, rel_l2(got, val))
    fm, ld, la = O.gan_losses(feats, 1, True)
    assert rel_l2(fm, g["fm"]) <= 1e-4 and rel_l2(ld, g["loss_dis"]) <= 1e-4
    names = sorted(g["grad_params"])
    pg = dict(disc.named_parameters(prefix="discriminator"))
    grads = torch.autograd.grad(fm + ld + la, [xg] + [pg[k] for k in names])
    assert rel_l2(grads[0], g["grad_x"]) <= 1e-3
    errs = sorted(((rel_l2(a, g["grad_params"][k]), k) for k, a in zip(names, grads[1:])), reverse=True)
    print("spectral discriminator gradient rel-L2, worst five:", [(k, f"{e:.2e}") for e, k in errs[:5]])
    for e, k in errs:
        assert e <= 1e-3, (k, e)


def test_spectral_discriminator_bf16_engine_vs_oracle():
    """bf16 mode: every EncodecConvNet conv as a one-layer wgmma chain, channel-last end to end, against the fp32
    oracle.  Features <= 3e-2 rel-L2; gradient cosine > 0.98 (input), > 0.95 (each tensor of >= 64 elements), > 0.99 (all
    parameters); no conv of the discriminator ran on the fp32 kernels."""
    import rave_b200
    from rave_b200 import _lib
    from rave_b200.discriminator import EncodecConvNet, MultiScaleSpectralDiscriminator
    torch.manual_seed(7)
    scales = [4096, 2048, 1024, 512, 256]
    disc = MultiScaleSpectralDiscriminator(scales, partial(EncodecConvNet, capacity=32))
    sd = {k: v.detach().clone() for k, v in disc.state_dict().items()}
    x = (0.5 * torch.randn(2, 1, 8192 + 3)).clamp(-1, 1)
    po = {k: v.clone().requires_grad_("window" not in k) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    want = S.multi_scale_spectral_discriminator(xo, po, "", scales)
    want = [f for s in want for f in s]
    probes = [torch.randn_like(b) for b in want]
    names = sorted(k for k, v in po.items() if v.requires_grad)
    g_o = torch.autograd.grad(sum((b * p).sum() for b, p in zip(want, probes)), [xo] + [po[k] for k in names])
    disc.cuda()
    rave_b200.set_precision("bf16")
    _lib.PROFILE = []
    try:
        xg = x.cuda().requires_grad_(True)
        assert disc.engine_ready(xg)
        got = [f for s in disc(xg) for f in s]
        assert len(got) == len(want) == 30
        for a, b in zip(got, want):
            assert a.shape == b.shape and rel_l2(a, b) < 3e-2, (a.shape, rel_l2(a, b))
        pg = dict(disc.named_parameters())
        g = torch.autograd.grad(sum((a * p.cuda()).sum() for a, p in zip(got, probes)), [xg] + [pg[k] for k in names])
        launched = {name for name, *_ in _lib.PROFILE}
    finally:
        _lib.PROFILE = None
        rave_b200.set_precision("fp32")
    assert "rave_conv1d_tc_fwd" in launched and "rave_conv1d_tc_wgrad" in launched
    assert "rave_leaky_fm_stack_dil_fwd" in launched and "rave_stft_frames_valid" in launched
    fp32_convs = {"rave_conv1d_gather_f32", "rave_conv1d_scatter_f32", "rave_conv1d_wgrad_f32"}
    assert not launched & fp32_convs, launched & fp32_convs
    assert cos(g[0], g_o[0]) > 0.98, cos(g[0], g_o[0])
    ga = torch.cat([a.detach().cpu().reshape(-1) for a in g[1:]])
    gb = torch.cat([b.reshape(-1) for b in g_o[1:]])
    assert cos(ga, gb) > 0.99, cos(ga, gb)
    for k, a, b in zip(names, g[1:], g_o[1:]):
        if a.numel() >= 64:
            assert cos(a, b) > 0.95, (k, cos(a, b))


def _run_spectral_golden_steps(precision):
    """Replays tests/golden/training_step_v2_spectral_tiny.pt (a phase-2 D-step and G-step of the reference's own
    RAVE.training_step with `--config v2 --config spectral_discriminator`, both from the same seeded parameters) through
    rave_b200.RAVE.training_step.  Returns per step (logs, the seeded sample of the stepped group's gradients)."""
    import rave_b200
    from rave_b200 import configs
    g = load("training_step_v2_spectral_tiny.pt")
    cfg = g["cfg"]
    m = configs.build_rave("v2_spectral", capacity=cfg["capacity"], latent_size=cfg["latent_size"],
                           disc_capacity=g["disc_capacity"], phase_1_duration=1000,
                           spectral_capacity=g["spectral_capacity"])
    m.update_discriminator_every = g["update_discriminator_every"]
    sd0 = dict(m.state_dict(), **S.seeded_params(g["param_shapes"], g["param_seed"]))
    m.cuda().train()
    Lz = g["T"] // cfg["n_band"] // math.prod(cfg["ratios"])
    rave_b200.set_precision(precision)
    out = []
    try:
        for st in g["steps"]:
            m.load_state_dict(sd0, strict=True)
            m.set_receptive_field(*g["receptive_field"])      # a buffer: after the load, which holds the built model's
            m.warmed_up = True
            for p in m.parameters():
                p.grad = None
            x = S.step_batch(g["B"], g["T"], st["seed"]).cuda()
            eps = S.step_eps(g["B"], cfg["latent_size"], Lz, st["seed"]).cuda()
            logs = m.training_step(x, st["batch_idx"], eps=eps)
            logs = {k: (v.detach().float().cpu() if torch.is_tensor(v) else torch.tensor(float(v))) for k, v in logs.items()}
            pg = dict(m.named_parameters())
            assert all(pg[k].grad is not None for k in st["grad_keys"]), st["name"]
            flat = torch.cat([pg[k].grad.detach().reshape(-1).cpu() for k in st["grad_keys"]])
            shape, idx, _ = st["grad_sample"]
            assert tuple(flat.shape) == tuple(shape)
            out.append((logs, flat[idx]))
    finally:
        rave_b200.set_precision("fp32")
    return g, out


def test_v2_spectral_training_step_matches_reference_goldens_fp32():
    """Logged losses <= 1e-4 of the reference's; the sampled gradient of the stepped group in direction (cos > 0.99:
    the phase-2 generator gradient is a sum of sign terms, see test_gpu_parity.py)."""
    g, out = _run_spectral_golden_steps("fp32")
    for st, (logs, gs) in zip(g["steps"], out):
        for k, want in st["logs"].items():
            if k == "beta_factor":
                continue
            assert k in logs, (st["name"], k)
            assert abs(float(logs[k]) - float(want)) <= 1e-4 * max(abs(float(want)), 1e-3), (st["name"], k,
                                                                                              float(logs[k]), float(want))
        c = cos(gs, st["grad_sample"][2])
        print(f"{st['name']} (fp32): gradient sample cos {c:.6f}")
        assert c > 0.99, (st["name"], c)


def test_v2_spectral_training_step_matches_reference_goldens_bf16():
    """Within the bounds of test_gpu_parity.py::test_training_step_matches_reference_goldens_bf16."""
    g, out = _run_spectral_golden_steps("bf16")
    for st, (logs, gs) in zip(g["steps"], out):
        for k, want in st["logs"].items():
            if k == "beta_factor":
                continue
            tol = 0.10 if k in ("feature_matching", "adversarial", "pred_fake", "pred_real") else 0.03
            assert abs(float(logs[k]) - float(want)) <= tol * max(abs(float(want)), 1e-3), (st["name"], k,
                                                                                           float(logs[k]), float(want))
        c = cos(gs, st["grad_sample"][2])
        print(f"{st['name']} (bf16): gradient sample cos {c:.4f}")
        assert c > 0.9, (st["name"], c)


def test_v2_spectral_graphed_steps_match_eager_and_are_deterministic(monkeypatch):
    """bf16, spectral discriminator on the engine: GraphedTrainer replays == eager training_step on the same data, and
    two graphed runs from the same state are bit-identical."""
    import rave_b200
    from rave_b200 import configs, discriminator
    from rave_b200.graphs import GraphedTrainer
    monkeypatch.setattr(discriminator, "DISC_STREAMS", 1)
    torch.manual_seed(0)
    rave_b200.set_precision("bf16")
    try:
        m1 = configs.build_rave("v2_spectral", capacity=16, latent_size=16, disc_capacity=16,
                                spectral_capacity=16).cuda().train()
        m1.warmed_up = True
        # freeze the reparametrisation noise so every run sees the same numbers
        m1.encoder.reparametrize = (lambda z, eps=None, enc=m1.encoder: type(enc).reparametrize(
            enc, z, torch.zeros_like(z[:, :z.shape[1] // 2])))
        m2, m3 = copy.deepcopy(m1), copy.deepcopy(m1)
        x = (0.5 * torch.randn(2, 1, 65536, device="cuda")).clamp(-1, 1)
        assert m1.discriminator.discriminators[1].engine_ready(torch.cat([x, x]))
        tr2 = GraphedTrainer(m2, x, warmup_steps=2)
        tr3 = GraphedTrainer(m3, x, warmup_steps=2)
        m1.optimizers(capturable=True)
        for i in range(4):
            l2 = tr2.step(x, i)
            l3 = tr3.step(x, i)
            l1 = m1.training_step(x, i)
        torch.cuda.synchronize()
    finally:
        rave_b200.set_precision("fp32")
    for k in ("fullband_spectral_distance", "feature_matching", "adversarial"):
        assert torch.equal(l2[k], l3[k]), k
        assert rel_l2(l2[k], l1[k]) < 2e-2, (k, float(l2[k]), float(l1[k]))
    for (n, p2), p3, p1 in zip(m2.named_parameters(), m3.parameters(), m1.parameters()):
        assert torch.equal(p2, p3), n
    w = lambda m: m.discriminator.discriminators[1].nets[0].net[1][0].weight_v
    assert rel_l2(w(m2), w(m1)) < 1e-2

"""GPU: multichannel (stereo, n_channels = 2) models -- the multichannel first-layer operand kernels (rave_im2col_cin /
rave_gather_cin) bit for bit and as an adjoint pair, the stereo first layer on the wgmma engine, the fused feature-matching
path of the v2 discriminator and the bf16 Descript discriminator in stereo, both stereo training steps against the
reference's, and CUDA-graph replays."""
import copy
import math
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import rave_oracle as O
from oracle import stereo_oracle as ST
from tests.conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu

FP32_CONVS = {"rave_conv1d_gather_f32", "rave_conv1d_scatter_f32", "rave_conv1d_wgrad_f32"}


def load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def cos(a, b):
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    return float(a @ b / (a.norm() * b.norm()).clamp_min(1e-30))


def _no_fp32_convs(monkeypatch):
    from rave_b200 import ops

    def boom(*a, **k):
        raise AssertionError("fp32 conv fallback in bf16 mode")
    monkeypatch.setattr(ops, "conv1d", boom)
    monkeypatch.setattr(ops, "conv_transpose1d", boom)


def _rows(src, Lin, period, pool):
    """Chain rows [Bs*period, cin, Lin] of src [Bs, cin, T]: zero-padded fold, or the mean of `pool` consecutive samples
    summed left to right and divided once, as the kernels do (so that the comparison can be bit for bit)."""
    Bs, cin, T = src.shape
    if period > 1:
        xp = F.pad(src, (0, Lin * period - T))
        return xp.reshape(Bs, cin, Lin, period).permute(0, 3, 1, 2).reshape(Bs * period, cin, Lin)
    v = src[..., 0:Lin * pool:pool].clone()
    for j in range(1, pool):
        v = v + src[..., j:Lin * pool:pool]
    return v / pool if pool > 1 else v


def _im2col_torch(src, Lin, Lout, out_pitch, K, stride, pad_l, period, pool, W):
    rows = _rows(src, Lin, period, pool)
    R, cin, _ = rows.shape
    X = torch.zeros(R, out_pitch, W, device=src.device)
    lpos = torch.arange(Lout, device=src.device)
    for c in range(cin):
        for k in range(K):
            pos = lpos * stride + k - pad_l
            ok = (pos >= 0) & (pos < Lin)
            X[:, lpos[ok], c * K + k] = rows[:, c, pos[ok]]
    return X.to(torch.bfloat16)


# (period, pool, K, stride, pad): the MPD (K = 5, stride 4) and MSD (K = 15, stride 4) first layers; period 29 at
# cin = 2 makes the staged tile exceed 96 KB (per-thread kernel)
IM2COL_CASES = [(p, 1, 5, 4, 2) for p in (2, 3, 5, 7, 11, 29)] + [(1, q, 15, 4, 7) for q in (1, 2, 4)] + \
               [(3, 1, 15, 4, 7), (1, 2, 5, 4, 2)]


@pytest.mark.parametrize("cin", [1, 2])
@pytest.mark.parametrize("case", IM2COL_CASES)
def test_im2col_cin_bit_exact(cin, case):
    from rave_b200 import ops
    period, pool, K, stride, pad = case
    Bs, T = 3, 3000 + 7                         # T not a multiple of any period
    g = torch.Generator().manual_seed(17 * period + pool + K + cin)
    src = torch.randn(Bs, cin, T, generator=g).cuda()
    Lin = (T + period - 1) // period if period > 1 else T // pool
    Lout = (Lin + 2 * pad - K) // stride + 1
    pitch = Lout + 3
    W = ops.cin_width(cin, K)
    X = ops.im2col_cin(src, Lin, Lout, pitch, K, stride, pad, period, pool)
    want = _im2col_torch(src, Lin, Lout, pitch, K, stride, pad, period, pool, W)
    assert X.shape == want.shape
    assert torch.equal(X.view(torch.int16), want.view(torch.int16))
    if cin == 1:
        assert W == 16
        X1 = ops.im2col_c1(src[:, 0].contiguous(), Lin, Lout, pitch, K, stride, pad, period, pool)
        assert torch.equal(X1.view(torch.int16), X.view(torch.int16))


@pytest.mark.parametrize("cin", [1, 2])
@pytest.mark.parametrize("case", IM2COL_CASES)
def test_gather_cin_is_the_adjoint(cin, case):
    """<im2col(x), P> = <x, gather(P)> to fp32 rounding (x on a grid the bf16 operand holds exactly, pooled means
    included), and the fake-half form (batch0) writes the second half only."""
    from rave_b200 import ops
    period, pool, K, stride, pad = case
    Bs, T = 4, 3000 + 7
    g = torch.Generator().manual_seed(31 * period + pool + K + cin)
    src = (torch.randint(-16, 17, (Bs, cin, T), generator=g).float() / 16).cuda()
    Lin = (T + period - 1) // period if period > 1 else T // pool
    Lout = (Lin + 2 * pad - K) // stride + 1
    W = ops.cin_width(cin, K)
    X = ops.im2col_cin(src, Lin, Lout, Lout, K, stride, pad, period, pool)
    P = torch.randn(X.shape, generator=g).cuda()
    dsrc = ops.gather_cin(P, (Bs, cin, T), Lin, Lout, K, stride, pad, period, pool)
    lhs = (X.double() * P.double()).sum()
    rhs = (src.double() * dsrc.double()).sum()
    assert abs(float(lhs - rhs)) <= 1e-5 * float((X.double() * P.double()).abs().sum()), (float(lhs), float(rhs))
    half = Bs // 2
    R_half = half * period
    d_half = ops.gather_cin(P[R_half:].contiguous(), (Bs, cin, T), Lin, Lout, K, stride, pad, period, pool, batch0=half)
    assert float(d_half[:half].abs().max()) == 0.0
    assert torch.equal(d_half[half:], dsrc[half:])
    if cin == 1:
        d1 = ops.gather_c1(P, (Bs, T), Lin, Lout, K, stride, pad, period, pool)
        assert torch.equal(d1, dsrc[:, 0])
        assert W == 16


@pytest.mark.parametrize("net,period,pool", [("msd", 1, 1), ("msd", 1, 2), ("msd", 1, 4), ("mpd", 2, 1),
                                             ("mpd", 11, 1)])
def test_stereo_first_layer_chain_vs_oracle(net, period, pool):
    """The first conv of a stereo ConvNet (capacity 16) as a one-layer bf16 chain reading [B, 2, T] in place: forward,
    input gradient (dgrad + gather) and weight gradient (wgrad of the G diagonal blocks) against F.conv1d / F.conv2d."""
    import rave_b200
    from rave_b200 import configs, engine
    torch.manual_seed(5)
    disc = configs.make_discriminator_v2(capacity=16, n_channels=2)
    layer = disc.discriminators[0 if net == "mpd" else 1].layers[0]
    conv = layer.net[0]
    B, T = 4, 16384 + 5
    x = (0.5 * torch.randn(B, 2, T)).clamp(-1, 1)
    xo = x.clone().requires_grad_(True)
    po = {k: v.detach().clone().requires_grad_(True) for k, v in conv.state_dict().items()}
    w = O.weight_norm(po["weight_v"], po["weight_g"])
    if net == "mpd":
        want = F.conv2d(O.mpd_fold(xo, period), w, po["bias"], conv.stride, conv.padding)
        want_cl = want.permute(0, 3, 2, 1).reshape(B * period, want.shape[2], want.shape[1])
        L = (T + period - 1) // period
    else:
        want = F.conv1d(F.avg_pool1d(xo, pool) if pool > 1 else xo, w, po["bias"], conv.stride, conv.padding)
        want_cl = want.permute(0, 2, 1)
        L = T // pool
    probe = torch.randn(want_cl.shape)
    names = ["weight_v", "weight_g", "bias"]
    g_o = torch.autograd.grad((want_cl * probe).sum(), [xo] + [po[k] for k in names])
    layer.cuda()
    rave_b200.set_precision("bf16")
    try:
        spec = layer._tc_specs()[0]
        xe = x.cuda().requires_grad_(True)
        (out,) = engine.run_chain(xe, [spec], L, src=(period, pool))
        got = out[:, :engine.chain_lengths([spec], L)[0], :spec.Cout]
        pg = dict(conv.named_parameters())
        g = torch.autograd.grad((got * probe.cuda()).sum(), [xe] + [pg[k] for k in names])
        torch.cuda.synchronize()
    finally:
        rave_b200.set_precision("fp32")
    assert got.shape == want_cl.shape
    assert rel_l2(got, want_cl) < 1e-2, rel_l2(got, want_cl)
    for k, a, b in zip(["x"] + names, g, g_o):
        assert a.shape == b.shape and rel_l2(a, b) < 2e-2, (k, rel_l2(a, b))


def test_stereo_v2_discriminator_fused_fm_bf16(monkeypatch):
    """v2 discriminator at capacity 16 on a stereo [real; fake] batch: the fused feature-matching path runs (first layers
    through rave_im2col_cin, no fp32 conv launch) and its losses and input gradient match the oracle and the generic
    engine path (per-layer features through RAVE's reference arithmetic)."""
    import rave_b200
    from rave_b200 import _lib, configs
    torch.manual_seed(5)
    m = configs.build_rave("v2", capacity=16, latent_size=16, disc_capacity=16, n_channels=2).cuda().train()
    sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items() if k.startswith("discriminator.")}
    xy = (0.5 * torch.randn(4, 2, 16384 + 3)).clamp(-1, 1)
    xo = xy.clone().requires_grad_(True)
    fm_o, ld_o, la_o = O.gan_losses(O.combine_discriminators_v2(xo, sd), 1, True)
    (gx_o,) = torch.autograd.grad(20 * fm_o + ld_o + la_o, xo)
    rave_b200.set_precision("bf16")
    _lib.PROFILE = []
    try:
        xg = xy.cuda().requires_grad_(True)
        assert m.discriminator.supports_fused_fm(xg)
        fm, ld, la, _, _ = m._fused_feature_matching(xg)
        (gx,) = torch.autograd.grad(20 * fm + ld + la, xg)
        torch.cuda.synchronize()
        launched = {name for name, *_ in _lib.PROFILE}
        _lib.PROFILE = None
        xh = xy.cuda().requires_grad_(True)
        fm_h, ld_h, la_h = O.gan_losses(m.discriminator(xh), 1, True)
        (gx_h,) = torch.autograd.grad(20 * fm_h + ld_h + la_h, xh)
    finally:
        _lib.PROFILE = None
        rave_b200.set_precision("fp32")
    assert "rave_im2col_cin" in launched and "rave_gather_cin" in launched
    assert not (launched & FP32_CONVS), launched & FP32_CONVS
    for got, want in ((fm, fm_o), (ld, ld_o)):
        assert rel_l2(got, want) < 3e-2
    assert abs(float(la) - float(la_o)) < 5e-2 * max(1.0, abs(float(la_o)))
    for got, want in ((fm, fm_h), (ld, ld_h)):
        assert rel_l2(got, want.cpu()) < 3e-2
    assert cos(gx, gx_o) > 0.95, cos(gx, gx_o)
    assert cos(gx, gx_h) > 0.95, cos(gx, gx_h)


def test_stereo_descript_discriminator_bf16_vs_oracle(monkeypatch):
    """DescriptDiscriminator in stereo, bf16: the 5 MPDs read the folded stereo rows through rave_im2col_cin, the 3 MRDs
    run channel-last on the interleaved [B, t, f, (c re/im)] spectrogram; no fp32 conv runs.  Features and gradients
    against the oracle."""
    import rave_b200
    from rave_b200.descript_discriminator import DescriptDiscriminator
    torch.manual_seed(1)
    dd = DescriptDiscriminator(n_channels=2)
    sd = {"discriminator." + k: v.detach().clone() for k, v in dd.state_dict().items()}
    x = (0.5 * torch.randn(2, 2, 8192 + 5)).clamp(-1, 1)
    po = {k: v.clone().requires_grad_(v.is_floating_point() and "window" not in k) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    want = O.descript_discriminator(xo, po)
    probes = [[torch.randn_like(b) for b in s] for s in want]
    names = sorted(k for k, v in po.items() if v.requires_grad)
    tot_o = sum((b * p).sum() for s, ps in zip(want, probes) for b, p in zip(s, ps))
    g_o = torch.autograd.grad(tot_o, [xo] + [po[k] for k in names])
    dd.cuda()
    _no_fp32_convs(monkeypatch)
    rave_b200.set_precision("bf16")
    try:
        xg = x.cuda().requires_grad_(True)
        got = dd(xg)
        assert [len(f) for f in got] == [6] * 5 + [26] * 3
        for fa, fb in zip(got, want):
            for a, b in zip(fa, fb):
                assert a.shape == b.shape and rel_l2(a, b) < 3e-2, (a.shape, rel_l2(a, b))
        pg = dict(dd.named_parameters(prefix="discriminator"))
        tot = sum((a * p.cuda()).sum() for s, ps in zip(got, probes) for a, p in zip(s, ps))
        g = torch.autograd.grad(tot, [xg] + [pg[k] for k in names])
        torch.cuda.synchronize()
    finally:
        rave_b200.set_precision("fp32")
    assert cos(g[0], g_o[0]) > 0.98, cos(g[0], g_o[0])
    ga = torch.cat([a.detach().cpu().reshape(-1) for a in g[1:]])
    gb = torch.cat([b.reshape(-1) for b in g_o[1:]])
    assert cos(ga, gb) > 0.99, cos(ga, gb)


def _run_golden_steps(kind, precision):
    """Replays tests/golden/training_step_{kind}_stereo_tiny.pt (a phase-2 D-step and G-step of the reference's own
    RAVE.training_step at n_channels = 2, both from the same seeded parameters) through rave_b200.RAVE.training_step."""
    import rave_b200
    from rave_b200 import configs
    g = load(f"training_step_{kind}_stereo_tiny.pt")
    cfg = g["cfg"]
    m = configs.build_rave(kind, capacity=cfg["capacity"], latent_size=cfg["latent_size"],
                           disc_capacity=g["disc_capacity"], phase_1_duration=1000, n_channels=cfg["n_channels"])
    m.update_discriminator_every = g["update_discriminator_every"]
    sd0 = dict(m.state_dict(), **ST.seeded_params(g["param_shapes"], g["param_seed"]))
    m.cuda().train()
    Lz = g["T"] // cfg["n_band"] // math.prod(cfg["ratios"])
    rave_b200.set_precision(precision)
    out = []
    try:
        for st in g["steps"]:
            m.load_state_dict(sd0, strict=True)
            m.set_receptive_field(*g["receptive_field"])
            m.warmed_up = True
            for p in m.parameters():
                p.grad = None
            x = ST.step_batch(g["B"], g["T"], st["seed"], cfg["n_channels"]).cuda()
            eps = ST.step_eps(g["B"], cfg["latent_size"], Lz, st["seed"]).cuda()
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


@pytest.mark.parametrize("kind", ["v2", "v3"])
def test_stereo_training_step_matches_reference_goldens_fp32(kind):
    """Logged losses <= 1e-4 of the reference's; the sampled gradient of the stepped group in direction (cos > 0.99)."""
    g, out = _run_golden_steps(kind, "fp32")
    for st, (logs, gs) in zip(g["steps"], out):
        for k, want in st["logs"].items():
            if k == "beta_factor":
                continue
            assert k in logs, (st["name"], k)
            assert abs(float(logs[k]) - float(want)) <= 1e-4 * max(abs(float(want)), 1e-3), (st["name"], k,
                                                                                              float(logs[k]), float(want))
        c = cos(gs, st["grad_sample"][2])
        print(f"{kind} {st['name']} (fp32): gradient sample cos {c:.6f}")
        assert c > 0.99, (st["name"], c)


@pytest.mark.parametrize("kind", ["v2", "v3"])
def test_stereo_training_step_matches_reference_goldens_bf16(kind):
    """Within the bounds of test_gpu_parity.py::test_training_step_matches_reference_goldens_bf16."""
    g, out = _run_golden_steps(kind, "bf16")
    for st, (logs, gs) in zip(g["steps"], out):
        for k, want in st["logs"].items():
            if k == "beta_factor":
                continue
            tol = 0.10 if k in ("feature_matching", "adversarial", "pred_fake", "pred_real") else 0.03
            assert abs(float(logs[k]) - float(want)) <= tol * max(abs(float(want)), 1e-3), (st["name"], k,
                                                                                           float(logs[k]), float(want))
        c = cos(gs, st["grad_sample"][2])
        print(f"{kind} {st['name']} (bf16): gradient sample cos {c:.4f}")
        assert c > 0.9, (st["name"], c)


def test_stereo_graphed_steps_match_eager_and_are_deterministic(monkeypatch):
    """bf16, stereo v2 at capacity 16 (the fused feature-matching path with multichannel first layers): GraphedTrainer
    replays == eager training_step on the same data, and two graphed runs from the same state are bit-identical."""
    import rave_b200
    from rave_b200 import configs, discriminator
    from rave_b200.graphs import GraphedTrainer
    monkeypatch.setattr(discriminator, "DISC_STREAMS", 1)
    torch.manual_seed(0)
    rave_b200.set_precision("bf16")
    try:
        m1 = configs.build_rave("v2", capacity=16, latent_size=16, disc_capacity=16, n_channels=2).cuda().train()
        m1.warmed_up = True
        m1.encoder.reparametrize = (lambda z, eps=None, enc=m1.encoder: type(enc).reparametrize(
            enc, z, torch.zeros_like(z[:, :z.shape[1] // 2])))
        m2, m3 = copy.deepcopy(m1), copy.deepcopy(m1)
        x = (0.5 * torch.randn(2, 2, 65536, device="cuda")).clamp(-1, 1)
        assert m1.discriminator.supports_fused_fm(torch.cat([x, x], 0))
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
    for k in ("fullband_spectral_distance", "multiband_spectral_distance", "feature_matching", "adversarial"):
        assert torch.equal(l2[k], l3[k]), k
        assert rel_l2(l2[k], l1[k]) < 2e-2, (k, float(l2[k]), float(l1[k]))
    for (n, p2), p3 in zip(m2.named_parameters(), m3.parameters()):
        assert torch.equal(p2, p3), n
    w = lambda m: m.discriminator.discriminators[1].layers[0].net[0].weight_v
    assert rel_l2(w(m2), w(m1)) < 1e-2

"""CPU: host logic of the tensor-core engine (rave_b200/engine.py) -- layer planning, transposed-conv /
strided-dgrad phase decomposition, row pitches, and the hand-written backward -- exercised against the
fp32 oracle with the kernels replaced by a torch emulation of their documented semantics
(tests/tc_emulator.py).  Tolerances are the bf16-mode ones (operands are rounded to bf16)."""
import pytest
import torch
import torch.nn as nn

from oracle import rave_oracle as O
from tests import tc_emulator
from tests.conftest import rel_l2


def cos(a, b):
    a, b = a.detach().double().reshape(-1), b.detach().double().reshape(-1)
    return (a @ b / (a.norm() * b.norm()).clamp_min(1e-30)).item()


@pytest.fixture(params=["exact_fp32", "bf16"])
def emu(request, monkeypatch):
    """exact_fp32: operands kept in fp32 -> the engine must reproduce the oracle to fp32 round-off (a pure
    logic check); bf16: operands/gradients rounded like on the device (tolerances of the bf16 mode)."""
    from rave_b200 import engine
    tc_emulator.install(monkeypatch)
    dt = torch.float32 if request.param == "exact_fp32" else torch.bfloat16
    monkeypatch.setattr(tc_emulator, "OPERAND_DTYPE", dt)
    monkeypatch.setattr(engine, "ACT_DTYPE", dt)
    return request.param


def tol(mode, exact, loose):
    return exact if mode == "exact_fp32" else loose


def test_phase_taps_cover_every_tap_once():
    from rave_b200.engine import _phase_taps
    for K, s, pad in [(8, 4, 3), (4, 2, 1), (8, 4, 2), (4, 2, 1), (15, 4, 7), (5, 4, 2), (5, 3, 2), (6, 2, 1)]:
        seen = []
        for p in range(s):
            order, padpp = _phase_taps(K, s, pad, p)
            for i, k in enumerate(order):
                # source row of tap i for output q: q + i - padpp must equal (q*s + p + pad - k)/s
                assert (p + pad - k) % s == 0
                assert i - padpp == (p + pad - k) // s
            seen += order
        assert sorted(seen) == list(range(K))


@pytest.mark.parametrize("name,ratios", [("v2", [4, 4, 4, 2]), ("v2", [4, 2, 2, 2]), ("v3", [4, 4, 4, 2])])
def test_encoder_generator_chain_vs_oracle(emu, name, ratios):
    """v3 = Snake activations (channel-last Snake kernels between the convs, alpha gradients, raw-stream skips) + AdaIN
    (identity in training)."""
    from rave_b200 import configs, engine
    torch.manual_seed(1)
    _, enc, dec = configs.make_autoencoder(name, capacity=16, latent_size=16, ratios=ratios)
    enc.train()
    dec.train()
    sd = {"encoder." + k: v.detach().clone() for k, v in enc.state_dict().items()}
    sd.update({"decoder." + k: v.detach().clone() for k, v in dec.state_dict().items()})
    cfg = O.ArchConfig(capacity=16, latent_size=16, ratios=ratios, activation="snake" if name == "v3" else "leaky",
                       adain=name == "v3")
    trainable = {"encoder." + k for k, _ in enc.named_parameters()} | {"decoder." + k for k, _ in dec.named_parameters()}
    B, L = 2, 512
    x_mb = torch.randn(B, 16, L)
    # ---------------- encoder
    specs = enc.encoder.net._tc_plan()
    assert specs is not None
    po = {k: v.clone().requires_grad_(k in trainable) for k, v in sd.items()}
    xo = x_mb.clone().requires_grad_(True)
    z_o = O.encoder_v2(xo, po, "encoder.encoder.", cfg)
    xe = x_mb.clone().requires_grad_(True)
    (out,) = engine.run_chain(engine.to_channel_last(xe), specs)
    z = engine.from_channel_last(out[:, :engine.chain_lengths(specs, L)[-1]].contiguous())
    assert z.shape == z_o.shape
    assert rel_l2(z, z_o) < tol(emu, 1e-5, 3e-2)
    probe = torch.randn_like(z_o)
    names = sorted(k for k in po if k.startswith("encoder.") and po[k].requires_grad)
    g_o = torch.autograd.grad((z_o * probe).sum(), [xo] + [po[k] for k in names])
    pe = dict(enc.named_parameters(prefix="encoder"))
    g_e = torch.autograd.grad((z * probe).sum(), [xe] + [pe[k] for k in names])
    assert rel_l2(g_e[0], g_o[0]) < tol(emu, 1e-5, 0.15)
    for k, a, b in zip(names, g_e[1:], g_o[1:]):
        assert a.shape == b.shape and rel_l2(a, b) < tol(emu, 2e-5, 0.2), (k, rel_l2(a, b))
    # ---------------- generator (up to the waveform conv, before x*sigmoid(a) -> tanh)
    specs = dec.net._tc_plan()
    zin = torch.randn(B, 16, z_o.shape[-1])
    taps = {}
    zo = zin.clone().requires_grad_(True)
    O.generator_v2(zo, po, "decoder.", cfg, taps)
    w_o = taps["wave"]
    ze = zin.clone().requires_grad_(True)
    (out,) = engine.run_chain(engine.to_channel_last(ze), specs)
    w = engine.from_channel_last(out[:, :engine.chain_lengths(specs, zin.shape[-1])[-1]].contiguous())
    assert w.shape == w_o.shape
    assert rel_l2(w, w_o) < tol(emu, 1e-5, 3e-2)
    probe = torch.randn_like(w_o)
    names = sorted(k for k in po if k.startswith("decoder.") and po[k].requires_grad)
    g_o = torch.autograd.grad((w_o * probe).sum(), [zo] + [po[k] for k in names])
    pd = dict(dec.named_parameters(prefix="decoder"))
    g_e = torch.autograd.grad((w * probe).sum(), [ze] + [pd[k] for k in names])
    assert rel_l2(g_e[0], g_o[0]) < tol(emu, 1e-5, 0.15)
    for k, a, b in zip(names, g_e[1:], g_o[1:]):
        assert a.shape == b.shape and rel_l2(a, b) < tol(emu, 2e-5, 0.2), (k, rel_l2(a, b))


def test_discriminator_chain_vs_oracle(emu):
    """MPD (folded, ragged lengths -> row pitches) and MSD ConvNets through the engine."""
    from rave_b200 import configs
    torch.manual_seed(2)
    disc = configs.make_discriminator_v2(capacity=16)
    sd = {"discriminator." + k: v.detach().clone() for k, v in disc.state_dict().items()}
    x = (0.5 * torch.randn(2, 1, 2048 + 3)).clamp(-1, 1)
    po = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    feats_o = O.combine_discriminators_v2(xo, po)
    xe = x.clone().requires_grad_(True)
    mpd, msd = disc.discriminators
    feats = []
    for layer, n in zip(mpd.layers, mpd.periods):
        feats.append(layer._forward_tc(mpd.fold(xe, n), layer._tc_specs()))
    xs = xe
    for layer in msd.layers:
        feats.append(layer._forward_tc(xs, layer._tc_specs()))
        xs = nn.functional.avg_pool1d(xs, 2)
    for fa, fb in zip(feats, feats_o):
        for a, b in zip(fa, fb):
            assert a.shape == b.shape
            assert rel_l2(a, b) < tol(emu, 1e-5, 3e-2), (a.shape, rel_l2(a, b))
    fm_o, ld_o, la_o = O.gan_losses(feats_o, 1, True)
    fm, ld, la = O.gan_losses(feats, 1, True)
    names = sorted(po)
    g_o = torch.autograd.grad(fm_o + ld_o + la_o, [xo] + [po[k] for k in names])
    pp = dict(disc.named_parameters(prefix="discriminator"))
    g_e = torch.autograd.grad(fm + ld + la, [xe] + [pp[k] for k in names])
    assert rel_l2(g_e[0], g_o[0]) < tol(emu, 2e-5, 0.2)
    for k, a, b in zip(names, g_e[1:], g_o[1:]):
        assert a.shape == b.shape and rel_l2(a, b) < tol(emu, 5e-5, 0.25), (k, rel_l2(a, b))


def test_fused_feature_matching_vs_oracle(emu):
    """RAVE._fused_feature_matching (stats computed by the engine from its operand stream) reproduces
    the reference's discrimination block (rave/model.py:348-379) and its gradients."""
    from functools import partial
    from rave_b200 import configs, core, engine
    torch.manual_seed(4)
    disc = configs.make_discriminator_v2(capacity=16)
    sd = {"discriminator." + k: v.detach().clone() for k, v in disc.state_dict().items()}
    x = (0.5 * torch.randn(4, 1, 2048 + 5)).clamp(-1, 1)
    po = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    fm_o, ld_o, la_o = O.gan_losses(O.combine_discriminators_v2(xo, po), 1, True)

    class Holder:            # the slice of RAVE that _fused_feature_matching touches
        pass
    from rave_b200.model import RAVE
    h = Holder()
    h.discriminator = disc
    h.feature_matching_fun = partial(core.mean_difference, norm="L1", relative=True)
    h.num_skipped_features = 1
    h.gan_loss = core.hinge_gan
    h._fused_tail = lambda nets, relative, skip: RAVE._fused_tail(h, nets, relative, skip)
    disc.supports_fused_fm = lambda xy: True            # (the real check also demands CUDA + bf16 mode)
    xe = x.clone().requires_grad_(True)
    fm, ld, la, pr, pf = RAVE._fused_feature_matching(h, xe)
    t = tol(emu, 2e-5, 3e-2)
    assert rel_l2(fm, fm_o) < t and rel_l2(ld, ld_o) < t and rel_l2(la, la_o) < t
    names = sorted(po)
    g_o = torch.autograd.grad(20 * fm_o + ld_o + la_o, [xo] + [po[k] for k in names], retain_graph=True)
    pp = dict(disc.named_parameters(prefix="discriminator"))
    g_e = torch.autograd.grad(20 * fm + ld + la, [xe] + [pp[k] for k in names])
    assert rel_l2(g_e[0], g_o[0]) < tol(emu, 5e-5, 0.25)
    for k, a, b in zip(names, g_e[1:], g_o[1:]):
        assert a.shape == b.shape and rel_l2(a, b) < tol(emu, 1e-4, 0.3), (k, rel_l2(a, b))
    # generator step: frozen discriminator, only the FAKE half's input gradient is wanted -> the backward runs on
    # that half alone; it must reproduce the oracle's gradient there (and leave the real half at zero)
    for p_ in disc.parameters():
        p_.requires_grad_(False)
    xf = x.clone().requires_grad_(True)
    fm2, ld2, la2, _, _ = RAVE._fused_feature_matching(h, xf, fake_grad_only=True)
    assert rel_l2(fm2, fm_o) < t and rel_l2(la2, la_o) < t
    (gf,) = torch.autograd.grad(20 * fm2 + la2, xf)
    (go,) = torch.autograd.grad(20 * fm_o + la_o, xo)
    half = x.shape[0] // 2
    assert float(gf[:half].abs().max()) == 0.0
    assert rel_l2(gf[half:], go[half:]) < tol(emu, 5e-5, 0.25)


@pytest.mark.parametrize("K,stride,pad", [(15, 4, 7), (5, 4, 2), (8, 4, 2), (4, 2, 1), (16, 8, 4), (7, 3, 3)])
def test_phase_fused_taps_reproduce_transposed_map(K, stride, pad):
    """engine._fused_phase_taps: the J-tap stride-1 conv over rows of `stride` positions equals the transposed map
    t = l*stride + k - pad (dgrad of a strided conv / forward of a transposed conv), checked on scalar 'channels'."""
    from rave_b200 import engine
    taps, J, pad_l = engine._fused_phase_taps(K, stride, pad)
    assert len(taps) == J * stride
    g = torch.Generator().manual_seed(K * 100 + stride)
    Lsrc = 23
    src = torch.randn(Lsrc, generator=g, dtype=torch.float64)
    w = torch.randn(K, generator=g, dtype=torch.float64)
    Lout = (Lsrc - 1) * stride - 2 * pad + K
    ref = torch.zeros(Lout + 4 * stride, dtype=torch.float64)
    for l in range(Lsrc):
        for k in range(K):
            t = l * stride + k - pad
            if 0 <= t < Lout:
                ref[t] += src[l] * w[k]
    got = torch.zeros_like(ref)
    rows = (Lout + stride - 1) // stride
    for q in range(rows):
        for j in range(J):
            l = q + j - pad_l
            if not (0 <= l < Lsrc):
                continue
            for p in range(stride):
                k = taps[j * stride + p]
                if k >= 0 and q * stride + p < Lout:
                    got[q * stride + p] += src[l] * w[k]
    assert torch.allclose(got, ref, atol=1e-12)


@pytest.mark.parametrize("K,stride,pad", [(15, 4, 7), (5, 4, 2), (8, 4, 3), (4, 2, 1)])
def test_wide_wgrad_slots_cover_every_tap_once(K, stride, pad):
    """engine._wide_wgrad_taps: tap k of a strided layer reads row l + j(k) / channel block p(k) of the operand viewed
    with `stride` positions per row; the slots are distinct and decode back to l*stride + k - pad."""
    from rave_b200 import engine
    J, pad_l, slots = engine._wide_wgrad_taps(K, stride, pad)
    assert len(set(slots)) == K and max(slots) < J * stride
    for k, sl in enumerate(slots):
        j, p = sl // stride - pad_l, sl % stride
        for l in range(5):
            assert (l + j) * stride + p == l * stride + k - pad


def test_split_operand_chain_reaches_fp32_accuracy(monkeypatch):
    """bf16x3 (x = hi + lo, hi*hi + lo*hi + hi*lo in fp32): the encoder and generator chains through the engine with
    the kernels emulated must sit within 1e-4 rel-L2 of the fp32 oracle (the north-star tolerance; single-pass bf16
    gives ~1e-2) -- checks the planning / layouts of the split mode (weights [hi slabs | lo slabs], [hi | lo] rows,
    per-position pairs after a phase-fused transposed conv, residual recovered from hi + lo)."""
    from rave_b200 import configs, engine
    tc_emulator.install(monkeypatch)
    torch.manual_seed(1)
    _, enc, dec = configs.make_autoencoder("v2", capacity=16, latent_size=16)
    sd = {"encoder." + k: v.detach().clone() for k, v in enc.state_dict().items()}
    sd.update({"decoder." + k: v.detach().clone() for k, v in dec.state_dict().items()})
    cfg = O.ArchConfig(capacity=16, latent_size=16)
    B, L = 2, 512
    x_mb = torch.randn(B, 16, L)
    with torch.no_grad():
        specs = enc.encoder.net._tc_plan()
        z_o = O.encoder_v2(x_mb, sd, "encoder.encoder.", cfg)
        (out,) = engine.run_chain(engine.to_channel_last(x_mb, x3=True), specs, x3=True)
        z = engine.from_channel_last(out[:, :engine.chain_lengths(specs, L)[-1]].contiguous())
        assert z.shape == z_o.shape
        print("bf16x3 encoder rel-L2", rel_l2(z, z_o))
        assert rel_l2(z, z_o) < 5e-5
        specs = dec.net._tc_plan()
        zin = torch.randn(B, 16, z_o.shape[-1])
        taps = {}
        O.generator_v2(zin, sd, "decoder.", cfg, taps)
        (out,) = engine.run_chain(engine.to_channel_last(zin, x3=True), specs, x3=True)
        w = engine.from_channel_last(out[:, :engine.chain_lengths(specs, zin.shape[-1])[-1]].contiguous())
        print("bf16x3 generator rel-L2", rel_l2(w, taps["wave"]))
        assert rel_l2(w, taps["wave"]) < 5e-5


def test_fused_units_are_planned_and_match_the_two_launch_form(emu, monkeypatch):
    """The engine runs Residual(DilatedUnit) blocks of width 96 / 192 / 384 through ops.dilated_unit_tc (one launch);
    with the kernel's semantics emulated, forward and every gradient must equal the unfused chain (same arithmetic)."""
    from rave_b200 import configs, engine
    calls = []
    real = tc_emulator.dilated_unit_tc

    def spy(*a, **k):
        calls.append(a[0].shape)
        return real(*a, **k)
    from rave_b200 import ops
    monkeypatch.setattr(ops, "dilated_unit_tc", spy)
    torch.manual_seed(4)
    _, enc, dec = configs.make_autoencoder("v2", capacity=96, latent_size=16, ratios=[4, 2])
    x_mb = torch.randn(1, 16, 256)
    outs = {}
    for fuse in (True, False):
        monkeypatch.setattr(engine, "FUSE_UNITS", fuse)
        if emu == "bf16":
            monkeypatch.setattr(engine, "ACT_DTYPE", torch.bfloat16)
        specs = enc.encoder.net._tc_plan()
        xe = x_mb.clone().requires_grad_(True)
        n0 = len(calls)
        (out,) = engine.run_chain(engine.to_channel_last(xe), specs)
        z = engine.from_channel_last(out[:, :engine.chain_lengths(specs, 256)[-1]].contiguous())
        pe = dict(enc.named_parameters())
        names = sorted(pe)
        g = torch.autograd.grad((z * torch.ones_like(z)).sum(), [xe] + [pe[k] for k in names])
        outs[fuse] = (z.detach(), [t.detach() for t in g], len(calls) - n0)
    if emu == "bf16":
        assert outs[True][2] == 6 and outs[False][2] == 0          # 3 units at C = 96, 3 at C = 192
        assert torch.equal(outs[True][0], outs[False][0])
        for a, b in zip(outs[True][1], outs[False][1]):
            assert torch.equal(a, b)
    else:
        assert outs[True][2] == 0               # fp32 operand emulation: the fused kernel is a bf16 kernel


def test_descript_mpd_chain_vs_oracle(emu):
    """v3 discriminator, MPD half: the whole period net as one engine chain (stride-3 k5 convs, slope 0.1, features =
    activation of each conv's output, Cin = 1 first layer reading the reflect-padded folded signal) against
    O.descript_mpd, features and gradients."""
    from rave_b200.descript_discriminator import MPD
    from rave_b200 import engine
    torch.manual_seed(4)
    period = 3
    mpd = MPD(period)
    # small channel counts keep the CPU test quick; same code path as the 1024-channel nets
    sd = {k: v.detach().clone() for k, v in mpd.state_dict().items()}
    x = (0.5 * torch.randn(2, 1, 2000)).clamp(-1, 1)
    po = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    want = O.descript_mpd(xo, po, "", period)
    specs = mpd._tc_specs()
    assert specs is not None
    xe = x.clone().requires_grad_(True)
    xp = mpd.pad_to_period(xe)
    got = mpd._forward_tc(xp.reshape(xp.shape[0], 1, -1, period), specs)
    assert len(got) == len(want) == 6
    for a, b in zip(got, want):
        assert a.shape == b.shape and rel_l2(a, b) < tol(emu, 1e-5, 3e-2), (a.shape, rel_l2(a, b))
    probes = [torch.randn_like(b) for b in want]
    names = sorted(po)
    g_o = torch.autograd.grad(sum((b * p).sum() for b, p in zip(want, probes)), [xo] + [po[k] for k in names])
    pg = dict(mpd.named_parameters())
    g_e = torch.autograd.grad(sum((a * p).sum() for a, p in zip(got, probes)), [xe] + [pg[k] for k in names])
    assert rel_l2(g_e[0], g_o[0]) < tol(emu, 2e-5, 0.15)
    for k, a, b in zip(names, g_e[1:], g_o[1:]):
        assert a.shape == b.shape
        if emu == "exact_fp32" or a.numel() >= 64:       # (the 1-element weight_g of conv_post is noise in bf16)
            assert rel_l2(a, b) < tol(emu, 5e-5, 0.2), (k, rel_l2(a, b))
    assert cos(torch.cat([a.reshape(-1) for a in g_e[1:]]), torch.cat([b.reshape(-1) for b in g_o[1:]])) > 0.99


def test_static_prepared_weights_follow_refresh(emu):
    """engine.enable_static_prep: a chain keeps using its persistent prepared weights until refresh_static_prep rewrites
    them in place (what GraphedTrainer relies on for the discriminator between D-steps, and the forward bench for the
    encoder / generator)."""
    from rave_b200 import configs, engine
    if emu != "bf16":
        pytest.skip("static prepared weights exist for the bf16 operand mode only")
    torch.manual_seed(7)
    _, enc, _ = configs.make_autoencoder("v2", capacity=16, latent_size=16)
    net = enc.encoder.net
    specs = net._tc_plan()
    x = torch.randn(2, 16, 256)

    def run():
        with torch.no_grad():
            (out,) = engine.run_chain(engine.to_channel_last(x), specs)
        return out.clone()
    y0 = run()
    engine.enable_static_prep(net)
    try:
        assert torch.equal(run(), y0)                      # first static call prepares from the current parameters
        with torch.no_grad():
            for n, p in net.named_parameters():
                if not n.endswith("bias"):                 # biases are read live by the epilogue, not prepared
                    p.mul_(1.5)
        assert torch.equal(run(), y0)                      # parameters moved, the static buffers did not
        n = engine.refresh_static_prep(net)
        assert n > 0
        y1 = run()
        assert not torch.equal(y1, y0)
    finally:
        engine.disable_static_prep(net)
    engine.invalidate_prepared()
    assert torch.equal(run(), y1)                          # same as a cold preparation from the moved parameters


def test_static_prepared_weights_of_a_one_layer_proxy_chain(emu):
    """The MRD's DiscConv2d plans its conv on a proxy holding permuted COPIES of its parameters: static preparation must
    reach that proxy (enabled before or after the first forward) and the refresh must rebuild the copies first."""
    from rave_b200 import engine
    from rave_b200.descript_discriminator import WNConv2d
    if emu != "bf16":
        pytest.skip("static prepared weights exist for the bf16 operand mode only")
    torch.manual_seed(11)
    for enable_first in (True, False):
        conv = WNConv2d(32, 32, (3, 9), (1, 2), padding=(1, 4))[0]
        root = torch.nn.Sequential(conv)
        xs = torch.randn(6, 40, 96).to(engine.ACT_DTYPE)

        def run():
            with torch.no_grad():
                (out,) = engine.run_chain(xs, [conv._tc_chain_spec(32)], 40)
            return out.clone()
        if enable_first:
            engine.enable_static_prep(root)
            y0 = run()
        else:
            y0 = run()
            engine.enable_static_prep(root)
        try:
            assert torch.equal(run(), y0)
            assert conv.__dict__["_tc_proxy"].__dict__.get("_tc_static"), "the proxy holds the static layouts"
            with torch.no_grad():
                conv.weight_v.mul_(torch.linspace(0.5, 2.0, 9).view(1, 1, 1, 9))
                conv.weight_g.mul_(1.5)
            assert torch.equal(run(), y0)                  # parameters moved, the static buffers did not
            assert engine.refresh_static_prep(root) == 1
            y1 = run()
            assert not torch.equal(y1, y0)
        finally:
            engine.disable_static_prep(root)
        engine.invalidate_prepared()
        assert torch.equal(run(), y1)                      # same as a cold preparation from the moved parameters


def test_fake_rows_only_backward_on_a_frozen_plain_chain(emu):
    """engine.fake_rows_only: a frozen plain conv chain over [real; fake] rows (Descript MPD in a generator step) runs
    its backward on the fake half: same input gradient on the fake rows, zeros on the real rows; trainable parameters
    switch the shortcut off; the feature-matching sums of the feature taps match torch."""
    from rave_b200.descript_discriminator import MPD
    from rave_b200 import engine
    torch.manual_seed(9)
    period = 2
    mpd = MPD(period)
    specs = mpd._tc_specs()
    x = (0.5 * torch.randn(4, 1, 1200)).clamp(-1, 1)

    def run(flag, frozen):
        for p in mpd.parameters():
            p.requires_grad_(not frozen)
        xe = x.clone().requires_grad_(True)
        xp = mpd.pad_to_period(xe)
        with engine.fake_rows_only(flag):
            feats = mpd._forward_tc(xp.reshape(xp.shape[0], 1, -1, period), specs)
        loss = 0.
        for f in feats[:-1]:
            st = f._fm_stats
            want = torch.stack([(f[:2] - f[2:]).abs().sum(), f[:2].abs().sum()])
            assert rel_l2(st, want) < 1e-5
            loss = loss + st[0] / f[:2].numel() + 0.1 * st[1] / f[:2].numel()
        loss = loss - feats[-1][2:].mean()
        (g,) = torch.autograd.grad(loss, xe)
        return g
    g_full = run(False, True)
    g_half = run(True, True)
    assert torch.count_nonzero(g_half[:2]) == 0 and torch.count_nonzero(g_full[:2]) > 0
    assert rel_l2(g_half[2:], g_full[2:]) < 1e-6
    g_train = run(True, False)                       # trainable parameters: the full backward runs
    assert rel_l2(g_train, g_full) < 1e-6
    for p in mpd.parameters():
        p.requires_grad_(True)


def test_fake_rows_only_backward_of_a_plain_operand_chain(emu):
    """Chains whose first layer reads a bf16 operand (the MRD's one-layer chains): under engine.fake_rows_only the last
    dgrad writes the fake rows' gradient straight into the second half of the full [zeros; fake] buffer."""
    from rave_b200 import engine
    from rave_b200.descript_discriminator import WNConv2d
    torch.manual_seed(13)
    for stride in (1, 2):
        conv = WNConv2d(32, 32, (3, 9), (1, stride), padding=(1, 4))[0]
        for p in conv.parameters():
            p.requires_grad_(False)
        xs0 = torch.randn(8, 40, 96).to(engine.ACT_DTYPE)
        probe = torch.randn(8, engine.chain_lengths([conv._tc_chain_spec(32)], 40)[0], 32)

        def run(flag):
            xs = xs0.clone().requires_grad_(True)
            with engine.fake_rows_only(flag):
                (out,) = engine.run_chain(xs, [conv._tc_chain_spec(32)], 40)
            (g,) = torch.autograd.grad((out[:, :probe.shape[1]] * probe).sum(), xs)
            return g.float()
        g_full, g_half = run(False), run(True)
        assert g_half.shape == g_full.shape
        assert torch.count_nonzero(g_half[:4]) == 0 and torch.count_nonzero(g_full[:4]) > 0
        assert torch.equal(g_half[4:], g_full[4:])


def test_mrd_channel_last_engine_path_vs_oracle(emu, monkeypatch):
    """The MRD's engine path (channel-last end to end, one-layer chains, feature taps that also write the next conv's
    time-stacked operand) against the oracle's Conv2d form of rave/descript_discriminator.py:118-184: every feature and
    the input gradient; the fused tap + stack and the separate passes give the same numbers."""
    from rave_b200 import descript_discriminator
    from rave_b200.descript_discriminator import MRD
    torch.manual_seed(21)
    mrd = MRD(256)
    sd = {k: v.detach().clone() for k, v in mrd.state_dict().items()}
    x = (0.5 * torch.randn(4, 1, 2048)).clamp(-1, 1)
    xo = x.clone().requires_grad_(True)
    want = O.descript_mrd(xo, sd, "", 256)
    probes = [torch.randn_like(f) for f in want]
    (g_o,) = torch.autograd.grad(sum((f * p).sum() for f, p in zip(want, probes)), xo)
    res = {}
    for fuse in (True, False):
        monkeypatch.setattr(descript_discriminator, "FUSE_TAP_STACK", fuse)
        xe = x.clone().requires_grad_(True)
        got = mrd._forward_cl(xe)
        assert len(got) == len(want) == 26
        for i, (a, b) in enumerate(zip(got, want)):
            assert a.shape == b.shape, (i, a.shape, b.shape)
            assert rel_l2(a, b) < tol(emu, 2e-5, 3e-2), (fuse, i, rel_l2(a, b))
        for f in got[:-1]:                                   # the taps' own feature-matching sums
            st = f._fm_stats
            ref = torch.stack([(f[:2] - f[2:]).abs().sum(), f[:2].abs().sum()])
            assert rel_l2(st, ref) < 1e-5
        (g_e,) = torch.autograd.grad(sum((f * p).sum() for f, p in zip(got, probes)), xe)
        assert rel_l2(g_e, g_o) < tol(emu, 5e-5, 0.1), (fuse, rel_l2(g_e, g_o))
        res[fuse] = ([f.detach().clone() for f in got], g_e)
    for a, b in zip(res[True][0], res[False][0]):
        assert torch.equal(a, b)
    assert rel_l2(res[True][1], res[False][1]) < 1e-6

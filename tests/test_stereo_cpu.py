"""CPU: multichannel (stereo, n_channels = 2) models -- module trees against the reference's, the oracle restatement
against the reference's stereo fixtures, and the engine's multichannel first layer (raw signal read in place through the
MPD fold / MSD pooling, operand rows of W = 16 or 32 columns) with the kernels emulated (tests/tc_emulator.py)."""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import rave_oracle as O
from oracle import stereo_oracle as ST
from tests import tc_emulator
from tests.conftest import GOLDEN, rel_l2


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def cos(a, b):
    a, b = a.detach().double().reshape(-1), b.detach().double().reshape(-1)
    return (a @ b / (a.norm() * b.norm()).clamp_min(1e-30)).item()


@pytest.mark.parametrize("name", ["v2", "v3"])
def test_stereo_state_dict_matches_reference(name):
    from rave_b200 import configs
    want = _load("state_dict_keys_stereo.pt")["rave_" + name]
    m = configs.build_rave(name, n_channels=2)
    got = {k: (tuple(v.shape), str(v.dtype)) for k, v in m.state_dict().items()}
    assert list(got) == list(want)
    assert got == want


def test_oracle_stereo_discriminator_vs_fixture():
    fx = _load("discriminator_v2_stereo.pt")
    po = {k: v.clone().requires_grad_(True) for k, v in fx["state_dict"].items()}
    x = fx["x"].clone().requires_grad_(True)
    feats = O.combine_discriminators_v2(x, po)
    for fs, ws in zip(feats, fx["features"]):
        for f, (shape, idx, vals) in zip(fs, ws):
            assert tuple(f.shape) == tuple(shape)
            assert rel_l2(f.reshape(-1)[idx], vals) < 1e-6
    fm, ld, la = O.gan_losses(feats, 1, True)
    for got, want in ((fm, fx["fm"]), (ld, fx["loss_dis"]), (la, fx["loss_adv"])):
        assert rel_l2(got, want) < 1e-6
    g = torch.autograd.grad(fm + ld + la, [x] + [po[k] for k in fx["grad_keys"]])
    assert rel_l2(g[0], fx["grad_x"]) < 1e-5
    _, idx, vals = fx["grad_sample"]
    assert rel_l2(torch.cat([t.reshape(-1) for t in g[1:]])[idx], vals) < 1e-5


@pytest.mark.parametrize("kind", ["v2", "v3"])
def test_oracle_stereo_training_step_vs_fixture(kind):
    """The logged losses of both steps from the seeded parameters."""
    g = _load(f"training_step_{kind}_stereo_tiny.pt")
    cfg = O.ArchConfig(**g["cfg"])
    sd = dict(ST.seeded_params(g["param_shapes"], g["param_seed"]), **{"pqmf.hk": g["hk"]})
    Lz = g["T"] // cfg.n_band
    for r in cfg.ratios:
        Lz //= r
    for st in g["steps"]:
        x = ST.step_batch(g["B"], g["T"], st["seed"])
        eps = ST.step_eps(g["B"], cfg.latent_size, Lz, st["seed"])
        losses, loss_dis = ST.train_step_losses(x, sd, cfg, eps, kind, receptive_field=g["receptive_field"])
        for k, v in losses.items():
            assert rel_l2(v, st["logs"][k]) < 1e-5, (st["name"], k)
        assert rel_l2(loss_dis, st["logs"]["loss_dis"]) < 1e-5


# ---- the engine's multichannel first layer, kernels emulated ---------------------------------------------------------

def _im2col_cin(src, Lin, Lout, out_pitch, K, stride, pad_l, period=1, pool=1):
    """ops.im2col_cin: X[r, l, c*K + k] = row_{r,c}[l*stride + k - pad_l], W = ops.cin_width(cin, K) columns."""
    from rave_b200 import ops
    Bs, cin, T = src.shape
    W = ops.cin_width(cin, K)
    per_c = [tc_emulator.im2col_c1(src[:, c].contiguous(), Lin, Lout, out_pitch, K, stride, pad_l, period, pool).float()
             for c in range(cin)]
    X = torch.zeros(per_c[0].shape[0], out_pitch, W)
    for c, Xc in enumerate(per_c):
        X[:, :, c * K:(c + 1) * K] = Xc[:, :, :K]
    return tc_emulator._bf16(X)


def _gather_cin(P_cl, src_shape, Lin, Lout, K, stride, pad_l, period=1, pool=1, batch0=0):
    Bs, cin, T = src_shape
    P16 = torch.zeros(P_cl.shape[0], P_cl.shape[1], 16)
    out = []
    for c in range(cin):
        P16[:, :, :K] = P_cl[:, :, c * K:(c + 1) * K].float()
        out.append(tc_emulator.gather_c1(P16, (Bs, T), Lin, Lout, K, stride, pad_l, period, pool, batch0))
    return torch.stack(out, 1)


@pytest.fixture(params=["exact_fp32", "bf16"])
def emu(request, monkeypatch):
    from rave_b200 import engine, ops
    tc_emulator.install(monkeypatch)
    monkeypatch.setattr(ops, "im2col_cin", _im2col_cin)
    monkeypatch.setattr(ops, "gather_cin", _gather_cin)
    dt = torch.float32 if request.param == "exact_fp32" else torch.bfloat16
    monkeypatch.setattr(tc_emulator, "OPERAND_DTYPE", dt)
    monkeypatch.setattr(engine, "ACT_DTYPE", dt)
    return request.param


@pytest.mark.parametrize("net,period,pool", [("msd", 1, 1), ("msd", 1, 4), ("mpd", 3, 1), ("mpd", 11, 1)])
def test_stereo_first_layer_reads_the_signal_in_place(emu, net, period, pool):
    """The first conv of a stereo ConvNet as a one-layer chain on the raw [B, 2, T] signal: MSD (K = 15: 30 columns, W =
    32, G = 2 positions per row) on the signal average-pooled by `pool`, MPD (K = 5: 10 columns, W = 16, G = 4) on its
    fold by `period` -- forward, input gradient and weight gradient against F.conv1d / F.conv2d."""
    from rave_b200 import configs, engine, ops
    torch.manual_seed(5)
    disc = configs.make_discriminator_v2(capacity=16, n_channels=2)
    layer = disc.discriminators[0 if net == "mpd" else 1].layers[0]
    spec = layer._tc_specs()[0]
    assert spec.Cin == 2 and engine.raw_input_ok(spec, 2)
    assert ops.cin_width(2, spec.K) == (32 if net == "msd" else 16)
    conv = layer.net[0]
    B, T = 2, 1024 + 5
    x = (0.5 * torch.randn(B, 2, T)).clamp(-1, 1)
    xo = x.clone().requires_grad_(True)
    w = O.weight_norm(conv.weight_v, conv.weight_g)
    if net == "mpd":
        want = F.conv2d(O.mpd_fold(xo, period), w, conv.bias, conv.stride, conv.padding)        # [B, Co, L', period]
        want_cl = want.permute(0, 3, 2, 1).reshape(B * period, want.shape[2], want.shape[1])
        L = (T + period - 1) // period
    else:
        want = F.conv1d(F.avg_pool1d(xo, pool) if pool > 1 else xo, w.squeeze(-1) if w.dim() == 4 else w, conv.bias,
                        conv.stride, conv.padding)
        want_cl = want.permute(0, 2, 1)
        L = T // pool
    xe = x.clone().requires_grad_(True)
    (out,) = engine.run_chain(xe, [spec], L, src=(period, pool))
    Lo = engine.chain_lengths([spec], L)[0]
    got = out[:, :Lo, :spec.Cout]
    assert got.shape == want_cl.shape
    t = 1e-6 if emu == "exact_fp32" else 1e-2
    assert rel_l2(got, want_cl) < t
    probe = torch.randn(want_cl.shape)
    names = ["weight_v", "weight_g", "bias"]
    g_o = torch.autograd.grad((want_cl * probe).sum(), [xo, conv.weight_v, conv.weight_g, conv.bias])
    g_e = torch.autograd.grad((got * probe).sum(), [xe, conv.weight_v, conv.weight_g, conv.bias])
    t = 1e-6 if emu == "exact_fp32" else 2e-2
    for n, a, b in zip(["x"] + names, g_e, g_o):
        assert a.shape == b.shape and rel_l2(a, b) < t, (n, rel_l2(a, b))


def test_stereo_fused_feature_matching_vs_oracle(emu):
    """RAVE._fused_feature_matching on a stereo signal: all 8 ConvNets read [B, 2, T] in place (no fold / pool copy), the
    losses and the input / parameter gradients reproduce the reference's discrimination block; the generator-step form
    (fake rows only) too."""
    from functools import partial
    from rave_b200 import configs, core
    from rave_b200.model import RAVE
    torch.manual_seed(4)
    disc = configs.make_discriminator_v2(capacity=16, n_channels=2)
    sd = {"discriminator." + k: v.detach().clone() for k, v in disc.state_dict().items()}
    x = (0.5 * torch.randn(4, 2, 2048 + 5)).clamp(-1, 1)
    po = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    fm_o, ld_o, la_o = O.gan_losses(O.combine_discriminators_v2(xo, po), 1, True)

    class Holder:            # the slice of RAVE that _fused_feature_matching touches
        pass
    h = Holder()
    h.discriminator = disc
    h.feature_matching_fun = partial(core.mean_difference, norm="L1", relative=True)
    h.num_skipped_features = 1
    h.gan_loss = core.hinge_gan
    h._fused_tail = lambda nets, relative, skip: RAVE._fused_tail(h, nets, relative, skip)
    disc.supports_fused_fm = lambda xy: True            # (the real check also demands CUDA + bf16 mode)
    xe = x.clone().requires_grad_(True)
    fm, ld, la, _, _ = RAVE._fused_feature_matching(h, xe)
    t = 2e-5 if emu == "exact_fp32" else 3e-2
    assert rel_l2(fm, fm_o) < t and rel_l2(ld, ld_o) < t and rel_l2(la, la_o) < t
    names = sorted(po)
    g_o = torch.autograd.grad(20 * fm_o + ld_o + la_o, [xo] + [po[k] for k in names], retain_graph=True)
    pp = dict(disc.named_parameters(prefix="discriminator"))
    g_e = torch.autograd.grad(20 * fm + ld + la, [xe] + [pp[k] for k in names])
    assert rel_l2(g_e[0], g_o[0]) < (5e-5 if emu == "exact_fp32" else 0.25)
    for k, a, b in zip(names, g_e[1:], g_o[1:]):
        assert a.shape == b.shape
        if emu == "exact_fp32":
            assert rel_l2(a, b) < 1e-4, (k, rel_l2(a, b))
    # bf16: single deep-layer weights of this tiny net sit near the 0.3 noise floor, the whole gradient does not
    assert cos(torch.cat([a.reshape(-1) for a in g_e[1:]]), torch.cat([b.reshape(-1) for b in g_o[1:]])) > 0.97
    for p_ in disc.parameters():
        p_.requires_grad_(False)
    xf = x.clone().requires_grad_(True)
    fm2, _, la2, _, _ = RAVE._fused_feature_matching(h, xf, fake_grad_only=True)
    (gf,) = torch.autograd.grad(20 * fm2 + la2, xf)
    (go,) = torch.autograd.grad(20 * fm_o + la_o, xo)
    half = x.shape[0] // 2
    assert float(gf[:half].abs().max()) == 0.0
    assert rel_l2(gf[half:], go[half:]) < (5e-5 if emu == "exact_fp32" else 0.25)

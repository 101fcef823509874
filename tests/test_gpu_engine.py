"""GPU: the channel-last tensor-core ENGINE (bf16 mode) end to end against the fp32 CPU oracle.

Stated bf16-mode tolerances (operands rounded to bf16, fp32 accumulate; SURVEY 7.2 measures 8.7-9.6e-3
for operand rounding alone through the v2 autoencoder): forward rel-L2 <= 3e-2; gradients (bf16 operand AND
bf16 gradient streams through ~56 layers of a tiny, untrained, low-redundancy model) rel-L2 <= 0.2 and
cosine >= 0.98 -- tests/test_engine_cpu.py shows the same engine is exact (1e-6) when operands stay fp32."""
import pytest
import torch
import torch.nn as nn

from oracle import rave_oracle as O
from tests.conftest import rel_l2

pytestmark = pytest.mark.gpu

FWD_TOL = 3e-2
BWD_TOL = 0.2


def cos(a, b):
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    return (a @ b / (a.norm() * b.norm()).clamp_min(1e-30)).item()


@pytest.fixture(autouse=True)
def bf16_mode():
    import rave_b200
    rave_b200.set_precision("bf16")
    yield
    rave_b200.set_precision("fp32")


@pytest.mark.parametrize("name,ratios", [("v2", [4, 4, 4, 2]), ("v2", [4, 2, 2, 2]), ("v3", [4, 4, 4, 2])])
def test_autoencoder_bf16_vs_oracle(name, ratios):
    """v3: Snake + AdaIN chains on the wgmma kernels (rave_snake_cl_fwd / _bwd between the convs)."""
    from rave_b200 import configs
    from rave_b200.model import _pqmf_decode, _pqmf_encode
    torch.manual_seed(3)
    pq, enc, dec = configs.make_autoencoder(name, capacity=16, latent_size=16, ratios=ratios)
    enc.train()
    dec.train()
    assert enc.encoder.net._tc_plan() is not None and dec.net._tc_plan() is not None
    holder = nn.Module()
    holder.pqmf, holder.encoder, holder.decoder = pq, enc, dec
    sd = {k: v.detach().clone() for k, v in holder.state_dict().items()}
    T = 16384
    x = (0.5 * torch.randn(2, 1, T)).clamp(-1, 1)
    cfg = O.ArchConfig(capacity=16, latent_size=16, ratios=ratios, activation="snake" if name == "v3" else "leaky",
                       adain=name == "v3")
    trainable = {k for k, _ in holder.named_parameters()}
    Lz = T // 16
    for r in ratios:
        Lz //= r
    eps = torch.randn(2, 16, Lz)
    probe = torch.randn(2, 1, T)
    # oracle forward/backward (fp32 CPU)
    params_o = {k: v.clone().requires_grad_(k in trainable and not k.startswith("pqmf")) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    taps = {}
    y_o = O.rave_forward(xo, params_o, cfg, eps, taps)
    names = sorted(k for k, v in params_o.items() if v.requires_grad)
    grads_o = torch.autograd.grad((y_o * probe).sum(), [xo] + [params_o[k] for k in names])
    # engine
    holder.cuda().train()
    xg = x.cuda().requires_grad_(True)
    z = enc(_pqmf_encode(pq, xg))
    zs, _ = enc.reparametrize(z, eps.cuda())
    y = _pqmf_decode(pq, dec(zs), batch_size=xg.shape[:-2], n_channels=1)
    assert y.shape == y_o.shape
    assert rel_l2(z, taps["z"]) < FWD_TOL
    assert rel_l2(y, y_o) < FWD_TOL
    pg = dict(enc.named_parameters(prefix="encoder"))
    pg.update(dict(dec.named_parameters(prefix="decoder")))
    grads_g = torch.autograd.grad((y * probe.cuda()).sum(), [xg] + [pg[k] for k in names])
    assert rel_l2(grads_g[0], grads_o[0]) < BWD_TOL and cos(grads_g[0], grads_o[0]) > 0.98
    # all parameter gradients together, and each tensor on its own (the tiny weight_g tensors are noisy)
    ga = torch.cat([a.detach().cpu().reshape(-1) for a in grads_g[1:]])
    gb = torch.cat([b.reshape(-1) for b in grads_o[1:]])
    assert cos(ga, gb) > 0.99 and rel_l2(ga, gb) < 0.15
    for k, a, b in zip(names, grads_g[1:], grads_o[1:]):
        assert cos(a, b) > 0.93, (k, cos(a, b), rel_l2(a, b))


def test_discriminator_bf16_vs_oracle():
    from rave_b200 import configs
    torch.manual_seed(5)
    holder = nn.Module()
    holder.discriminator = configs.make_discriminator_v2(capacity=16)
    sd = {k: v.detach().clone() for k, v in holder.state_dict().items()}
    x = (0.5 * torch.randn(4, 1, 8192 + 3)).clamp(-1, 1)
    params_o = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    feats_o = O.combine_discriminators_v2(xo, params_o)
    fm_o, ld_o, la_o = O.gan_losses(feats_o, 1, True)
    names = sorted(params_o)
    grads_o = torch.autograd.grad(fm_o + ld_o + la_o, [xo] + [params_o[k] for k in names])
    disc = holder.discriminator.cuda()
    xg = x.cuda().requires_grad_(True)
    feats = disc(xg)
    assert len(feats) == 8
    for fa, fb in zip(feats, feats_o):
        assert len(fa) == 5
        for a, b in zip(fa, fb):
            assert a.shape == b.shape
            assert rel_l2(a, b) < FWD_TOL
    fm, ld, la = O.gan_losses(feats, 1, True)
    assert rel_l2(fm, fm_o) < FWD_TOL and rel_l2(ld, ld_o) < FWD_TOL
    pp = dict(disc.named_parameters(prefix="discriminator"))
    grads = torch.autograd.grad(fm + ld + la, [xg] + [pp[k] for k in names])
    assert cos(grads[0], grads_o[0]) > 0.98 and rel_l2(grads[0], grads_o[0]) < 0.2
    for k, a, b in zip(names, grads[1:], grads_o[1:]):
        assert cos(a, b) > 0.97, (k, cos(a, b), rel_l2(a, b))


def test_training_step_bf16_runs():
    import rave_b200
    from rave_b200 import _lib, configs
    torch.manual_seed(0)
    m = configs.build_rave("v2", capacity=16, latent_size=16, disc_capacity=16).cuda().train()
    x = (0.5 * torch.randn(2, 1, 65536, device="cuda")).clamp(-1, 1)
    w0 = m.decoder.net[0].weight_v.detach().clone()
    m.training_step(x, 1)
    assert not torch.equal(w0, m.decoder.net[0].weight_v)
    m.warmed_up = True
    d0 = m.discriminator.discriminators[1].layers[0].net[0].weight_v.detach().clone()
    logs = m.training_step(x, 0)
    assert not torch.equal(d0, m.discriminator.discriminators[1].layers[0].net[0].weight_v)
    logs = m.training_step(x, 1)
    for k in ("fullband_spectral_distance", "feature_matching", "adversarial", "loss_dis"):
        assert torch.isfinite(logs[k]), k


def test_fused_feature_matching_bf16_vs_oracle():
    """The fused discrimination block (no fp32 features in HBM) against the oracle's gan_losses."""
    from rave_b200 import configs
    torch.manual_seed(5)
    m = configs.build_rave("v2", capacity=16, latent_size=16, disc_capacity=16).cuda().train()
    sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items() if k.startswith("discriminator.")}
    xy = (0.5 * torch.randn(4, 1, 8192)).clamp(-1, 1)
    feats_o = O.combine_discriminators_v2(xy, sd)
    fm_o, ld_o, la_o = O.gan_losses(feats_o, 1, True)
    assert m.discriminator.supports_fused_fm(xy.cuda())
    fm, ld, la, pr, pf = m._fused_feature_matching(xy.cuda())
    assert rel_l2(fm, fm_o) < FWD_TOL and rel_l2(ld, ld_o) < FWD_TOL and rel_l2(la, la_o) < 5e-2


@pytest.mark.parametrize("streams", ["1", "8"])
def test_cuda_graph_training_matches_eager(streams, monkeypatch):
    """GraphedTrainer replays == eager training_step on the same data (same kernels, same order); with the
    discriminator nets captured on 8 side streams against a single-stream eager twin."""
    import copy
    monkeypatch.setenv("RAVE_DISC_STREAMS", streams)
    from rave_b200 import configs
    from rave_b200.graphs import GraphedTrainer
    torch.manual_seed(0)
    m1 = configs.build_rave("v2", capacity=16, latent_size=16, disc_capacity=16).cuda().train()
    m1.warmed_up = True
    m2 = copy.deepcopy(m1)
    x = (0.5 * torch.randn(2, 1, 65536, device="cuda")).clamp(-1, 1)
    # freeze the reparametrisation noise so both runs see the same numbers
    for m in (m1, m2):
        m.encoder.reparametrize = (lambda z, eps=None, enc=m.encoder: type(enc).reparametrize(enc, z, torch.zeros_like(z[:, :z.shape[1] // 2])))
    w_before = m2.decoder.net[0].weight_v.detach().clone()
    enc_before = [p.detach().clone() for p in m2.encoder.parameters()]
    tr = GraphedTrainer(m2, x, warmup_steps=2)
    # the trainer's eager warm-up is undone (parameters, buffers, optimiser state restored) and capture itself executes
    # nothing: the twin starts from the same state without any catching up
    assert torch.equal(w_before, m2.decoder.net[0].weight_v)
    monkeypatch.setenv("RAVE_DISC_STREAMS", "1")
    m1.optimizers(capturable=True)
    for i in range(4):
        la = tr.step(x, i)
        lb = m1.training_step(x, i)
    torch.cuda.synchronize()
    for k in ("fullband_spectral_distance", "feature_matching", "adversarial"):
        assert rel_l2(la[k], lb[k]) < 2e-2, (k, float(la[k]), float(lb[k]))
    w1 = m1.decoder.net[0].weight_v
    w2 = m2.decoder.net[0].weight_v
    assert rel_l2(w2, w1) < 1e-2
    # phase 2 never moves the encoder (detached latent: rave/blocks.py:739-743) -- what lets the trainer keep the encoder's
    # prepared weights in static buffers
    assert tr.static_encoder
    for (n, p), q in zip(m2.encoder.named_parameters(), enc_before):
        assert torch.equal(p, q), n
    for (n, p), q in zip(m1.encoder.named_parameters(), enc_before):
        assert torch.equal(p, q), n


# ------------------------------------------------------------------------------------ the benched configuration
def test_autoencoder_capacity96_bf16_vs_oracle():
    """BASELINE config 3's encoder / generator at FULL width (capacity 96: the 96/192/384/768-channel stages, 1536-channel
    up/down convs) and full length (T = 65536), bf16 engine against the fp32 CPU oracle, forward and every gradient.
    Also bounds the drift of the bf16 residual stream (the skip is recovered from the unit's bf16 operand) over the 11
    residual blocks of each stack.  Per-tensor numbers are printed (pytest -s)."""
    from rave_b200 import configs
    from rave_b200.model import _pqmf_decode, _pqmf_encode
    torch.manual_seed(0)
    pq, enc, dec = configs.make_autoencoder("v2")
    holder = nn.Module()
    holder.pqmf, holder.encoder, holder.decoder = pq, enc, dec
    sd = {k: v.detach().clone() for k, v in holder.state_dict().items()}
    B, T = 2, 65536
    x = (0.5 * torch.randn(B, 1, T, generator=torch.Generator().manual_seed(1234))).clamp(-1, 1)
    cfg = O.ArchConfig()
    eps = torch.randn(B, 128, 32, generator=torch.Generator().manual_seed(4321))
    probe = torch.randn(B, 1, T, generator=torch.Generator().manual_seed(7))
    params_o = {k: v.clone().requires_grad_(v.is_floating_point() and not k.startswith("pqmf")) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    taps = {}
    y_o = O.rave_forward(xo, params_o, cfg, eps, taps)
    names = sorted(k for k, v in params_o.items() if v.requires_grad)
    grads_o = torch.autograd.grad((y_o * probe).sum(), [xo] + [params_o[k] for k in names])
    holder.cuda().train()
    xg = x.cuda().requires_grad_(True)
    z = enc(_pqmf_encode(pq, xg))
    zs, _ = enc.reparametrize(z, eps.cuda())
    y = _pqmf_decode(pq, dec(zs), batch_size=xg.shape[:-2], n_channels=1)
    rz, ry = rel_l2(z, taps["z"]), rel_l2(y, y_o)
    print(f"capacity 96 bf16: z rel-L2 {rz:.3e}  y rel-L2 {ry:.3e}")
    assert rz < FWD_TOL and ry < FWD_TOL
    pg = dict(enc.named_parameters(prefix="encoder"))
    pg.update(dict(dec.named_parameters(prefix="decoder")))
    grads_g = torch.autograd.grad((y * probe.cuda()).sum(), [xg] + [pg[k] for k in names])
    print(f"  grad_x rel-L2 {rel_l2(grads_g[0], grads_o[0]):.3e} cos {cos(grads_g[0], grads_o[0]):.4f}")
    assert rel_l2(grads_g[0], grads_o[0]) < BWD_TOL and cos(grads_g[0], grads_o[0]) > 0.98
    ga = torch.cat([a.detach().cpu().reshape(-1) for a in grads_g[1:]])
    gb = torch.cat([b.reshape(-1) for b in grads_o[1:]])
    print(f"  all parameter gradients: rel-L2 {rel_l2(ga, gb):.3e} cos {cos(ga, gb):.4f}")
    assert cos(ga, gb) > 0.99 and rel_l2(ga, gb) < 0.15
    worst = min((cos(a, b), k) for k, a, b in zip(names, grads_g[1:], grads_o[1:]))
    print(f"  worst tensor: cos {worst[0]:.4f} ({worst[1]})")
    for k, a, b in zip(names, grads_g[1:], grads_o[1:]):
        assert cos(a, b) > 0.93, (k, cos(a, b), rel_l2(a, b))


def test_discriminator_capacity96_bf16_vs_oracle():
    """BASELINE config 3's MPD + MSD at capacity 96 (the 96/192/384/768-channel k15 / (5,1) layers), [real; fake] batch
    of 2 + 2 x 65536, fused feature-matching path of the bf16 engine against the oracle's losses and input gradient."""
    from rave_b200 import configs
    torch.manual_seed(5)
    m = configs.build_rave("v2").cuda().train()
    sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items() if k.startswith("discriminator.")}
    xy = (0.5 * torch.randn(4, 1, 65536, generator=torch.Generator().manual_seed(11))).clamp(-1, 1)
    xo = xy.clone().requires_grad_(True)
    feats_o = O.combine_discriminators_v2(xo, sd)
    fm_o, ld_o, la_o = O.gan_losses(feats_o, 1, True)
    (gx_o,) = torch.autograd.grad(20 * fm_o + la_o, xo)
    for p in m.discriminator.parameters():
        p.requires_grad_(False)                      # generator step: frozen discriminator
    xg = xy.cuda().requires_grad_(True)
    assert m.discriminator.supports_fused_fm(xg)
    fm, ld, la, pr, pf = m._fused_feature_matching(xg, fake_grad_only=True)
    print(f"capacity 96 disc bf16: fm {float(fm):.5f} vs {float(fm_o):.5f}; loss_dis {float(ld):.5f} vs {float(ld_o):.5f}; "
          f"adv {float(la):.5f} vs {float(la_o):.5f}")
    assert rel_l2(fm, fm_o) < FWD_TOL and rel_l2(ld, ld_o) < FWD_TOL and abs(float(la) - float(la_o)) < 5e-2 * max(1.0, abs(float(la_o)))
    (gx,) = torch.autograd.grad(20 * fm + la, xg)
    half = xy.shape[0] // 2
    c, r = cos(gx[half:], gx_o[half:]), rel_l2(gx[half:], gx_o[half:])
    print(f"  fake-half input gradient: cos {c:.4f} rel-L2 {r:.3e}")
    assert c > 0.9

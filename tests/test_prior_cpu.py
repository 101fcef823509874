"""CPU: the latent prior (rave_b200.prior) -- the restatement against the reference's fixtures, the module tree and
state_dict against the reference's, the receptive-field arithmetic, and the training-step plan of the new kernels
(torch emulations of csrc/prior.cu, kept here) against the reference's loss and gradients."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import prior_oracle as P
from tests.conftest import GOLDEN, rel_l2


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


@pytest.fixture(scope="module")
def fx():
    return _load("prior_tiny.pt")


def _tiny_rave(fx):
    from rave_b200 import configs
    v = fx["vae_cfg"]
    return configs.build_rave("v2", capacity=v["capacity"], latent_size=v["latent_size"], disc_capacity=4)


def _prior_sd(fx):
    return P.seeded_params(fx["prior_param_shapes"], fx["param_seed"] + 1)


def test_oracle_matches_golden(fx):
    R, D = fx["prior_cfg"]["resolution"], fx["D"]
    cls = P.latent_classes(fx["z"], fx["eps"], fx["latent_mean"], fx["latent_pca"], D, R)
    assert torch.equal(cls, fx["classes"])
    sd = {k: v.requires_grad_(True) for k, v in _prior_sd(fx).items()}
    taps = {}
    loss = P.loss(cls, sd, fx["prior_cfg"], D, taps)
    assert rel_l2(taps["logits"], fx["logits"]) < 1e-6
    assert rel_l2(loss, fx["loss"]) < 1e-6
    names = [k for k, _ in fx["prior_param_shapes"]]
    grads = torch.autograd.grad(loss, [sd[k] for k in names], allow_unused=True)
    for k, g in zip(names, grads):
        if fx["grads"][k] is None:
            assert g is None, k
        else:
            assert rel_l2(g, fx["grads"][k]) < 1e-5, k
    assert torch.equal(P.stack_one_hot(P.quantize(fx["quant_in"], R), R), fx["quant_enc"])
    assert torch.equal(P.diagonal_shift(fx["quant_in"]), fx["shift_fwd"])
    assert torch.equal(P.diagonal_shift_inverse(fx["quant_in"]), fx["shift_inv"])
    assert torch.equal(P.generate(fx["gen_in"], _prior_sd(fx), fx["prior_cfg"], D), fx["gen_out"])


def test_quantized_normal_and_shift_modules(fx):
    from rave_b200.prior import DiagonalShift, QuantizedNormal
    R = fx["prior_cfg"]["resolution"]
    qn = QuantizedNormal(R, dither=False)
    assert torch.equal(qn.encode(fx["quant_in"]), fx["quant_enc"])
    assert torch.allclose(qn.decode(fx["quant_enc"]), fx["quant_dec"], rtol=0, atol=1e-6)
    ds = DiagonalShift()
    assert torch.equal(ds(fx["quant_in"]), fx["shift_fwd"])
    assert torch.equal(ds.inverse(fx["quant_in"]), fx["shift_inv"])


def _own(sd_shapes):
    """The prior's own entries (the pretrained RAVE's, `synth.*`, are pinned by the RAVE's state_dict tests)."""
    return {k: v for k, v in sd_shapes.items() if not k.startswith("synth.")}


def test_state_dict_matches_reference():
    from rave_b200 import configs
    want = _load("state_dict_keys_prior.pt")
    m = configs.build_rave("v2")
    prior = configs.build_prior(m, latent_size=16)
    got = _own({k: tuple(v.shape) for k, v in prior.state_dict().items()})
    assert list(got) == list(_own(want["latent_size_16"]))
    assert got == _own(want["latent_size_16"])
    # a reference prior checkpoint's own entries load strictly into the prior's module tree
    own = {k: torch.zeros(s) for k, s in got.items()}
    sd = dict(prior.state_dict(), **own)
    prior.load_state_dict(sd, strict=True)
    f = want["fidelity"]
    m.fidelity.copy_(f["buffer"])
    pf = configs.build_prior(m, fidelity=f["value"])
    assert pf.latent_size == f["latent_size"]
    assert _own({k: tuple(v.shape) for k, v in pf.state_dict().items()}) == _own(f["shapes"])
    for name in ["pre_net.0", "post_net.0", "post_net.2"] + [f"residuals.{i}.{c}" for i in range(10)
                                                             for c in ("dconv", "rconv", "sconv")]:
        assert prior.get_submodule(name).bias is not None, name


def test_constructor_contract():
    from rave_b200 import configs
    from rave_b200.prior import VariationalPrior
    m = configs.build_rave("v2", capacity=8, latent_size=16, disc_capacity=4)
    assert configs.build_prior(m, latent_size=12).latent_size == 16          # rounded up to a power of two
    with pytest.raises(RuntimeError):
        configs.build_prior(m)
    w = configs.build_rave("v2_wasserstein", capacity=8, disc_capacity=4)
    with pytest.raises(NotImplementedError):
        VariationalPrior(32, 512, 256, 3, 4, 10, pretrained_vae=w, latent_size=8)
    p = configs.build_prior(m, latent_size=8, sr=44100)
    assert p.sr == 44100 and configs.build_prior(m, latent_size=8).sr == m.sr
    assert p.dilations == (1, 2, 4, 8, 1, 2, 4, 8, 1, 2)


def test_receptive_field_arithmetic(fx):
    from rave_b200 import configs
    m = configs.build_rave("v2")
    prior = configs.build_prior(m, latent_size=16)
    assert prior.get_model_ratio() == P.model_ratio(16, [4, 4, 4, 2]) == 2048
    assert prior.min_receptive_field == P.min_receptive_field(P.PRIOR_V1, 2048) == 262144
    assert prior.min_receptive_field == _load("state_dict_keys_prior.pt")["min_receptive_field"]
    tiny = configs.build_prior(_tiny_rave(fx), latent_size=fx["D"], **fx["prior_cfg"])
    assert tiny.get_model_ratio() == fx["model_ratio"]
    assert tiny.min_receptive_field == fx["min_receptive_field"]


def test_no_cpu_training_path(fx):
    from rave_b200 import _lib, configs
    prior = configs.build_prior(_tiny_rave(fx), latent_size=fx["D"], **fx["prior_cfg"])
    with pytest.raises(_lib.RaveB200Error):
        prior.step_loss(fx["classes"].permute(0, 2, 1).int().contiguous())


# ---------------------------------------------------------------------------------------------------------------------
# torch emulations of the kernels of csrc/prior.cu, on [B, C, T] fp32 (the parity layout), and the step plan of
# rave_b200/prior/model.py (_step_forward / _step_backward) written with them


def emu_latent_classes(z, eps, lmean, pca, D, R):
    """rave_prior_latent_classes -> [B, T', D]"""
    mean, scale = z.chunk(2, 1)
    s = eps * (F.softplus(scale) + 1e-4) + mean - lmean[:, None]
    y = torch.einsum("dc,bct->bdt", pca[:D], s)
    B, _, T = y.shape
    Tp = T - D + 1
    t = torch.arange(Tp)[None, :] + (D - 1 - torch.arange(D))[:, None]          # [D, T']
    ys = y.gather(2, t[None].expand(B, D, Tp))
    k = torch.floor(0.5 * (1 + torch.erf(ys / math.sqrt(2))) * R).clamp(0, R - 1).long()
    return k.permute(0, 2, 1)


def emu_embed_fwd(cls, w, b, slope=0.2):
    """rave_prior_embed_fwd: sum of gathered weight columns, then LeakyReLU -> [B, Cout, T']"""
    B, Tp, D = cls.shape
    Cout, R, K = w.shape
    d_of = torch.arange(Cout) // (Cout // D)
    y = b[None, :, None].expand(B, Cout, Tp).clone()
    for k in range(K):
        s = k - (K - 1)
        src = cls[:, :Tp - max(0, -s), :]                                         # class at t + s, t >= -s
        gathered = torch.stack([w[o, src[:, :, d_of[o]].long(), k] for o in range(Cout)], 1)   # [B, Cout, T'+s]
        y[:, :, max(0, -s):] += gathered
    return F.leaky_relu(y, slope)


def emu_embed_wgrad(cls, dout, x, w_shape, slope=0.2):
    B, Tp, D = cls.shape
    Cout, R, K = w_shape
    dy = dout * torch.where(x > 0, 1.0, slope)
    d_of = torch.arange(Cout) // (Cout // D)
    dw = torch.zeros(w_shape)
    for k in range(K):
        s = k - (K - 1)
        t0 = max(0, -s)
        src = cls[:, :Tp - t0, :]                                                  # source class of output t0..
        for o in range(Cout):
            oh = F.one_hot(src[:, :, d_of[o]].long(), R).to(dy.dtype)                     # [B, T'-t0, R]
            dw[o, :, k] = torch.einsum("btr,bt->r", oh, dy[:, o, t0:])
    return dw, dy.sum((0, 2))


def emu_gate_fwd(h):
    a, b = h.chunk(2, 1)
    return torch.sigmoid(a) * torch.tanh(b)


def emu_gate_bwd(dg, h):
    a, b = h.chunk(2, 1)
    s, t = torch.sigmoid(a), torch.tanh(b)
    return torch.cat([dg * t * s * (1 - s), dg * s * (1 - t * t)], 1)


def _head_logits(p, w, b, D, slope):
    x = F.leaky_relu(p, slope)
    return F.conv1d(x, w, b, groups=D)                                           # [B, R·D, T']


def emu_head_ce_fwd(p, w, b, cls, slope=0.2):
    B, Tp, D = cls.shape
    R = w.shape[0] // D
    lg = _head_logits(p, w, b, D, slope)[..., :-1].reshape(B, D, R, Tp - 1)
    return F.cross_entropy(lg.permute(0, 1, 3, 2).reshape(-1, R), cls[:, 1:, :].permute(0, 2, 1).reshape(-1).long())


def emu_head_ce_bwd(p, w, b, cls, gloss, slope=0.2):
    B, Tp, D = cls.shape
    R = w.shape[0] // D
    x = F.leaky_relu(p, slope)
    lg = F.conv1d(x, w, b, groups=D).reshape(B, D, R, Tp)
    sm = torch.softmax(lg, 2)
    tgt = F.one_hot(cls[:, 1:, :].permute(0, 2, 1).long(), R).permute(0, 1, 3, 2).to(sm.dtype)   # [B, D, R, T'-1]
    dl = torch.zeros_like(lg)
    dl[..., :-1] = gloss / (B * D * (Tp - 1)) * (sm[..., :-1] - tgt)
    dl = dl.reshape(B, D * R, Tp)
    Cg = w.shape[1]
    dx = torch.cat([torch.einsum("brt,rj->bjt", dl[:, d * R:(d + 1) * R], w[d * R:(d + 1) * R, :, 0])
                    for d in range(D)], 1)
    dx = dx * torch.where(p > 0, 1.0, slope)
    dw = torch.stack([torch.einsum("bt,bjt->j", dl[:, o], x[:, (o // R) * Cg:(o // R + 1) * Cg]) for o in range(D * R)])
    return dx, dw[:, :, None], dl.sum((0, 2))


class _EmuPlan:
    """_ConvPlan's fp32 branch on torch convs (left padding only, stride 1)."""

    def conv(self, x, w, b, dil=1, pad_l=0, res=None, want_f32=True, want_op=False):
        y = F.conv1d(F.pad(x, (pad_l, 0)), w, b, dilation=dil)
        return ((y + res if res is not None else y),) * 2

    def dgrad(self, dy, w, dil=1, pad_l=0, res=None, want_f32=True, want_op=False):
        K = w.shape[-1]
        pr = (K - 1) * dil - pad_l
        dx = F.conv1d(F.pad(dy, (pr, pad_l)), w.flip(-1).transpose(0, 1), dilation=dil)
        return ((dx + res if res is not None else dx),) * 2

    def wgrad(self, dy, x, w, dil=1, pad_l=0):
        K = w.shape[-1]
        xp = F.pad(x, (pad_l, 0))
        T = dy.shape[-1]
        dw = torch.stack([torch.einsum("bot,bit->oi", dy, xp[..., k * dil:k * dil + T]) for k in range(K)], -1)
        return dw, dy.sum((0, 2))


def test_step_plan_emulated_matches_golden(fx, monkeypatch):
    """rave_b200.prior.model's forward / backward plan with every library call replaced by the emulations above
    reproduces the reference's loss and gradients."""
    from rave_b200.prior import model as PM
    R, D = fx["prior_cfg"]["resolution"], fx["D"]
    cls = emu_latent_classes(fx["z"], fx["eps"], fx["latent_mean"], fx["latent_pca"], D, R)
    assert torch.equal(cls.permute(0, 2, 1), fx["classes"])
    emu = dict(
        prior_embed_fwd=lambda c, w, b, cl, slope: (emu_embed_fwd(c, w, b, slope), None),
        prior_embed_wgrad=lambda c, dout, x, shape, cl, slope: emu_embed_wgrad(c, dout, x, shape, slope),
        gate_fwd=lambda h, cl: emu_gate_fwd(h),
        gate_bwd=lambda dg, h, cl: emu_gate_bwd(dg, h),
        prior_head_ce_fwd=lambda p, w, b, c, cl, slope: emu_head_ce_fwd(p, w, b, c, slope),
        prior_head_ce_bwd=lambda p, w, b, c, g, cl, slope: emu_head_ce_bwd(p, w, b, c, g, slope),
    )
    for k, v in emu.items():
        monkeypatch.setattr(PM.ops, k, v)
    monkeypatch.setattr(PM, "_ConvPlan", lambda cl: _EmuPlan())
    sd = _prior_sd(fx)
    names = [k for k, _ in fx["prior_param_shapes"]]
    params = [sd[k] for k in names]
    dil = tuple(P.dilations(fx["prior_cfg"]))
    c = cls.int()
    loss, saved = PM._step_forward(c, params, dil, False)
    assert rel_l2(loss, fx["loss"]) < 1e-6
    grads = PM._step_backward(c, params, dil, False, saved, torch.ones(()))
    for k, g in zip(names, grads):
        if fx["grads"][k] is None:
            assert g is None, k
        else:
            assert rel_l2(g, fx["grads"][k]) < 1e-5, k

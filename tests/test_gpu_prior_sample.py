"""GPU: cached sampling from the latent prior (Prior.sample, csrc/prior_sample.cu) and the decode of its classes
(Prior.decode_classes) against the reference's generate fixture, the float64 restatement (tests/prior_sample_ref.py) and
the module's own ATen composition; its distribution, batch invariance, determinism, launch plan and argument checks."""
import os

import pytest
import torch

from oracle import prior_oracle as P
from tests import prior_sample_ref as S
from tests.conftest import GOLDEN, rel_l2
from tests.test_gpu_prior import _tiny_prior

pytestmark = pytest.mark.gpu

ODD = dict(resolution=16, res_size=96, skp_size=48, kernel_size=5, cycle_size=3, n_layers=5)
D128 = dict(P.PRIOR_V1, n_layers=2)


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(GOLDEN, "prior_tiny.pt"), weights_only=False)


def _prior(cfg, D, seed=0):
    from rave_b200.prior import VariationalPrior
    torch.manual_seed(seed)
    return VariationalPrior(latent_size=D, **cfg).cuda()


def _sd64(prior):
    return {k: v.detach().double() for k, v in prior.state_dict().items() if not k.startswith("synth.")}


def _classes(B, T, D, R, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, R, (B, T, D), generator=g, dtype=torch.int32).cuda()


def _uniform(B, T, D, seed):
    return torch.rand(B, T, D, generator=torch.Generator().manual_seed(seed)).cuda()


def test_argmax_sample_matches_reference_generate(fx):
    prior = _tiny_prior(fx)
    R, D = fx["prior_cfg"]["resolution"], fx["D"]
    B, _, T = fx["gen_in"].shape
    prefix = fx["gen_in"][:, :, :1].reshape(B, D, R, 1).argmax(2).permute(0, 2, 1).to(torch.int32).cuda()
    cls = prior.sample(prefix, T, argmax=True)
    assert cls.shape == (B, T, D) and cls.dtype == torch.int32
    assert torch.equal(P.stack_one_hot(cls.permute(0, 2, 1).long().cpu(), R), fx["gen_out"])


@pytest.mark.parametrize("name", ["tiny", "prior_v1", "d128", "odd"])
def test_teacher_forced_logits_match_dense_forward(fx, name):
    """P = T: every step is teacher-forced, so the cached logits of step i are the dense forward's at frame i.  At
    prior_v1, T = 256 is more than 3x the 67-frame receptive field: every ring wraps."""
    if name == "tiny":
        prior, cfg, D, B, T = _tiny_prior(fx), fx["prior_cfg"], fx["D"], 2, 40
    else:
        cfg, D, B, T = {"prior_v1": (P.PRIOR_V1, 16, 2, 256), "d128": (D128, 128, 2, 40),
                        "odd": (ODD, 8, 3, 60)}[name]
        prior = _prior(cfg, D)
    R = cfg["resolution"]
    cls = _classes(B, T, D, R, 1)
    got_cls, lg = prior.sample(cls, T, argmax=True, return_logits=True)
    assert torch.equal(got_cls, cls)
    want = S.teacher_logits(cls, _sd64(prior), cfg, D)
    r = rel_l2(lg, want)
    print(f"{name}: logits rel-L2 {r:.2e}")
    assert lg.shape == (B, T - 1, D, R) and r < 1e-5


def test_sampler_matches_float64_inverse_cdf():
    """Each step's class is the float64 inverse-CDF class of the float64 logits on the same history, except where u lies
    within 1e-5 of a CDF edge; with no such case the whole trajectory equals the float64 sampler's."""
    cfg, D, B, T = P.PRIOR_V1, 16, 4, 48
    prior = _prior(cfg, D, seed=1)
    sd = _sd64(prior)
    u = _uniform(B, T, D, 2)
    prefix = _classes(B, 1, D, cfg["resolution"], 3)
    cls = prior.sample(prefix, T, uniform=u)
    lg = S.teacher_logits(cls, sd, cfg, D)
    uu = u[:, 1:].double()
    want = S.inverse_cdf(lg, uu)
    near = S.cdf_edge_distance(lg, uu) < 1e-5
    diff = cls[:, 1:].long() != want
    print(f"sampler: {int(diff.sum())} of {diff.numel()} classes differ, {int(near.sum())} draws within 1e-5 of an edge")
    assert not (diff & ~near).any()
    if not near.any():
        ref, _ = S.sample(prefix, u.double(), sd, cfg, D, T)
        assert torch.equal(cls.long(), ref)


def test_class_distribution_matches_softmax():
    """With every weight zero the logits of group d are post_net.2.bias[d R : (d + 1) R] at every step."""
    from scipy.stats import chisquare
    cfg, D, B, T = P.PRIOR_V1, 16, 64, 512
    R = cfg["resolution"]
    prior = _prior(cfg, D)
    g = torch.Generator().manual_seed(7)
    bias = 1.5 * torch.randn(D, R, generator=g)
    with torch.no_grad():
        for p in prior._trained_parameters():
            p.zero_()
        prior.post_net[2].bias.copy_(bias.reshape(-1))
    torch.manual_seed(8)
    cls = prior.sample(torch.zeros(B, 1, D, dtype=torch.int32, device="cuda"), T)[:, 1:].cpu().long()
    prob = torch.softmax(bias.double(), -1)
    for d in range(D):
        counts = torch.bincount(cls[:, :, d].reshape(-1), minlength=R).double()
        pv = chisquare(counts.numpy(), (prob[d] * counts.sum()).numpy()).pvalue
        print(f"group {d}: chi-square p = {pv:.3g}")
        assert pv > 1e-3, (d, pv)


def test_prefix_state_equals_generated_state():
    cfg, D, B, T, Pn = P.PRIOR_V1, 16, 3, 100, 37
    prior = _prior(cfg, D, seed=2)
    u = _uniform(B, T, D, 4)
    first = prior.sample(_classes(B, 1, D, cfg["resolution"], 5), T, uniform=u)
    again = prior.sample(first[:, :Pn].contiguous(), T, uniform=u)
    assert torch.equal(first, again)


def test_batch_invariance_determinism_and_precision_modes():
    import rave_b200
    cfg, D, T = ODD, 8, 70
    prior = _prior(cfg, D, seed=3)
    prefix = _classes(5, 2, D, cfg["resolution"], 6)
    u = _uniform(5, T, D, 7)
    c5, l5 = prior.sample(prefix, T, uniform=u, return_logits=True)
    c1, l1 = prior.sample(prefix[:1].contiguous(), T, uniform=u[:1].contiguous(), return_logits=True)
    assert torch.equal(c5[:1], c1) and torch.equal(l5[:1], l1)
    torch.manual_seed(9)
    a = prior.sample(prefix, T)
    torch.manual_seed(9)
    b = prior.sample(prefix, T)
    assert torch.equal(a, b)
    rave_b200.set_precision("bf16")
    try:
        torch.manual_seed(9)
        c = prior.sample(prefix, T)
    finally:
        rave_b200.set_precision("fp32")
    assert torch.equal(a, c)


def test_sample_launch_plan(fx, monkeypatch):
    """One library call whatever the number of frames; the one-hot and torch.multinomial are never used."""
    from rave_b200 import _lib
    prior = _tiny_prior(fx)
    D = fx["D"]

    def forbidden(*a, **k):
        raise AssertionError("called on the sampling path")
    monkeypatch.setattr(torch.nn.functional, "one_hot", forbidden)
    monkeypatch.setattr(torch, "multinomial", forbidden)
    calls = {}
    for n in (8, 64):
        _lib.PROFILE = []
        try:
            prior.sample(torch.zeros(2, 1, D, dtype=torch.int32, device="cuda"), n)
            torch.cuda.synchronize()
            calls[n] = [e[0] for e in _lib.PROFILE]
        finally:
            _lib.PROFILE = None
    assert calls[8] == calls[64] == ["rave_prior_sample"], calls


def test_classes_to_latent_matches_float64(fx):
    from rave_b200 import ops
    prior = _tiny_prior(fx)
    R, D = fx["prior_cfg"]["resolution"], fx["D"]
    L = prior.synth.latent_pca.shape[0]
    B, T = 3, 20
    cls = _classes(B, T, D, R, 10)
    g = torch.Generator().manual_seed(11)
    dither = torch.rand(B, T, D, generator=g)
    cls[0, :, :] = 0
    dither[0] = 0.0                                       # erfinv(-1) = -inf before the clamp
    cls[1, :, :] = R - 1
    dither[1] = 1.0 - 2.0 ** -24                          # the largest float below 1
    cls[2, ::2, ::2] = 0
    dither[2, 1::2] = 2.0 ** -24
    noise = torch.randn(B, L - D, T - D + 1, generator=g)
    z = ops.prior_classes_to_latent(cls, dither.cuda(), noise.cuda(), prior.synth.latent_pca,
                                    prior.synth.latent_mean, R)
    want = S.classes_to_latent(cls.cpu(), dither.double(), noise.double(), prior.synth.latent_pca.double().cpu(),
                               prior.synth.latent_mean.double().cpu(), R)
    assert z.shape == (B, L, T - D + 1)
    assert rel_l2(z, want) < 1e-6
    # identity PCA, zero mean: the first D channels are the clamped normals themselves
    y = ops.prior_classes_to_latent(cls, dither.cuda(), noise.cuda(), torch.eye(L, device="cuda"),
                                    torch.zeros(L, device="cuda"), R)[:, :D].cpu()
    assert torch.equal(y[0], torch.full_like(y[0], -4.0)) and torch.equal(y[1], torch.full_like(y[1], 4.0))


def test_decode_classes_default_draws_match_module_composition(fx, monkeypatch):
    """Under one seed the default draws (dither, then noise) are the ones the module's own ATen path makes:
    QuantizedNormal.decode's rand_like, then pre_process_latent's randn."""
    prior = _tiny_prior(fx)
    R, D = fx["prior_cfg"]["resolution"], fx["D"]
    cls = _classes(2, 24, D, R, 12)
    monkeypatch.setattr(prior.synth, "decode", lambda z: z)
    torch.manual_seed(13)
    got = prior.decode_classes(cls)
    torch.manual_seed(13)
    one_hot = P.stack_one_hot(cls.permute(0, 2, 1).long(), R).cuda()
    want = prior.pre_process_latent(prior.diagonal_shift.inverse(prior.quantized_normal.decode(one_hot)))
    assert got.shape == want.shape
    assert rel_l2(got, want) < 1e-6


def test_validation_epoch_end_tiny(fx):
    prior = _tiny_prior(fx)
    D = fx["D"]
    T_lat = fx["z"].shape[-1]
    prior.validation_epoch_end([fx["x"].cuda()])
    y = prior.logged["generation"]
    assert y.shape == (fx["x"].shape[0], 1, (T_lat - 2 * D + 2) * fx["model_ratio"])
    assert torch.isfinite(y).all() and prior.val_idx == 1


def test_validation_epoch_end_full_size():
    """prior_v1 on a full-size v2 RAVE, D = 16, B = 8 x 256 latent frames, bf16 decode."""
    import rave_b200
    from rave_b200 import configs
    torch.manual_seed(0)
    prior = configs.build_prior(configs.build_rave("v2"), latent_size=16).cuda()
    ratio = prior.get_model_ratio()
    x = (0.3 * torch.randn(8, 1, 256 * ratio, device="cuda")).clamp(-1, 1)
    rave_b200.set_precision("bf16")
    try:
        prior.validation_epoch_end([x])
        torch.cuda.synchronize()
    finally:
        rave_b200.set_precision("fp32")
    y = prior.logged["generation"]
    assert y.shape == (8, 1, (256 - 2 * 16 + 2) * ratio)
    assert torch.isfinite(y).all()


def test_sample_argument_errors(fx):
    from rave_b200._lib import RaveB200Error
    prior = _tiny_prior(fx)
    D = fx["D"]
    prefix = torch.zeros(1, 1, D, dtype=torch.int32, device="cuda")
    with pytest.raises(RaveB200Error):
        prior.sample(prefix.cpu(), 8)
    with pytest.raises(RaveB200Error, match="B = 65"):
        prior.sample(torch.zeros(65, 1, D, dtype=torch.int32, device="cuda"), 8)
    with pytest.raises(RaveB200Error, match="P <= T"):
        prior.sample(torch.zeros(1, 10, D, dtype=torch.int32, device="cuda"), 5)
    u = torch.rand(1, 8, D, device="cuda")
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RaveB200Error, match="capture"):
        with torch.cuda.graph(g):
            prior.sample(prefix, 8, uniform=u)
    # the library still works after the refused call
    assert prior.sample(prefix, 8, uniform=u).shape == (1, 8, D)

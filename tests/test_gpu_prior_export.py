"""GPU: the exported model's `prior(temp)` (ExportedRAVE.prior, csrc/prior_sample.cu prior_stream) against the
reference's fixture (tests/golden/prior_export.pt) and the float64 restatement (tests/prior_export_ref.py); call
splitting, row independence, reset, the argmax limit of a low temperature, the kept frame graph and its re-capture, the
refusal inside a stream capture, and decode(prior(temp)) end to end."""
import os

import pytest
import torch

from oracle import prior_oracle as P
from tests import prior_export_ref as E
from tests.conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu

TINY_VAE = dict(capacity=4, latent_size=8)


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(GOLDEN, "prior_export.pt"), weights_only=False)


def _model():
    from rave_b200 import configs
    torch.manual_seed(0)
    return configs.build_rave("v2", disc_capacity=4, **TINY_VAE).cuda()


def _exported(cfg, D, param_seed, model=None):
    """ExportedRAVE of a tiny v2 with a prior of `cfg` at D, the prior's parameters from seeded_params."""
    from rave_b200 import configs
    from rave_b200.export import ExportedRAVE
    model = model or _model()
    prior = configs.build_prior(model, latent_size=D, **cfg)
    shapes = [(k, tuple(v.shape)) for k, v in prior.named_parameters() if not k.startswith("synth.")]
    prior.load_state_dict(dict(prior.state_dict(), **P.seeded_params(shapes, param_seed)), strict=True)
    prior.cuda()
    sd = {k: v.detach().double().cpu() for k, v in prior.state_dict().items() if not k.startswith("synth.")}
    return ExportedRAVE(model, prior=prior), sd


def _draws(B, T, D, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, T, D, generator=g).cuda(), torch.rand(B, T, D, generator=g).cuda()


def test_calls_match_reference_fixture(fx):
    """Output latents against the fixture and the float64 restatement.  Every class of the fixture is at least 1e-3 from
    a CDF edge, and a different class would move its decoded value by far more than 1e-3, so the element-wise bound
    checks every class.  The reference decodes in float32 with the kernel's operations; against float64, erfinv near
    +-1 magnifies the float32 rounding of 2 x - 1."""
    cfg = fx["prior_cfg"]
    for case in fx["cases"]:
        ex, sd = _exported(cfg, case["D"], case["param_seed"])
        ref = E.StreamRef(sd, cfg, case["D"], case["B"])
        for c in case["calls"]:
            got = ex.prior(c["temp_in"].cuda(), uniform=c["uniform"].cuda(), dither=c["dither"].cuda())
            want, cls = ref(c["temp_in"], c["uniform"], c["dither"])
            assert torch.equal(cls, c["classes"])
            assert got.shape == c["out"].shape and got.dtype == torch.float32
            assert (got.cpu().double() - c["out"].double()).abs().max() < 1e-3
            assert rel_l2(got, c["out"]) < 1e-6 and rel_l2(got, want) < 1e-4


def test_call_split_is_bit_identical():
    cfg, D, B, T = dict(P.PRIOR_V1, n_layers=4), 8, 2, 12
    ex, _ = _exported(cfg, D, 7)
    u, d = _draws(B, T, D, 1)
    temp = torch.full((B, 1, T), 0.5, device="cuda")          # the same temperature for every split
    whole = ex.prior(temp, u, d)
    ex.reset_prior()
    parts, t0 = [], 0
    for n in (3, 5, 4):
        parts.append(ex.prior(temp[..., t0:t0 + n], u[:, t0:t0 + n].contiguous(), d[:, t0:t0 + n].contiguous()))
        t0 += n
    assert torch.equal(torch.cat(parts, -1), whole)


def test_rows_are_independent_and_reset_restarts():
    from rave_b200.export import ExportedRAVE
    cfg, D, B, T = dict(P.PRIOR_V1, n_layers=4), 8, 5, 9
    ex, _ = _exported(cfg, D, 8)
    u, d = _draws(B, T, D, 2)
    temp = torch.linspace(-2, 3, B, device="cuda")[:, None, None] + torch.randn(B, 1, T, device="cuda")
    first = ex.prior(temp, u, d)
    second = ex.prior(temp, u, d)
    for b in range(B):
        ex.reset_prior()
        one = ex.prior(temp[b:b + 1], u[b:b + 1], d[b:b + 1])
        assert torch.equal(one, first[b:b + 1]), b
        assert torch.equal(ex.prior(temp[b:b + 1], u[b:b + 1], d[b:b + 1]), second[b:b + 1]), b
    fresh = ExportedRAVE(ex.model, prior=ex.prior_module)
    assert torch.equal(fresh.prior(temp, u, d), first)
    with pytest.raises(ValueError, match="reset_prior"):
        fresh.prior(temp[:2], u[:2], d[:2])


def test_low_temperature_is_argmax():
    """An input of -30 gives softplus(-30) / ln 2 ~ 1.4e-13: the logits are scaled by ~7e12 and the softmax is one-hot."""
    cfg, D, B = dict(P.PRIOR_V1, n_layers=3), 8, 2
    ex, sd = _exported(cfg, D, 9)
    ref = E.StreamRef(sd, cfg, D, B, argmax=True)
    for T, seed in ((4, 3), (7, 4)):
        u, d = _draws(B, T, D, seed)
        temp = torch.full((B, 1, T), -30.0)
        got = ex.prior(temp.cuda(), u, d)
        want, _ = ref(temp, u.cpu(), d.cpu())
        assert (got.cpu().double() - want).abs().max() < 1e-3 and rel_l2(got, want) < 1e-4


def test_frame_graph_is_captured_once_and_recaptured_when_parameters_move():
    from rave_b200 import _lib
    cfg, D, B = dict(P.PRIOR_V1, n_layers=3), 8, 2
    ex, _ = _exported(cfg, D, 10)
    draws = [_draws(B, T, D, 10 + T) for T in (3, 6, 2)]
    temps = [torch.zeros(B, 1, T, device="cuda") for T in (3, 6, 2)]
    want = [ex.prior(t, u, d) for t, (u, d) in zip(temps[:2], draws[:2])]
    state = ex._prior_state
    n0 = _lib.launch_count()
    want.append(ex.prior(temps[2], *draws[2]))
    assert _lib.launch_count() - n0 == 1 + 2                   # the prologue and two replays
    assert state.captures == 1 and ex._prior_state is state
    ex.reset_prior()
    got = [ex.prior(temps[0], *draws[0])]
    w = ex.prior_module.post_net[2].weight
    w.data = w.data.clone()                                     # the same values in new storage
    got += [ex.prior(t, u, d) for t, (u, d) in zip(temps[1:], draws[1:])]
    assert ex._prior_state.captures == 2
    for a, b in zip(got, want):
        assert torch.equal(a, b)


def test_refuses_inside_a_stream_capture():
    from rave_b200._lib import RaveB200Error
    cfg, D = dict(P.PRIOR_V1, n_layers=2), 8
    ex, _ = _exported(cfg, D, 11)
    temp = torch.zeros(1, 1, 3, device="cuda")
    u, d = _draws(1, 3, D, 5)
    ex.prior(temp, u, d)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RaveB200Error, match="capture"):
        with torch.cuda.graph(g):
            ex.prior(temp, u, d)
    ex.reset_prior()
    g2 = torch.cuda.CUDAGraph()
    with pytest.raises(RaveB200Error, match="capture"):
        with torch.cuda.graph(g2):
            ex.prior(temp, u, d)
    assert ex.prior(temp, u, d).shape == (1, D, 3)


def test_decode_of_prior_end_to_end():
    cfg, D, B, T = dict(P.PRIOR_V1, n_layers=3), 4, 2, 6
    ex, _ = _exported(cfg, D, 12)
    torch.manual_seed(1)
    z = ex.prior(torch.zeros(B, 1, T, device="cuda"))
    y = ex.decode(z)
    assert z.shape == (B, D, T) and y.shape == (B, 1, T * ex.encode_ratio)
    assert torch.isfinite(z).all() and torch.isfinite(y).all()

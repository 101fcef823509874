"""CPU: the float64 restatement of the exported model's `prior(temp)` (tests/prior_export_ref.py) against the fixture the
unmodified reference's prior modules produced (tests/golden/prior_export.pt, oracle/make_golden_prior_export.py), and
the host logic of ExportedRAVE's prior: constructor validation, the call without a prior and the row-count check, with
the library's stream state replaced by a fake (the product has no CPU path).  The GPU twin is
tests/test_gpu_prior_export.py."""
import os

import pytest
import torch

from oracle import prior_oracle as P
from rave_b200 import blocks, ops
from rave_b200.export import ExportedRAVE
from rave_b200.prior import VariationalPrior
from tests import prior_export_ref as E
from tests.conftest import GOLDEN, rel_l2
from tests.test_export_cpu import FakeRAVE, _identity, oracle_ops  # noqa: F401  (fixture)


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(GOLDEN, "prior_export.pt"), weights_only=False)


def test_restatement_reproduces_reference_fixture(fx):
    cfg = fx["prior_cfg"]
    for case in fx["cases"]:
        sd = {k: v.double() for k, v in P.seeded_params(case["param_shapes"], case["param_seed"]).items()}
        ref = E.StreamRef(sd, cfg, case["D"], case["B"])
        for c in case["calls"]:
            assert torch.allclose(E.temperature(c["temp_in"]), c["temperature"].double()[:, 0, 0], rtol=1e-6)
            out, cls = ref(c["temp_in"], c["uniform"], c["dither"])
            assert torch.equal(cls, c["classes"]), (case["D"], case["B"])
            # the reference decodes in float32, where erfinv near +-1 magnifies the rounding of 2 x - 1
            assert out.shape == c["out"].shape and rel_l2(out, c["out"]) < 1e-4


def test_zero_input_is_temperature_one():
    assert E.temperature(torch.zeros(2, 1, 5)).tolist() == [1.0, 1.0]


def _prior(model, D=4):
    p = VariationalPrior(latent_size=D, resolution=8, res_size=32, skp_size=16, kernel_size=3, cycle_size=2,
                         n_layers=3)
    p.synth = model
    return p


def test_constructor_validation(oracle_ops):  # noqa: F811
    m = FakeRAVE(blocks.VariationalEncoder(_identity), 8, enc_out=16)
    plain = ExportedRAVE(m)
    assert plain.prior_module is None and not any(k.startswith("prior_module") for k in plain.state_dict())
    with pytest.raises(RuntimeError, match="without a prior"):
        plain.prior(torch.zeros(1, 1, 2))
    ex = ExportedRAVE(m, prior=_prior(m))
    assert ex.prior_module is not None and "prior_module.pre_net.0.weight" in ex.state_dict()
    assert set(plain.state_dict()) <= set(ex.state_dict())
    with pytest.raises(ValueError, match="VariationalPrior"):
        ExportedRAVE(m, prior=torch.nn.Linear(2, 2))
    other = FakeRAVE(blocks.VariationalEncoder(_identity), 8, enc_out=16)
    with pytest.raises(ValueError, match="synth"):
        ExportedRAVE(m, prior=_prior(other))
    m4 = FakeRAVE(blocks.VariationalEncoder(_identity), 4, enc_out=8)
    with pytest.raises(ValueError, match="latent_size"):
        ExportedRAVE(m4, prior=_prior(m4, D=8))


class _FakeStream:
    def __init__(self, params, cycle, B, R, D):
        self.B, self.D, self.device = B, D, params[0].device
        self.calls = []

    def __call__(self, params, temp, uniform, dither):
        self.calls.append((temp, uniform, dither))
        return torch.zeros(self.B, self.D, temp.shape[-1])


def test_row_count_is_kept_until_reset(oracle_ops, monkeypatch):  # noqa: F811
    monkeypatch.setattr(ops, "PriorStream", _FakeStream)
    m = FakeRAVE(blocks.VariationalEncoder(_identity), 8, enc_out=16)
    ex = ExportedRAVE(m, prior=_prior(m))
    assert ex.prior(torch.zeros(2, 1, 3)).shape == (2, 4, 3)
    assert ex.prior(torch.zeros(2, 1, 1), uniform=torch.rand(2, 1, 4), dither=torch.rand(2, 1, 4)).shape == (2, 4, 1)
    with pytest.raises(ValueError, match="reset_prior"):
        ex.prior(torch.zeros(3, 1, 2))
    with pytest.raises(ValueError, match="uniform"):
        ex.prior(torch.zeros(2, 1, 2), uniform=torch.rand(2, 4, 2))
    with pytest.raises(ValueError, match=r"\[B, 1, T\]"):
        ex.prior(torch.zeros(2, 2, 2))
    ex.reset_prior()
    assert ex.prior(torch.zeros(3, 1, 2)).shape == (3, 4, 2)

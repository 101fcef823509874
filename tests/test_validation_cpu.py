"""CPU: the validation pass's host logic -- the float64 PCA restatement against the reference's own buffers, the
model's validation_epoch_end decisions, the receptive-field probe's save / restore, and GraphedTrainer's
receptive-field guard -- with the CUDA library ops replaced by torch stand-ins (test infrastructure; the product has no
CPU path).  The GPU twin is tests/test_gpu_validation.py."""
import os

import numpy as np
import pytest
import torch
import torch.nn as nn

from oracle import validation_oracle as V
from tests.conftest import GOLDEN


def _fixture():
    return torch.load(os.path.join(GOLDEN, "validation_v2_tiny.pt"), weights_only=False)


def _moments_standin(z, D, state):
    """rave_latent_moments restated in torch float64: block moments of the rows z[b, :D, t], Chan-merged into state."""
    x = z[:, :D].double().permute(0, 2, 1).reshape(-1, D)
    nb, mb = x.shape[0], x.mean(0)
    c = x - mb
    Mb = c.T @ c
    n = float(state[0])
    nn_ = n + nb
    d = mb - state[1:1 + D]
    M2 = state[1 + D:].reshape(D, D)
    M2 += Mb + torch.outer(d, d) * (n * nb / nn_)
    state[1:1 + D] += d * (nb / nn_)
    state[0] = nn_
    return state


@pytest.fixture
def torch_moments(monkeypatch):
    from rave_b200 import ops
    monkeypatch.setattr(ops, "latent_moments", _moments_standin)


def test_oracle_reproduces_reference_pca():
    g = _fixture()
    means = [b["mean"] for b in g["batches"]]
    mean, comps, ev, fid = V.latent_analysis(means)
    assert np.abs(fid - g["fidelity"].double().numpy()).max() <= 1e-5
    assert np.abs(mean - g["latent_mean"].double().numpy()).max() <= 1e-5
    sep = V.separated(ev)
    assert len(sep) >= len(ev) // 2
    for i in sep:
        assert float(np.dot(comps[i], g["latent_pca"][i].double().numpy())) >= 0.9999, i
    assert V.fidelity_logs(fid) == {k: float(v) for k, v in g["fidelity_logs"].items()}
    # the Chan merge equals one pass over all rows
    rows = np.concatenate([V.rows(m) for m in means])
    n, m1, M2 = V.moments(means)
    assert n == rows.shape[0]
    assert np.allclose(m1, rows.mean(0), rtol=0, atol=1e-12)
    c = rows - rows.mean(0)
    assert np.allclose(M2, c.T @ c, rtol=1e-12, atol=1e-12)


def test_latent_analysis_matches_oracle(torch_moments):
    from rave_b200 import core
    g = _fixture()
    means = [b["mean"] for b in g["batches"]]
    mean, comps, fid = core.latent_analysis(means, 16)
    m_o, c_o, ev_o, f_o = V.latent_analysis(means)
    assert mean.dtype == comps.dtype == fid.dtype == torch.float32
    assert np.abs(fid.double().numpy() - f_o).max() <= 1e-6
    for i in V.separated(ev_o):
        assert float(np.dot(comps[i].double().numpy(), c_o[i])) >= 0.99999, i
    # sklearn's sign rule: the largest-|.| entry of each component is positive
    piv = comps.gather(1, comps.abs().argmax(1, keepdim=True))
    assert bool((piv > 0).all())


def test_latent_analysis_refuses_too_few_rows(torch_moments):
    from rave_b200 import core
    with pytest.raises(ValueError):
        core.latent_analysis([torch.randn(1, 16, 15)], 16)
    core.latent_analysis([torch.randn(1, 16, 8), torch.randn(1, 16, 8)], 16)


def _model(name="v2"):
    from rave_b200 import configs
    torch.manual_seed(0)
    return configs.build_rave(name, capacity=8, latent_size=16, disc_capacity=4)


def _probe_counter(monkeypatch, rf=(1000, 500)):
    from rave_b200 import core
    calls = []
    monkeypatch.setattr(core, "get_rave_receptive_field", lambda model, n_channels=1: calls.append(1) or rf)
    return calls


def test_epoch_end_fits_pca_in_phase_1_of_a_variational_model(monkeypatch, torch_moments):
    g = _fixture()
    m = _model()
    calls = _probe_counter(monkeypatch)
    out = [(None, b["mean"]) for b in g["batches"]]
    m.validation_epoch_end(out)
    assert len(calls) == 1 and m.receptive_field.tolist() == [1000, 500]
    assert torch.allclose(m.fidelity, g["fidelity"], atol=1e-5)
    assert torch.allclose(m.latent_mean, g["latent_mean"], atol=1e-5)
    assert set(k for k in m.logged if k.startswith("fidelity_")) == {f"fidelity_{p}" for p in (.8, .9, .95, .99)}
    for k, v in g["fidelity_logs"].items():
        assert float(m.logged[k]) == float(v), k
    assert m.eval_number == 1
    # the receptive field is probed once; phase 2 leaves the PCA alone
    m.warmed_up = True
    before = [t.clone() for t in (m.latent_mean, m.latent_pca, m.fidelity)]
    m.validation_epoch_end([(None, 3 * b["mean"]) for b in g["batches"]])
    assert len(calls) == 1 and m.eval_number == 2
    assert all(torch.equal(a, b) for a, b in zip(before, (m.latent_mean, m.latent_pca, m.fidelity)))


def test_epoch_end_with_empty_out_only_probes(monkeypatch):
    m = _model()
    calls = _probe_counter(monkeypatch)
    m.validation_epoch_end([])
    assert len(calls) == 1 and m.receptive_field.tolist() == [1000, 500]
    assert m.eval_number == 0 and torch.equal(m.latent_pca, torch.eye(16)) and not m.fidelity.any()


def test_epoch_end_non_variational_gets_receptive_field_only(monkeypatch):
    m = _model("v2_wasserstein")
    calls = _probe_counter(monkeypatch)
    m.validation_epoch_end([(None, None), (None, None)])
    assert len(calls) == 1 and m.receptive_field.tolist() == [1000, 500] and m.eval_number == 1
    assert torch.equal(m.latent_pca, torch.eye(m.latent_size)) and not m.fidelity.any()


class _Recurrent(nn.Module):
    """A module the probe must switch off: an unbounded causal recurrence (running sum) when enabled."""

    def __init__(self):
        super().__init__()
        self.register_buffer("gru_state", torch.tensor(0))
        self.enabled = True
        self.seen = []

    def forward(self, x):
        self.seen.append(self.enabled)
        return torch.cumsum(x, -1) if self.enabled else x

    def disable(self):
        self.enabled = False

    def enable(self):
        self.enabled = True


class _Reparam(nn.Module):
    def reparametrize(self, z):
        return z, None


class _ToyRave(nn.Module):
    """encode = conv k=5 (pad 2, 2), decode = recurrence + conv k=3 dilation 2 (pad 2, 2): input support of an output sample: 4 samples each side."""

    def __init__(self):
        super().__init__()
        self.n_channels = 1
        self.enc = nn.Conv1d(1, 2, 5, padding=2)
        self.encoder = _Reparam()
        self.rec = _Recurrent()
        self.dec = nn.Conv1d(2, 1, 3, padding=2, dilation=2)

    def encode(self, x):
        return self.enc(x)

    def decode(self, z):
        return self.dec(self.rec(z))


def test_probe_restores_state_and_leaves_no_parameter_grad():
    import rave_b200
    from rave_b200 import core, engine
    m = _ToyRave().train()
    rave_b200.set_precision("bf16")
    try:
        assert core.get_rave_receptive_field(m) == (4, 5)     # the right half holds the centre sample
        assert engine.precision() == "bf16"
    finally:
        rave_b200.set_precision("fp32")
    assert m.training and m.rec.enabled and m.rec.seen and not any(m.rec.seen)
    assert all(p.grad is None for p in m.parameters())
    m.eval()
    core.get_rave_receptive_field(m)
    assert not m.training


def test_graphed_trainer_refuses_a_changed_receptive_field():
    from rave_b200.graphs import GraphedTrainer
    m = _model()
    gt = GraphedTrainer.__new__(GraphedTrainer)          # the guard runs before anything touches the device
    gt.model, gt.phase2 = m, False
    gt._weights_at_capture = dict(m.weights)
    gt._receptive_field_at_capture = m._receptive_field_host()
    m.set_receptive_field(27117, 26428)
    with pytest.raises(RuntimeError, match="receptive_field changed"):
        gt.step(torch.zeros(1, 1, 8), 0)

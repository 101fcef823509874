"""The EMA callback without a GPU: the float32 restatement (oracle/ema_oracle.py) against the reference's own EMA class
(tests/golden/ema.pt), and the host logic of rave_b200/ema.py -- keys, first-call clone, swap, load_state_dict,
the empty-state message, a replaced parameter -- with the two kernel launches replaced by torch stand-ins (test
infrastructure; the product has no CPU path).  The GPU twin is tests/test_gpu_ema.py."""
import os

import pytest
import torch
import torch.nn as nn

from oracle import ema_oracle as E
from rave_b200 import configs
from rave_b200.ema import EMA

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _fixture():
    return torch.load(os.path.join(GOLDEN, "ema.pt"), weights_only=False)


@pytest.fixture
def torch_ema(monkeypatch):
    """EMA's two launches as torch ops on the tensors the table describes."""

    def update(self):
        f, g = self.factor, 1 - self.factor
        with torch.no_grad():
            for i, (p, e) in enumerate(zip(self._params, self._views.values())):
                e.copy_(e * f + p * g if int(self._state[i]) else p)
            self._state[:-1] = 1

    def swap(self):
        with torch.no_grad():
            for p, e in zip(self._params, self._views.values()):
                t = p.clone()
                p.copy_(e)
                e.copy_(t)

    monkeypatch.setattr(EMA, "_launch_update", update)
    monkeypatch.setattr(EMA, "_launch_swap", swap)


class _Holder(nn.Module):
    def __init__(self, shapes):
        super().__init__()
        self.ps = nn.ParameterList([nn.Parameter(torch.zeros(s)) for s in shapes])

    def set(self, values):
        with torch.no_grad():
            for p, v in zip(self.ps, values):
                p.copy_(v)


def test_restatement_matches_reference_fixture_exactly():
    fx = _fixture()
    names = [n for n, _ in fx["names_shapes"]]
    snaps = E.snapshots([s for _, s in fx["names_shapes"]], fx["n_calls"], fx["seed"])
    assert set(fx["cases"]) == set(E.FACTORS)
    for factor, case in fx["cases"].items():
        w = {}
        for k, snap in enumerate(snaps):
            E.update(w, list(zip(names, snap)), factor)
            assert E.digest(w[n] for n in names) == case["digests"][k], (factor, k)
        if factor == .999:
            for n in names:
                assert torch.equal(w[n], fx["last_999"][n]), n
        params = [nn.Parameter(t.clone()) for t in snaps[-1]]
        E.swap(w, list(zip(names, params)))
        assert (E.digest(params), E.digest(w[n] for n in names)) == case["swapped"]
        E.swap(w, list(zip(names, params)))
        assert (E.digest(params), E.digest(w[n] for n in names)) == case["swapped_back"]
    # the fixture separates two roundings from a fused multiply-add
    assert fx["cases"][.999]["fma_fraction"] > .05 and fx["cases"][.9]["fma_fraction"] > .05


def test_host_logic_matches_reference_fixture(torch_ema):
    fx = _fixture()
    names = [n for n, _ in fx["names_shapes"]]
    snaps = E.snapshots([s for _, s in fx["names_shapes"]], fx["n_calls"], fx["seed"])
    for factor, case in fx["cases"].items():
        m = _Holder([s for _, s in fx["names_shapes"]])
        ema = EMA(factor)
        for k, snap in enumerate(snaps):
            m.set(snap)
            ema.on_train_batch_end(None, m, None, None, k)
            assert E.digest(ema.state_dict().values()) == case["digests"][k]
        ema.swap_weights(m)
        assert (E.digest(m.parameters()), E.digest(ema.state_dict().values())) == case["swapped"]
        ema.swap_weights(m)
        assert (E.digest(m.parameters()), E.digest(ema.state_dict().values())) == case["swapped_back"]
    assert len(names) == len(m.ps)


@pytest.mark.parametrize("name", ["v2", "v3", "discrete"])
def test_keys_are_the_parameter_names(torch_ema, name):
    m = configs.build_rave(name, capacity=4, disc_capacity=2)
    ema = EMA()
    ema.on_train_batch_end(None, m, None, None, 0)
    sd = ema.state_dict()
    named = dict(m.named_parameters())
    assert list(sd) == list(named)
    for n, v in sd.items():
        assert v.shape == named[n].shape and v.dtype == torch.float32
        assert v.untyped_storage().data_ptr() == ema.flat.untyped_storage().data_ptr()       # a view of the buffer
        assert v.data_ptr() % 16 == 0
    # the reference's checkpoint keys: every average has a key of the same shape in the reference's state dict
    ref = torch.load(os.path.join(GOLDEN, "state_dict_keys.pt"), weights_only=False).get(f"rave_{name}")
    if ref is not None:
        full = configs.build_rave(name)
        for n, p in full.named_parameters():
            assert tuple(ref[n][0]) == tuple(p.shape), n
    # what export does with them
    twin = configs.build_rave(name, capacity=4, disc_capacity=2)
    twin.load_state_dict(sd, strict=False)
    for n, p in twin.named_parameters():
        assert torch.equal(p, named[n])


def test_first_call_clones_then_averages(torch_ema):
    m = _Holder([(3, 5), (7,)])
    m.set([torch.randn(3, 5), torch.randn(7)])
    ema = EMA(.9)
    assert ema.state_dict() == {}
    ema.on_train_batch_end(None, m, None, None, 0)
    for p, v in zip(m.parameters(), ema.state_dict().values()):
        assert torch.equal(p, v) and p.data_ptr() != v.data_ptr()
    before = [v.clone() for v in ema.state_dict().values()]
    m.set([torch.randn(3, 5), torch.randn(7)])
    ema.on_train_batch_end(None, m, None, None, 1)
    for p, b, v in zip(m.parameters(), before, ema.state_dict().values()):
        assert torch.equal(v, b * .9 + p.detach() * (1 - .9))


def test_swap_twice_is_the_identity(torch_ema):
    m = _Holder([(4, 4), (9,)])
    ema = EMA(.5)
    m.set([torch.randn(4, 4), torch.randn(9)])
    ema.on_train_batch_end(None, m, None, None, 0)
    m.set([torch.randn(4, 4), torch.randn(9)])
    ema.on_train_batch_end(None, m, None, None, 1)
    p0 = [p.detach().clone() for p in m.parameters()]
    e0 = [v.clone() for v in ema.state_dict().values()]
    ema.on_validation_epoch_start(None, m)
    assert all(torch.equal(p, e) for p, e in zip(m.parameters(), e0))
    assert all(torch.equal(v, p) for v, p in zip(ema.state_dict().values(), p0))
    ema.on_validation_epoch_end(None, m)
    assert all(torch.equal(p, q) for p, q in zip(m.parameters(), p0))
    assert all(torch.equal(v, e) for v, e in zip(ema.state_dict().values(), e0))


def test_load_state_dict_updates_in_place(torch_ema):
    m = _Holder([(2, 3), (5,)])
    m.set([torch.randn(2, 3), torch.randn(5)])
    ema = EMA(.9)
    ema.on_train_batch_end(None, m, None, None, 0)
    views = dict(ema.state_dict())
    keep = views["ps.1"].clone()
    new0 = torch.randn(2, 3)
    ema.load_state_dict({"ps.0": new0})
    sd = ema.state_dict()
    assert sd["ps.0"] is views["ps.0"] or sd["ps.0"].data_ptr() == views["ps.0"].data_ptr()
    assert torch.equal(sd["ps.0"], new0) and torch.equal(sd["ps.1"], keep)

    # resuming: a fresh EMA loaded from a checkpoint averages from its next step instead of cloning
    saved = {k: v.clone() for k, v in ema.state_dict().items()}
    fresh = EMA(.9)
    fresh.load_state_dict(saved)
    assert set(fresh.state_dict()) == set(saved)
    m.set([torch.randn(2, 3), torch.randn(5)])
    fresh.on_train_batch_end(None, m, None, None, 1)
    for (n, s), p in zip(saved.items(), m.parameters()):
        assert torch.equal(fresh.state_dict()[n], s * .9 + p.detach() * (1 - .9)), n

    # a partial load into a fresh EMA: the names it lacks are cloned at the next step, as the reference's dict does
    part = EMA(.9)
    part.load_state_dict({"ps.1": saved["ps.1"]})
    part.on_train_batch_end(None, m, None, None, 2)
    assert torch.equal(part.state_dict()["ps.0"], m.ps[0].detach())
    assert torch.equal(part.state_dict()["ps.1"], saved["ps.1"] * .9 + m.ps[1].detach() * (1 - .9))


def test_empty_state_validation_message(torch_ema, capsys):
    m = _Holder([(3,)])
    ema = EMA()
    ema.on_validation_epoch_start(None, m)
    ema.on_validation_epoch_end(None, m)
    assert capsys.readouterr().out == "no ema weights available\n" * 2
    ema.on_train_batch_end(None, m, None, None, 0)          # binding alone does not count: the first update does
    ema.on_validation_epoch_start(None, m)
    assert capsys.readouterr().out == ""


def test_replaced_parameter_raises(torch_ema):
    m = _Holder([(3,), (4,)])
    ema = EMA()
    ema.on_train_batch_end(None, m, None, None, 0)
    m.ps[1] = nn.Parameter(torch.zeros(4))
    with pytest.raises(RuntimeError, match="replaced"):
        ema.on_train_batch_end(None, m, None, None, 1)
    with pytest.raises(RuntimeError, match="replaced"):
        ema.swap_weights(m)
    with pytest.raises(RuntimeError, match="another module"):
        ema.on_train_batch_end(None, _Holder([(3,), (4,)]), None, None, 1)


def test_no_cpu_path():
    m = _Holder([(3,)])
    with pytest.raises(RuntimeError, match="no CPU path"):
        EMA().on_train_batch_end(None, m, None, None, 0)

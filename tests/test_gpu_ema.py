"""The EMA kernels on the GPU (csrc/ema.cu through rave_b200/ema.py): bit-identical to torch's own CUDA expression
`w * factor + p * (1 - factor)` over full-size v2 / v3 parameter sets, ragged sizes and misaligned parameters, and to
the reference's EMA class (tests/golden/ema.pt); swap / swap back; the engine's static prepared weights after a swap;
and the update captured in GraphedTrainer's graphs."""
import copy
import gc
import os

import pytest
import torch
import torch.nn as nn

import rave_b200
from oracle import ema_oracle as E
from rave_b200 import _lib, configs
from rave_b200.ema import EMA
from rave_b200.graphs import GraphedTrainer

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ema.pt")


@pytest.fixture(autouse=True)
def _release_device_memory():
    """Full-size models, averages and captured graphs (whose modules hold reference cycles) are freed when each test
    ends, not whenever the cycle collector next runs: later tests start from the device memory they would see without
    this file."""
    yield
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _check_against_torch(m, factors, steps=3, seed=0):
    """Perturb the parameters in place between updates; after each update the averages must equal torch's expression
    bit for bit.  Then swap twice."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    for factor in factors:
        ema = EMA(factor)
        ref = None
        for step in range(steps):
            with torch.no_grad():
                for p in m.parameters():
                    p.add_(torch.randn(p.shape, device="cuda", generator=g) * 1e-3)
            ema.on_train_batch_end(None, m, None, None, step)
            if ref is None:
                ref = {n: p.detach().clone() for n, p in m.named_parameters()}
            else:
                ref = {n: ref[n] * factor + p.detach() * (1 - factor) for n, p in m.named_parameters()}
            sd = ema.state_dict()
            for n in ref:
                assert torch.equal(sd[n], ref[n]), (factor, step, n)
        p0 = [p.detach().clone() for p in m.parameters()]
        ema.swap_weights(m)
        for (n, p) in m.named_parameters():
            assert torch.equal(p, ref[n]), n
        ema.swap_weights(m)
        assert all(torch.equal(p, q) for p, q in zip(m.parameters(), p0))
        assert all(torch.equal(ema.state_dict()[n], ref[n]) for n in ref)


@pytest.mark.parametrize("name", ["v2", "v3"])
def test_update_bit_identical_to_torch_full_size(name):
    torch.manual_seed(0)
    m = configs.build_rave(name).cuda()
    _check_against_torch(m, (.999, .9), steps=3)


def test_ragged_and_misaligned_parameters():
    """Sizes around the vector width and the chunk size, parameters at every 4-byte offset of a shared storage (only
    the scalar path can serve those), and an empty one."""
    sizes = [1, 2, 3, 4, 5, 7, 4095, 4096, 4097, 8191, 16385, 100003]
    base = torch.randn(sum(sizes) * 4 + 64, device="cuda")
    m = nn.Module()
    off = 0
    for i, n in enumerate(sizes):
        for shift in range(4):
            start = off + shift
            m.register_parameter(f"p{i}_{shift}", nn.Parameter(base[start:start + n]))
            off = start + n
        off += (-off) % 4
    m.register_parameter("empty", nn.Parameter(torch.zeros(0, device="cuda")))
    assert {p.data_ptr() % 16 for p in m.parameters() if p.numel()} == {0, 4, 8, 12}
    _check_against_torch(m, (.999, .9, .75), steps=3, seed=1)


def test_matches_reference_fixture():
    fx = torch.load(GOLDEN, weights_only=False)
    names = [n for n, _ in fx["names_shapes"]]
    snaps = E.snapshots([s for _, s in fx["names_shapes"]], fx["n_calls"], fx["seed"])
    for factor, case in fx["cases"].items():
        m = nn.Module()
        m.ps = nn.ParameterList([nn.Parameter(t.clone()) for t in snaps[0]]).cuda()
        ema = EMA(factor)
        for k, snap in enumerate(snaps):
            with torch.no_grad():
                for p, v in zip(m.ps, snap):
                    p.copy_(v)
            ema.on_train_batch_end(None, m, None, None, k)
            assert E.digest(ema.state_dict().values()) == case["digests"][k], (factor, k)
        if factor == .999:
            for v, n in zip(ema.state_dict().values(), names):
                assert torch.equal(v.cpu(), fx["last_999"][n]), n
        ema.swap_weights(m)
        assert (E.digest(m.parameters()), E.digest(ema.state_dict().values())) == case["swapped"]
        ema.swap_weights(m)
        assert (E.digest(m.parameters()), E.digest(ema.state_dict().values())) == case["swapped_back"]


# ------------------------------------------------------------------------------------ GraphedTrainer, bf16
def _model(seed):
    torch.manual_seed(seed)
    m = configs.build_rave("v2", capacity=16, latent_size=16, disc_capacity=16).cuda().train()
    m.warmed_up = True           # phase 2: a G-step and a D-step graph, static discriminator and encoder prep
    return m


@pytest.fixture(scope="module")
def bf16():
    rave_b200.set_precision("bf16")
    yield
    rave_b200.set_precision("fp32")


def _snapshot(m):
    return [p.detach().clone() for p in m.parameters()]


def _same(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def test_graphed_trainer_averages_bit_exact(bf16):
    x = (0.5 * torch.randn(2, 1, 65536, device="cuda")).clamp(-1, 1)
    m = _model(0)
    ema = EMA(.99)
    ema.on_train_batch_end(None, m, None, None, 0)          # an average that already exists, before the trainer
    p0, e0, s0 = _snapshot(m), ema.flat.clone(), ema._state.clone()
    tr = GraphedTrainer(m, x, warmup_steps=1, ema=ema)
    torch.cuda.synchronize()
    # constructing the trainer moves neither the model nor the average
    assert _same(_snapshot(m), p0)
    assert torch.equal(ema.flat, e0) and torch.equal(ema._state, s0)

    # one library launch more per graph than the same trainer without an EMA
    m0 = _model(0)
    tr0 = GraphedTrainer(m0, x, warmup_steps=1)
    assert set(tr.launches) == set(tr0.launches) == {True, False}
    for k in tr.launches:
        assert tr.launches[k] == tr0.launches[k] + 1, (k, tr.launches, tr0.launches)

    ref = {n: v.clone() for n, v in ema.state_dict().items()}
    kinds = set()
    for i in range(6):
        kinds.add(m.is_discriminator_step(i))
        tr.step(x, i)
        ref = {n: ref[n] * .99 + p.detach() * (1 - .99) for n, p in m.named_parameters()}
        sd = ema.state_dict()
        for n in ref:
            assert torch.equal(sd[n], ref[n]), (i, n)
    assert kinds == {True, False}
    assert not _same(_snapshot(m), p0)

    # the trainer owns the update: wiring the callback as well would average twice
    with pytest.raises(RuntimeError, match="GraphedTrainer"):
        ema.on_train_batch_end(None, m, None, None, 6)


def _outputs(m, x):
    with torch.no_grad():
        torch.manual_seed(11)
        y = m(x)
        feats = m.discriminator(x)
    return [y] + [t for scale in feats for t in scale]


def test_swap_refreshes_static_prep(bf16):
    """After on_validation_epoch_start the model must compute with the averages: the same outputs, bit for bit, as a
    second model loaded with ema.state_dict() -- through the generator and through the discriminator, whose prepared
    weights a GraphedTrainer keeps in static buffers.  After on_validation_epoch_end, the training weights again."""
    x = (0.5 * torch.randn(2, 1, 65536, device="cuda")).clamp(-1, 1)
    m = _model(1)
    ema = EMA(.5)
    tr = GraphedTrainer(m, x, warmup_steps=1, ema=ema)
    assert tr.static_prep and tr.static_encoder
    for i in range(4):
        tr.step(x, i)
    m.eval()
    train_out = _outputs(m, x)                 # eval-mode prepared weights of the training weights now exist
    train_sd = copy.deepcopy(m.state_dict())
    avg_sd = {n: v.clone() for n, v in ema.state_dict().items()}

    twin = _model(2).eval()
    twin.load_state_dict(train_sd)
    twin.load_state_dict(avg_sd, strict=False)
    ema.on_validation_epoch_start(None, m)
    got, want = _outputs(m, x), _outputs(twin, x)
    for a, b, t in zip(got, want, train_out):
        assert torch.equal(a, b)
    assert not all(torch.equal(a, t) for a, t in zip(got, train_out))     # the averages do change the outputs

    ema.on_validation_epoch_end(None, m)
    twin.load_state_dict(train_sd)
    got, want = _outputs(m, x), _outputs(twin, x)
    for a, b, t in zip(got, want, train_out):
        assert torch.equal(a, b) and torch.equal(a, t)

"""GPU: the validation pass -- rave_latent_moments against numpy float64, validation_step / validation_epoch_end against
the reference's own outputs (tests/golden/validation_*_tiny.pt, oracle/make_golden_validation.py), the receptive-field
probe against the reference's integers, and train -> validate -> build the prior end to end."""
import os

import numpy as np
import pytest
import torch

from oracle import validation_oracle as V
from oracle.spectral_oracle import seeded_params, step_batch, step_eps
from tests.conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _np_moments(z, D):
    x = z[:, :D].double().cpu().permute(0, 2, 1).reshape(-1, D).numpy()
    m = x.mean(0)
    c = x - m
    return x.shape[0], m, c.T @ c


def _moments(z, D, chunks=1):
    from rave_b200 import ops
    state = torch.zeros(1 + D + D * D, dtype=torch.float64, device="cuda")
    for part in z.chunk(chunks, 0):
        ops.latent_moments(part, D, state)
    return state


def _check(state, ref, D, tol=1e-12):
    n, m, M2 = ref
    s = state.cpu().numpy()
    assert s[0] == n
    assert np.abs(s[1:1 + D] - m).max() <= tol * max(1.0, np.abs(m).max())
    assert np.abs(s[1 + D:].reshape(D, D) - M2).max() <= tol * np.abs(M2).max()


@pytest.mark.parametrize("D", [1, 8, 20, 128, 256])
@pytest.mark.parametrize("wide", [False, True])
def test_latent_moments_vs_numpy(D, wide):
    """Rows z[b, :D, t] of z [B, C, L] with C = D or 2D (the mean half of an encoder output, read in place), 3 x 117 = 351
    rows (not a multiple of the row block); chunked accumulation equals one pass; two runs and a graph replay give the same
    bits."""
    torch.manual_seed(D)
    C = 2 * D if wide else D
    z = (torch.randn(3, C, 117, device="cuda") * torch.linspace(0.1, 3, C, device="cuda")[None, :, None] + 0.5)
    zin = z[:, :D] if wide else z
    ref = _np_moments(z, D)
    s1 = _moments(zin, D)
    _check(s1, ref, D)
    _check(_moments(zin, D, chunks=3), ref, D)
    assert torch.equal(s1, _moments(zin, D))
    from rave_b200 import ops
    state = torch.zeros(1 + D + D * D, dtype=torch.float64, device="cuda")
    ops.latent_moments(zin, D, state)                  # warm-up outside the capture
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        state.zero_()
        ops.latent_moments(zin, D, state)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(state, s1)


def test_latent_moments_many_blocks():
    """32 000 rows: the rows split into ~125 blocks merged in order."""
    torch.manual_seed(1)
    z = torch.randn(8, 128, 4000, device="cuda") * 2 + 1
    ref = _np_moments(z, 128)
    _check(_moments(z, 128), ref, 128, tol=1e-11)
    _check(_moments(z, 128, chunks=8), ref, 128, tol=1e-11)


def test_latent_moments_refuses_large_latents():
    from rave_b200 import _lib, ops
    z = torch.randn(1, 257, 64, device="cuda")
    with pytest.raises(_lib.RaveB200Error):
        ops.latent_moments(z, 257, torch.zeros(1 + 257 + 257 * 257, dtype=torch.float64, device="cuda"))


def test_latent_moments_offset_channel_keeps_its_variance():
    """A channel with mean 1e3 and spread 1e-3 (a collapsed latent): its variance to <= 1e-9 relative, where the
    X^T X - n m m^T form in float32 loses every digit."""
    torch.manual_seed(2)
    z = torch.randn(16, 8, 640, device="cuda")
    z[:, 3] = 1e3 + 1e-3 * torch.randn(16, 640, device="cuda")
    n, m, M2 = _np_moments(z, 8)
    s = _moments(z, 8, chunks=4).cpu().numpy()
    var, var_ref = s[1 + 8 + 3 * 8 + 3] / (n - 1), M2[3, 3] / (n - 1)
    assert abs(var - var_ref) <= 1e-9 * var_ref, (var, var_ref)


# ------------------------------------------------------------------------------------------ model against the reference
def _tiny_v2(g):
    from rave_b200 import configs
    torch.manual_seed(0)
    m = configs.build_rave("v2", capacity=g["cfg"]["capacity"], latent_size=g["cfg"]["latent_size"],
                           disc_capacity=g["disc_capacity"])
    # the fixture's encoder / decoder parameters; the discriminator takes no part in validation
    assert not m.load_state_dict(seeded_params(g["param_shapes"], g["param_seed"]), strict=False).unexpected_keys
    return m.cuda().eval()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_validation_step_matches_reference(precision):
    """Logged `validation` and posterior means: fp32 <= 1e-4 / 1e-4 rel-L2, bf16 (wgmma engine) <= 3 % / 3e-2."""
    import rave_b200
    g = _load("validation_v2_tiny.pt")
    m = _tiny_v2(g)
    tol_v, tol_m = (1e-4, 1e-4) if precision == "fp32" else (3e-2, 3e-2)
    rave_b200.set_precision(precision)
    try:
        B, T, D = g["B"], g["T"], g["cfg"]["latent_size"]
        for i, b in enumerate(g["batches"]):
            x = step_batch(B, T, b["x_seed"])
            eps = step_eps(B, D, T // 2048, b["eps_seed"])
            xy, mean = m.validation_step(x.cuda(), i, eps=eps.cuda())
            v, want = float(m.logged["validation"]), float(b["validation"])
            assert abs(v - want) <= tol_v * abs(want), (i, v, want)
            assert rel_l2(mean, b["mean"]) <= tol_m, (i, rel_l2(mean, b["mean"]))
            assert xy.shape[-1] == 2 * T and torch.equal(xy[..., :T].cpu(), x)
    finally:
        rave_b200.set_precision("fp32")


def test_validation_epoch_end_matches_reference():
    """latent_mean / latent_pca / fidelity from the fixture's means: fidelity <= 1e-5 of the reference's, each component
    separated from its neighbours by >= 1e-3 with the same sign and |cos| >= 0.9999; against the float64 oracle
    fidelity <= 1e-6 and cos >= 0.99999."""
    g = _load("validation_v2_tiny.pt")
    m = _tiny_v2(g)
    m.set_receptive_field(*g["receptive_field"])
    m.validation_epoch_end([(None, b["mean"].cuda()) for b in g["batches"]])
    assert m.eval_number == 1
    fid, pca, lm = m.fidelity.cpu(), m.latent_pca.cpu(), m.latent_mean.cpu()
    assert (fid - g["fidelity"]).abs().max() <= 1e-5
    assert (lm - g["latent_mean"]).abs().max() <= 1e-5
    _, c_o, ev_o, f_o = V.latent_analysis([b["mean"] for b in g["batches"]])
    assert np.abs(fid.double().numpy() - f_o).max() <= 1e-6
    sep = V.separated(ev_o)
    assert sep
    for i in sep:
        assert float(pca[i].double() @ g["latent_pca"][i].double()) >= 0.9999, i
        assert float(np.dot(pca[i].double().numpy(), c_o[i])) >= 0.99999, i
    for k, v in g["fidelity_logs"].items():
        assert float(m.logged[k]) == float(v), k


def test_probe_matches_reference_on_tiny_models():
    from rave_b200 import configs
    g = _load("validation_v2_tiny.pt")
    m = _tiny_v2(g).train()
    assert tuple(m.receptive_field.tolist()) == (0, 0)
    m.validation_epoch_end([])
    assert tuple(m.receptive_field.tolist()) == g["receptive_field"] and m.training
    h = _load("validation_hybrid_tiny.pt")
    mh = configs.build_rave("v2_hybrid", capacity=h["cfg"]["capacity"], latent_size=h["cfg"]["latent_size"],
                            disc_capacity=h["disc_capacity"])
    assert not mh.load_state_dict(seeded_params(h["param_shapes"], h["param_seed"]), strict=False).unexpected_keys
    mh.cuda().train()
    from rave_b200 import core
    assert core.get_rave_receptive_field(mh) == h["receptive_field"]
    assert all(mod.enabled for mod in mh.modules() if hasattr(mod, "gru_state"))
    assert all(p.grad is None for p in mh.parameters())


@pytest.mark.parametrize("name", ["v2", "v2_small"])
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_probe_full_size_matches_reference(name, precision):
    import rave_b200
    from rave_b200 import configs, core, engine
    want = _load("validation_v2_tiny.pt")["full_size_receptive_field"][name]
    torch.manual_seed(0)
    m = configs.build_rave(name, disc_capacity=4).cuda()
    rave_b200.set_precision(precision)
    try:
        got = core.get_rave_receptive_field(m)
        if name == "v2_small":
            # the reference's NoiseGeneratorV2 filters by FFT convolution, whose rounding reaches two samples past the
            # FIR's support on the left; the fused FIR kernel here has exact zeros there (DESIGN §5.7)
            assert got[1] == want[1] and 0 <= want[0] - got[0] <= 2, (got, want)
        else:
            assert got == want
        assert engine.precision() == precision
    finally:
        rave_b200.set_precision("fp32")


# ------------------------------------------------------------------------------------------ end to end
def test_train_validate_build_prior():
    """A few graphed training steps, a validation epoch, then build_prior(fidelity=0.95) and one graphed prior step; a
    graphed step after a validation epoch (receptive field already set) gives the same bits as without that epoch."""
    from rave_b200 import configs
    from rave_b200.graphs import GraphedTrainer
    from rave_b200.prior import GraphedPriorTrainer

    def model():
        torch.manual_seed(0)
        m = configs.build_rave("v2", capacity=16, latent_size=16, disc_capacity=8).cuda().train()
        m.set_receptive_field(27117, 26428)
        return m

    torch.manual_seed(5)
    # 131072 samples (train.py's crop): the multiband loss keeps 8192 - (27117 + 26428) / 16 frames after the crop
    x = (0.5 * torch.randn(2, 1, 131072, device="cuda")).clamp(-1, 1)
    val = [(0.5 * torch.randn(4, 1, 131072, device="cuda")).clamp(-1, 1) for _ in range(3)]
    m = model()
    tr = GraphedTrainer(m, x, warmup_steps=2)
    for i in range(3):
        torch.cuda.manual_seed(10 + i)
        tr.step(x, i)
    m.eval()
    out = [m.validation_step(v, i) for i, v in enumerate(val)]
    m.validation_epoch_end(out)
    m.train()
    assert m.eval_number == 1 and float(m.fidelity[-1]) == pytest.approx(1.0, abs=1e-5)
    assert not torch.equal(m.latent_pca.cpu(), torch.eye(16))
    torch.cuda.manual_seed(20)
    logs_after = {k: v.clone() for k, v in tr.step(x, 3).items() if torch.is_tensor(v)}

    twin = model()
    tr2 = GraphedTrainer(twin, x, warmup_steps=2)
    for i in range(3):
        torch.cuda.manual_seed(10 + i)
        tr2.step(x, i)
    torch.cuda.manual_seed(20)
    logs_plain = tr2.step(x, 3)
    for k, v in logs_plain.items():                 # logs_after also holds the epoch's `validation` and fidelities
        if torch.is_tensor(v):
            assert torch.equal(logs_after[k], v), k

    prior = configs.build_prior(m, fidelity=0.95, resolution=8, res_size=32, skp_size=16, cycle_size=2, n_layers=3).cuda()
    ptr = GraphedPriorTrainer(prior, val[0])
    loss = ptr.step(val[0])
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()

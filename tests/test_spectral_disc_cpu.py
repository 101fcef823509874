"""CPU: the multi-scale spectral discriminator (rave/discriminator.py:12-74, 139-153; configs/spectral_discriminator.gin).
The oracle restatement reproduces the goldens the unmodified reference wrote (oracle/make_golden_spectral.py),
the "v2_spectral" model has the reference's state_dict, and the module's fp32 forward runs its shape logic on CPU
tensors up to the first library call."""
import math
import os

import pytest
import torch

from oracle import rave_oracle as O
from oracle import spectral_oracle as S
from tests.conftest import GOLDEN, rel_l2


def load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def test_spectral_discriminator_oracle_matches_reference_golden():
    g = load("discriminator_spectral.pt")
    feats = S.multi_scale_spectral_discriminator(g["x"], g["params"], "discriminator.", g["scales"])
    assert len(feats) == 5 and all(len(f) == 6 for f in feats)
    for fa, fb in zip(feats, g["features"]):
        for a, (shape, idx, val) in zip(fa, fb):
            assert tuple(a.shape) == tuple(shape) and rel_l2(a.reshape(-1)[idx], val) <= 1e-6, (shape,)
    fm, ld, la = O.gan_losses(feats, 1, True)
    assert rel_l2(fm, g["fm"]) <= 1e-6 and rel_l2(ld, g["loss_dis"]) <= 1e-6 and rel_l2(la, g["loss_adv"]) <= 1e-6


def test_spectral_training_step_restatement_reproduces_reference_steps():
    """training_step_v2_spectral_tiny.pt: a phase-2 D-step and G-step of the reference's own RAVE.training_step with the
    MSD + spectral discriminator, from seeded parameters; the restatement's logged losses."""
    g = load("training_step_v2_spectral_tiny.pt")
    cfg = O.ArchConfig(**g["cfg"])
    sd = dict(S.seeded_params(g["param_shapes"], g["param_seed"]), **{"pqmf.hk": g["hk"]})
    Lz = g["T"] // cfg.n_band // math.prod(cfg.ratios)
    for st in g["steps"]:
        x = S.step_batch(g["B"], g["T"], st["seed"])
        eps = S.step_eps(g["B"], cfg.latent_size, Lz, st["seed"])
        parts, loss_dis = S.train_step_losses(x, sd, cfg, eps, receptive_field=tuple(g["receptive_field"]))
        for k, v in parts.items():
            assert rel_l2(v, st["logs"][k]) <= 1e-6, (st["name"], k)
        assert rel_l2(loss_dis, st["logs"]["loss_dis"]) <= 1e-6


def test_v2_spectral_state_dict_contract_full_size():
    from rave_b200 import configs
    ks = load("state_dict_keys_spectral.pt")["rave_v2_spectral"]
    sd = {k: (tuple(v.shape), str(v.dtype)) for k, v in configs.build_rave("v2_spectral").state_dict().items()}
    assert set(sd) == set(ks), sorted(set(sd) ^ set(ks))[:20]
    assert sd == ks, [k for k in sd if sd[k] != ks[k]][:20]


def test_tiny_spectral_golden_state_dicts_load_strictly():
    from rave_b200 import configs
    g = load("training_step_v2_spectral_tiny.pt")
    m = configs.build_rave("v2_spectral", capacity=g["cfg"]["capacity"], latent_size=g["cfg"]["latent_size"],
                           disc_capacity=g["disc_capacity"], spectral_capacity=g["spectral_capacity"])
    sd = m.state_dict()
    params = S.seeded_params(g["param_shapes"], g["param_seed"])
    assert set(params) == {k for k, _ in m.named_parameters() if not k.startswith("pqmf.")}
    for k, v in params.items():
        assert sd[k].shape == v.shape, k
    m.load_state_dict(dict(sd, **params), strict=True)
    assert torch.equal(m.state_dict()["pqmf.hk"], g["hk"])


def test_spectral_discriminator_cpu_shape_logic_reaches_the_library():
    """Spectrogram (torch.stft on CPU tensors: uncentred, divided by ||window||_2) and the first conv's time-stacked
    operand; the conv itself is a library call, which refuses host tensors (no CPU fallback)."""
    from rave_b200 import _lib
    from rave_b200.discriminator import EncodecConvNet, MultiScaleSpectralDiscriminator, SpectralConv2d, spectrogram
    from functools import partial
    torch.manual_seed(0)
    x = torch.randn(2, 1, 4096 + 5)
    spec = spectrogram(1024)
    assert list(dict(spec.state_dict())) == ["window"]
    z = spec(x)
    want = S.spectrogram(x, 1024)
    assert z.shape == want.shape == (2, 1, 513, 1 + (4096 + 5 - 1024) // 256)
    assert rel_l2(torch.view_as_real(z), torch.view_as_real(want)) <= 1e-6
    net = EncodecConvNet(capacity=4)
    convs = net.convs()
    assert all(isinstance(c, SpectralConv2d) for c in convs)
    assert [c.dilation for c in convs] == [(1, 1), (1, 1), (1, 2), (1, 4), (1, 1), (1, 1)]
    assert [c.padding for c in convs] == [(4, 1), (4, 1), (4, 2), (4, 4), (1, 1), (1, 1)]
    assert [c.stride for c in convs] == [(1, 1), (2, 1), (2, 1), (2, 1), (1, 1), (1, 1)]
    with pytest.raises(_lib.RaveB200Error, match="CUDA"):
        net(torch.cat([z.real, z.imag], 1))
    disc = MultiScaleSpectralDiscriminator([1024, 512], partial(EncodecConvNet, capacity=4))
    assert not disc.engine_ready(x)
    with pytest.raises(_lib.RaveB200Error, match="CUDA"):
        disc(x)
    with pytest.raises(_lib.RaveB200Error):
        SpectralConv2d(2, 4, (9, 3), padding=(4, 2), dilation=(1, 1))     # time padding must be dt (kt - 1) / 2

"""CPU: the two v2 regularisation options (`--config v2 --config wasserstein` / `spherical`) -- module trees against the
reference's, the build_rave bindings, which encoder a phase-2 graph may freeze, the oracle restatement against the
reference's fixtures, and the host branch of WasserteinEncoder.reparametrize against the reference's expression."""
import os

import pytest
import torch

from oracle import regularization_oracle as G
from oracle import rave_oracle as O
from tests.conftest import GOLDEN, rel_l2


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _loss_err(got, want, floor=1e-2):
    """Relative error with the scale floored at `floor` (oracle/make_golden_regularization.py::check_loss)."""
    return abs(float(got) - float(want)) / max(abs(float(want)), floor)


@pytest.mark.parametrize("kind", ["wasserstein", "spherical"])
def test_state_dict_matches_reference(kind):
    from rave_b200 import configs
    want = _load("state_dict_keys_regularization.pt")[f"rave_v2_{kind}"]
    m = configs.build_rave(f"v2_{kind}")
    got = {k: (tuple(v.shape), str(v.dtype)) for k, v in m.state_dict().items()}
    assert list(got) == list(want)
    assert got == want


@pytest.mark.parametrize("kind", ["wasserstein", "spherical"])
def test_build_rave_bindings(kind):
    from rave_b200 import blocks, configs
    m = configs.build_rave(f"v2_{kind}")
    enc_cls = blocks.WasserteinEncoder if kind == "wasserstein" else blocks.SphericalEncoder
    assert type(m.encoder) is enc_cls
    assert m.latent_size == 16 and m.latent_pca.shape == (16, 16)
    assert m.encoder.encoder.net[-1].out_channels == 16                  # EncoderV2.n_out = 1
    assert m.decoder.net[0].in_channels == (144 if kind == "wasserstein" else 16)
    assert m.warmup == 200000
    if kind == "wasserstein":
        assert m.encoder.noise_augmentation == 128
        assert m.weights == {"audio_distance": 1., "multiband_audio_distance": 1., "adversarial": 2,
                             "feature_matching": 20, "fullband_spectral_distance": 2, "multiband_spectral_distance": 2}
    else:
        assert m.weights == {"audio_distance": 1., "multiband_audio_distance": 1., "adversarial": 1.,
                             "feature_matching": 20}
    small = configs.build_rave(f"v2_{kind}", latent_size=8, capacity=8, disc_capacity=4)
    assert small.encoder.encoder.net[-1].out_channels == 8
    with pytest.raises(NotImplementedError):
        configs.build_rave(f"v2_{kind}", hybrid=True)


def test_existing_configurations_keep_their_bindings():
    from rave_b200 import blocks, configs
    m = configs.build_rave("v2", capacity=8, disc_capacity=4)
    assert type(m.encoder) is blocks.VariationalEncoder and m.latent_size == 128
    assert m.encoder.encoder.net[-1].out_channels == 256
    assert m.weights["feature_matching"] == 20 and m.weights["adversarial"] == 1.


def test_encoder_is_frozen_only_for_the_detaching_encoders():
    from rave_b200 import configs
    from rave_b200.graphs import _encoder_is_frozen
    for kind, frozen in (("wasserstein", True), ("spherical", False)):
        m = configs.build_rave(f"v2_{kind}", capacity=8, disc_capacity=4)
        assert not _encoder_is_frozen(m)
        m.warmed_up = True
        assert _encoder_is_frozen(m) is frozen, kind


def test_oracle_autoencoder_vs_fixture():
    fx = _load("autoencoder_v2_wasserstein_tiny.pt")
    cfg = O.ArchConfig(**fx["cfg"])
    sd = fx["state_dict"]
    po = {k: v.clone().requires_grad_(v.is_floating_point() and not k.startswith("pqmf.")) for k, v in sd.items()}
    x = fx["x"].clone().requires_grad_(True)
    taps = {}
    y, reg = G.rave_forward(x, po, cfg, "wasserstein", fx["prior"], fx["noise"], taps)
    assert rel_l2(y, fx["y"]) < 1e-6
    assert rel_l2(taps["z"], fx["z"]) < 1e-6
    assert rel_l2(reg, fx["mmd"]) < 1e-6
    terms = torch.stack(G.mmd_terms(fx["z"], fx["prior"]))
    assert rel_l2(terms, fx["mmd_terms"]) < 1e-6
    names = sorted(fx["grad_params"])
    g = torch.autograd.grad((y * fx["probe"]).sum() + fx["beta"] * reg, [x] + [po[n] for n in names])
    assert rel_l2(g[0], fx["grad_x"]) < 1e-5
    for n, a in zip(names, g[1:]):
        assert rel_l2(a, fx["grad_params"][n]) < 1e-5, n


@pytest.mark.parametrize("kind", ["wasserstein", "spherical"])
def test_oracle_training_step_vs_fixture(kind):
    fx = _load(f"training_step_v2_{kind}_tiny.pt")
    cfg = O.ArchConfig(**fx["cfg"])
    sd = G.seeded_params(fx["param_shapes"], fx["param_seed"])
    sd["pqmf.hk"] = fx["hk"]
    B, T = fx["B"], fx["T"]
    Lz = T // cfg.n_band // int(torch.tensor(cfg.ratios).prod())
    for st in fx["steps"]:
        x = G.step_batch(B, T, st["seed"])
        prior, noise = G.draws(B, cfg.latent_size, Lz, st["seed"]) if kind == "wasserstein" else (None, None)
        losses, ldis, _ = G.train_step_losses(x, sd, cfg, kind, st["warmed_up"], prior, noise, fx["beta_factor"],
                                              receptive_field=fx["receptive_field"])
        for k, v in losses.items():
            if k == "regularization" and k not in st["logs"]:      # the reference skips a zero regulariser
                assert kind == "spherical" and float(v) == 0.0
                continue
            assert _loss_err(v, st["logs"][k]) < 2e-6, (st["name"], k)
        if st["warmed_up"]:
            assert _loss_err(ldis, st["logs"]["loss_dis"]) < 2e-6
    names = [st["name"] for st in fx["steps"]]
    assert names == (["phase1_gen", "phase2_dis", "phase2_gen"] if kind == "wasserstein" else
                     ["phase1_gen", "phase2_gen"])
    # the WAE's phase-1 encoder gradient carries the MMD term; in phase 2 its encoder is detached, the sphere's is not
    enc = {st["name"]: st.get("encoder_sample") for st in fx["steps"]}
    assert enc["phase1_gen"] is not None
    assert (enc["phase2_gen"] is None) == (kind == "wasserstein")


def test_wae_host_reparametrize_vs_reference_expression():
    """The CPU branch: the reference's expression on injected draws, and by default the draws in the reference's order
    (prior sample first, then the noise)."""
    from rave_b200 import blocks
    enc = blocks.WasserteinEncoder(lambda n_channels: torch.nn.Identity(), noise_augmentation=128)
    g = torch.Generator().manual_seed(5)
    z = torch.randn(3, 16, 7, generator=g, dtype=torch.float64)
    prior, noise = G.draws(3, 16, 7, 9)
    prior, noise = prior.double(), noise.double()
    zs, reg = enc.reparametrize(z, (prior, noise))
    assert torch.equal(zs, torch.cat([z, noise], 1))
    assert torch.equal(reg, G.mmd(z, prior))
    x = z.permute(0, 2, 1).reshape(-1, 16)
    direct = sum(torch.exp(-((a[:, None] - b[None]) ** 2).sum(2) / 256).mean() * s
                 for a, b, s in ((x, x, 1), (prior, prior, 1), (x, prior, -2)))
    assert abs(float(reg) - float(direct)) < 1e-12
    z32 = z.float()
    torch.manual_seed(9)
    zs2, reg2 = enc.reparametrize(z32)
    p32, n32 = G.draws(3, 16, 7, 9)
    assert torch.equal(zs2[:, 16:], n32)
    assert torch.equal(reg2, G.mmd(z32, p32))
    enc0 = blocks.WasserteinEncoder(lambda n_channels: torch.nn.Identity())
    zs3, _ = enc0.reparametrize(z32, (p32, None))
    assert zs3 is z32


def test_sphere_host_reparametrize_and_warm_up_flags():
    from rave_b200 import blocks
    z = torch.randn(2, 16, 5)
    sph = blocks.SphericalEncoder(lambda n_channels: torch.nn.Identity())
    out, reg = sph.reparametrize(z)
    want, _ = G.reparametrize(z, "spherical")
    assert torch.equal(out, want) and float(reg) == 0.0
    sph.set_warmed_up(True)
    zi = z.clone().requires_grad_(True)
    assert sph(zi).requires_grad                               # keeps training in phase 2
    wae = blocks.WasserteinEncoder(lambda n_channels: torch.nn.Identity())
    wae.set_warmed_up(True)
    assert int(wae.warmed_up) == 1 and not wae(zi).requires_grad
    wae.set_warmed_up(False)
    assert int(wae.warmed_up) == 0 and wae(zi).requires_grad

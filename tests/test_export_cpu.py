"""CPU: the float64 oracle of the exported model's latent arithmetic against the fixture the unmodified reference
produced (tests/golden/export_latent.pt, oracle/make_golden_export.py), and the host logic of rave_b200.ExportedRAVE --
the latent_size rules, the `channels` handling and the AdaIN flag sequence -- with the CUDA library ops replaced by the
oracle (test infrastructure; the product has no CPU path).  The GPU twin is tests/test_gpu_export.py."""
import os

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import export_oracle as EO
from rave_b200 import blocks, ops, quantization
from rave_b200.export import ExportedRAVE
from tests.conftest import GOLDEN


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(GOLDEN, "export_latent.pt"), weights_only=False)


def _close(a, b, tol=1e-12):
    assert a.shape == b.shape
    assert torch.allclose(a, b, rtol=tol, atol=tol), (a - b).abs().max()


# ------------------------------------------------------------------ oracle vs reference
def test_variational_oracle_matches_reference(fx):
    for c in fx["variational"]:
        _close(EO.variational_post(c["z"], c["eps"], c["latent_mean"], c["latent_pca"], c["l"]), c["post"])
        _close(EO.variational_pre(c["post"], c["noise"], c["latent_mean"], c["latent_pca"]), c["pre"])


def test_discrete_oracle_matches_reference(fx):
    for c in fx["discrete"]:
        assert torch.equal(EO.rvq_encode(c["x"], c["codebooks"]).double(), c["codes"]), c["name"]
        noise = c["noise"] if c["noise"].shape[1] else None
        _close(EO.rvq_decode(c["decode_in"], c["codebooks"], noise), c["pre"])


def test_wasserstein_oracle_matches_reference(fx):
    for c in fx["wasserstein"]:
        assert torch.equal(c["post"], c["z"])
        noise = c["noise"] if c["noise"].shape[1] else None
        assert torch.equal(EO.wasserstein_pre(c["z"], noise), c["pre"])


def test_spherical_oracle_matches_reference(fx):
    for c in fx["spherical"]:
        got, want = EO.sphere_to_angles(c["x"]), c["angles"]
        assert torch.equal(torch.isnan(got), torch.isnan(want)), c["name"]
        fin = ~torch.isnan(want)
        _close(got[fin], want[fin])
        assert torch.isnan(got[-1, :, -1]).all()                   # the all-zero frame
        _close(EO.angles_to_sphere(c["angles_in"]), c["sphere"])


def test_latent_size_rules(fx):
    for c in fx["latent_size"]:
        assert EO.latent_size("variational", c["fidelity"], c["f"]) == c["latent_size"], c["name"]
    assert EO.latent_size("discrete", num_quantizers=16) == 16
    assert EO.latent_size("wasserstein", full=16) == 16
    assert EO.latent_size("spherical", full=16) == 15


# ------------------------------------------------------------------ ExportedRAVE host logic
@pytest.fixture
def oracle_ops(monkeypatch):
    for name in ("rvq_encode", "rvq_decode", "sphere_to_angles", "angles_to_sphere"):
        monkeypatch.setattr(ops, name, getattr(EO, name))
    monkeypatch.setattr(ops, "latent_project", EO.variational_post)
    monkeypatch.setattr(ops, "latent_unproject", EO.variational_pre)


class FakeRAVE(nn.Module):
    """The attributes and methods ExportedRAVE reads: encode = a strided conv, decode = a transposed conv with one extra
    output sample (cropped by ExportedRAVE), latent buffers, update_adain."""

    def __init__(self, encoder, latent_size, n_channels=1, ratio=4, enc_out=None, dec_in=None, dec_weight=None,
                 adain=False):
        super().__init__()
        g = torch.Generator().manual_seed(5)
        self.encoder, self.latent_size, self.n_channels, self.ratio = encoder, latent_size, n_channels, ratio
        self.register_buffer("latent_pca", torch.linalg.qr(torch.randn(latent_size, latent_size, generator=g))[0])
        self.register_buffer("latent_mean", torch.randn(latent_size, generator=g) * .1)
        self.register_buffer("fidelity", torch.linspace(.5, 1., latent_size))
        self.w_enc = torch.randn(enc_out or latent_size, n_channels, ratio, generator=g)
        self.w_dec = dec_weight if dec_weight is not None else torch.randn(dec_in or latent_size, n_channels,
                                                                           ratio + 1, generator=g)
        self.adain = blocks.AdaptiveInstanceNormalization(2) if adain else None
        self.adain_calls = []

    def encode(self, x):
        return F.conv1d(x, self.w_enc.to(x.dtype), stride=self.ratio)

    def decode(self, z):
        return F.conv_transpose1d(z, self.w_dec.to(z.dtype), stride=self.ratio)

    def update_adain(self, *flags):
        self.adain_calls.append(tuple(bool(f) for f in flags))
        return blocks.update_adain(self, *flags)


def _identity(n_channels=1):
    return nn.Identity()


def test_latent_size_and_value_errors(oracle_ops):
    m = FakeRAVE(blocks.VariationalEncoder(_identity), 8, enc_out=16)
    m.fidelity.copy_(torch.linspace(.5, 1., 8))                       # first index above .95: 7 -> 8
    assert ExportedRAVE(m, fidelity=.95).latent_size == 8
    assert ExportedRAVE(m, fidelity=.7).latent_size == 4              # index 3 -> 4
    m6 = FakeRAVE(blocks.VariationalEncoder(_identity), 6, enc_out=12)
    m6.fidelity.copy_(torch.linspace(.5, 1., 6))                      # index 5 -> 8 > 6
    with pytest.raises(ValueError):
        ExportedRAVE(m6, fidelity=.95)
    m6.fidelity.zero_()                                               # untrained: 1
    assert ExportedRAVE(m6).latent_size == 1
    with pytest.raises(ValueError):
        ExportedRAVE(FakeRAVE(nn.Identity(), 4))
    with pytest.raises(ValueError):
        ExportedRAVE(FakeRAVE(blocks.WasserteinEncoder(_identity), 2, adain=True), channels=2)
    sph = ExportedRAVE(FakeRAVE(blocks.SphericalEncoder(_identity), 5))
    assert (sph.latent_size, sph.full_latent_size, sph.encode_ratio) == (4, 5, 4)
    rvq = lambda: quantization.ResidualVectorQuantization(num_quantizers=3, dim=4, codebook_size=8)  # noqa: E731
    disc = ExportedRAVE(FakeRAVE(blocks.DiscreteEncoder(_identity, rvq, 3, noise_augmentation=2), 4, dec_in=6))
    assert (disc.latent_size, disc.n_noise) == (3, 2)


def test_channels_match_reference_at_batch_one(fx, oracle_ops):
    for c in fx["channels"]:
        nc, tc, w = c["n_channels"], c["target_channels"], c["weight"]
        C = c["z"].shape[1]
        n_noise = w.shape[0] - C
        m = FakeRAVE(blocks.WasserteinEncoder(_identity, noise_augmentation=n_noise), C, n_channels=nc,
                     ratio=c["ratio"], dec_weight=w).double()
        ex = ExportedRAVE(m, channels=tc)
        assert (ex.target_channels, ex.encode_ratio) == (tc, c["ratio"])
        y = ex.decode(c["z"].float(), noise=c["noise"].float())
        assert y.shape == c["y"].shape, c["name"]
        # the model ran in float32 here (ExportedRAVE's latent path is fp32): float32 tolerance against float64
        assert torch.allclose(y.double(), c["y"], rtol=1e-5, atol=1e-5), c["name"]


def test_channels_shapes_and_batch_rows(oracle_ops):
    m = FakeRAVE(blocks.WasserteinEncoder(_identity, noise_augmentation=1), 3, n_channels=1, dec_in=4)
    ex = ExportedRAVE(m, channels=3)
    z = torch.randn(2, 3, 5)
    noise = torch.randn(6, 1, 5)
    y = ex.decode(z, noise=noise)
    assert y.shape == (2, 3, 20)
    for b in range(2):
        for i in range(3):
            one = m.decode(torch.cat([z[b:b + 1], noise[3 * b + i:3 * b + i + 1]], 1))[..., :20]
            assert torch.allclose(y[b, i], one[0, 0], rtol=1e-6, atol=1e-6)    # batched vs single conv
    with pytest.raises(ValueError):
        ex.decode(z, noise=torch.randn(2, 1, 5))                        # one draw per decoded row is needed
    m2 = FakeRAVE(blocks.WasserteinEncoder(_identity), 3, n_channels=2)
    assert ExportedRAVE(m2, channels=1).decode(torch.randn(2, 3, 5)).shape == (2, 1, 20)


def test_latent_round_trips_through_the_oracle_ops(oracle_ops):
    m = FakeRAVE(blocks.VariationalEncoder(_identity), 4, enc_out=8)
    m.fidelity.copy_(torch.tensor([.5, .97, .99, 1.]))
    ex = ExportedRAVE(m)
    x = torch.randn(2, 1, 32)
    eps = torch.randn(2, 4, 8)
    z = ex.encode(x, eps=eps)
    assert z.shape == (2, ex.latent_size, 8) and ex.latent_size == 1
    want = EO.variational_post(m.encode(x), eps, m.latent_mean, m.latent_pca, 1)
    assert torch.equal(z, want)
    noise = torch.randn(2, 3, 8)
    assert torch.equal(ex.decode(z, noise=noise), m.decode(EO.variational_pre(z, noise, m.latent_mean,
                                                                              m.latent_pca))[..., :32])


def test_adain_flag_sequence(oracle_ops):
    m = FakeRAVE(blocks.WasserteinEncoder(_identity), 2, adain=True)
    ex = ExportedRAVE(m)
    assert ex.is_using_adain and m.adain_calls == [(False, False, False, False)]   # the encode of the constructor
    m.adain_calls.clear()
    x = torch.randn(1, 1, 16)
    ex.learn_target, ex.reset_source = True, True
    z = ex.encode(x)
    assert m.adain_calls[-1] == (True, False, False, True) and m.adain.learn_y.item() == 1
    assert not ex.reset_source and ex.learn_target                    # resets clear, learn flags stay
    ex.decode(z)
    assert m.adain_calls[-1] == (True, False, False, False)
    ex.learn_target, ex.learn_source, ex.reset_target = False, True, True
    n = len(m.adain_calls)
    ex(x)                                                             # forward: one application, before encode
    assert m.adain_calls[n:] == [(False, True, True, False)] and not ex.reset_target
    assert m.adain.learn_x.item() == 1 and m.adain.learn_y.item() == 0

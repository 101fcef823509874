"""Training-batch transforms without a GPU: the numpy restatement (oracle/transforms_oracle.py) against the reference's
own outputs (tests/golden/transforms.pt), the host draw logic of rave_b200/transforms.py and its argument errors."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import transforms_oracle as TO
from oracle.make_golden_transforms import make_input
from rave_b200 import transforms as T

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "transforms.pt")


def _fixture():
    return torch.load(GOLDEN, weights_only=False)


def _case_inputs(case):
    C, N, L, seed = case["C"], case["N"], case["L"], case["seed"]
    raw = make_input(seed, C, L, case["kind"])
    np.random.seed(seed)
    noise = np.random.rand(C, N)
    return raw, noise


def test_restatement_matches_reference_fixture_exactly():
    fx = _fixture()
    assert len(fx["cases"]) >= 10
    for case in fx["cases"]:
        raw, noise = _case_inputs(case)
        got = TO.transform_example(raw, case["N"], case["draws"].tolist(), noise, case["normalize"],
                                   case["derivative"])
        ref = case["out"].numpy()
        assert np.array_equal(got.view(np.int32), ref.view(np.int32)), case["name"]


def test_fixture_covers_the_paths():
    cases = _fixture()["cases"]
    d = torch.stack([c["draws"] for c in cases])
    assert (d[:, 1] == 1).any() and (d[:, 1] == 0).any()          # allpass applied and skipped
    assert (d[:, 3] == 0).any() and (d[:, 3] == 1).any()          # muted and kept
    assert {c["C"] for c in cases} == {1, 2}
    assert any(c["normalize"] and c["draws"][1] == 0 for c in cases)
    assert any(c["kind"] == "silent" and c["normalize"] for c in cases)
    assert any(c["derivative"] for c in cases) and any("gain" in c["augmentations"] for c in cases)


def test_crop_offsets_inclusive_range():
    g = torch.Generator().manual_seed(0)
    d = T.sample_draws(20000, 110, 100, 44100, generator=g)
    off = d[:, 0]
    assert off.min() == 0 and off.max() == 10 and torch.equal(off, off.floor())
    counts = torch.bincount(off.long(), minlength=11).double()
    assert (counts - 20000 / 11).abs().max() < 5 * math.sqrt(20000 / 11)
    d0 = T.sample_draws(50, 100, 100, 44100, generator=g)          # L = n_signal: offset 0 only
    assert (d0[:, 0] == 0).all()


def test_apply_rate_log_uniform_frequency_and_keep_rate():
    g = torch.Generator().manual_seed(1)
    n = 200000
    d = T.sample_draws(n, 10, 10, 48000, keep_prob=0.9, generator=g)
    assert abs(d[:, 1].mean().item() - 0.8) < 5 * math.sqrt(0.16 / n)
    assert abs(d[:, 3].mean().item() - 0.9) < 5 * math.sqrt(0.09 / n)
    f = d[:, 2] * 48000 / (2 * math.pi)
    assert f.min() >= 20 * (1 - 1e-12) and f.max() <= 2000 * (1 + 1e-12)
    lf = (f.log() - math.log(20)) / (math.log(2000) - math.log(20))
    hist = torch.histc(lf, bins=20, min=0, max=1)
    assert (hist - n / 20).abs().max() < 5 * math.sqrt(n / 20)
    # the same formula as random_angle for the same uniform
    u = torch.rand(100, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    lo, hi = math.log(20), math.log(2000)
    omega = torch.exp(u * (hi - lo) + lo) * (2 * math.pi) / 48000
    ref = np.array([TO.random_angle(float(v), 20, 2000, 48000) for v in u])
    np.testing.assert_allclose(omega.numpy(), ref, rtol=4e-16, atol=0)


def test_coefficients_are_the_references_allpass():
    for omega in (2 * math.pi * 20 / 44100, 0.1, 2 * math.pi * 2000 / 44100):
        b, a = TO.pole_to_z_filter(omega, .99)
        re, im = .99 * math.cos(omega), .99 * math.sin(omega)
        r2 = math.hypot(re, im) ** 2
        np.testing.assert_allclose(b, [r2, -2 * re, 1], rtol=1e-15)
        np.testing.assert_allclose(a, [1, -2 * re, r2], rtol=1e-15)
        # allpass: unit magnitude response
        w = np.exp(-1j * np.linspace(0, np.pi, 33))
        h = np.polyval(b[::-1], w) / np.polyval(a[::-1], w)
        np.testing.assert_allclose(np.abs(h), 1, rtol=1e-9)


def test_mute_probability_combines_and_gain_is_identity():
    t = T.get_transforms(44100, 100, augmentations=[T.RandomMute(0.1), T.RandomGain(), T.RandomMute(0.5)])
    assert t.keep_prob == pytest.approx(0.9 * 0.5)
    assert T.get_transforms(44100, 100).keep_prob == 1.0


@pytest.mark.parametrize("kwargs", [dict(rand_pitch=[0.7, 1.3]), dict(sr_dataset=48000)])
def test_not_built_options_raise(kwargs):
    with pytest.raises(NotImplementedError):
        T.get_transforms(44100, 100, **kwargs)


@pytest.mark.parametrize("name", ["Compress", "RandomCompress", "FrequencyMasking", "Unknown"])
def test_not_built_augmentations_raise(name):
    aug = type(name, (), {})()
    with pytest.raises(NotImplementedError):
        T.get_transforms(44100, 100, augmentations=[aug])


def test_malformed_input_raises():
    t = T.get_transforms(44100, 100, n_channels=2)
    with pytest.raises(ValueError):
        t(torch.zeros(2, 2, 200, dtype=torch.int16))            # CPU tensor
    with pytest.raises(ValueError):
        t(np.zeros((2, 2, 200), np.int16))
    if torch.cuda.is_available():
        with pytest.raises(TypeError):
            t(torch.zeros(2, 2, 200, dtype=torch.float64, device="cuda"))
        with pytest.raises(ValueError):
            t(torch.zeros(2, 2, 99, dtype=torch.int16, device="cuda"))
        with pytest.raises(ValueError):
            t(torch.zeros(2, 1, 200, dtype=torch.int16, device="cuda"))

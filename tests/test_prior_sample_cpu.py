"""CPU: the float64 restatement of the prior's sampler and class decode (tests/prior_sample_ref.py) against the
reference's fixtures (tests/golden/prior_tiny.pt) and a direct cumulative sum."""
import math
import os

import pytest
import torch

from oracle import prior_oracle as P
from tests import prior_sample_ref as S
from tests.conftest import GOLDEN, rel_l2


@pytest.fixture(scope="module")
def fx():
    return torch.load(os.path.join(GOLDEN, "prior_tiny.pt"), weights_only=False)


def test_oracle_argmax_sample_reproduces_reference_generate(fx):
    R, D, cfg = fx["prior_cfg"]["resolution"], fx["D"], fx["prior_cfg"]
    sd = P.seeded_params(fx["prior_param_shapes"], fx["param_seed"] + 1)
    B = fx["gen_in"].shape[0]
    prefix = fx["gen_in"][:, :, :1].reshape(B, D, R, 1).argmax(2).permute(0, 2, 1)
    T = fx["gen_in"].shape[-1]
    cls, logits = S.sample(prefix, None, sd, cfg, D, T, argmax=True)
    assert logits.shape == (B, T - 1, D, R)
    assert torch.equal(P.stack_one_hot(cls.permute(0, 2, 1), R), fx["gen_out"])


def test_inverse_cdf_rule_matches_a_direct_cumsum():
    g = torch.Generator().manual_seed(0)
    N, R = 400, 13
    lg = 3 * torch.randn(N, R, generator=g, dtype=torch.float64)
    lg[0] = torch.tensor([-1e4] * (R - 2) + [0., -1e4], dtype=torch.float64)     # one class of non-zero probability
    u = torch.rand(N, generator=g, dtype=torch.float64)
    u[1] = 1.0                                                                    # no running sum exceeds it
    got = S.inverse_cdf(lg, u)
    for n in range(N):
        p = [math.exp(v - max(lg[n].tolist())) for v in lg[n].tolist()]
        s = sum(p)
        cum, want, last = 0.0, None, 0
        for r in range(R):
            if p[r] / s > 0:
                last = r
            cum += p[r] / s
            if want is None and cum > u[n].item():
                want = r
        want = last if want is None else want
        if S.cdf_edge_distance(lg[n], u[n]).item() > 1e-12 or n < 2:
            assert got[n].item() == want, (n, got[n].item(), want)
    assert got[0].item() == R - 2 and got[1].item() == R - 1


def test_oracle_class_decode_matches_reference_modules(fx):
    R, D = fx["prior_cfg"]["resolution"], fx["D"]
    q = fx["quant_in"]                                   # [B, D, T] standard-normal latents
    cls = P.quantize(q, R).permute(0, 2, 1)              # [B, T, D]
    B, T, _ = cls.shape
    zero = torch.zeros(B, T, D)
    # QuantizedNormal.decode (dither off) then DiagonalShift.inverse; identity PCA, zero mean, no noise channels
    z = S.classes_to_latent(cls, zero, torch.zeros(B, 0, T - D + 1), torch.eye(D), torch.zeros(D), R)
    assert rel_l2(z, P.diagonal_shift_inverse(fx["quant_dec"])) < 1e-6
    assert torch.equal(P.diagonal_shift_inverse(q), fx["shift_inv"])
    # the PCA projection and the noise channels as pre_process_latent
    g = torch.Generator().manual_seed(1)
    L = 6
    pca = torch.linalg.qr(torch.randn(L, L, generator=g, dtype=torch.float64))[0]
    mean = torch.randn(L, generator=g, dtype=torch.float64)
    noise = torch.randn(B, L - D, T - D + 1, generator=g, dtype=torch.float64)
    dither = torch.rand(B, T, D, generator=g, dtype=torch.float64)
    z = S.classes_to_latent(cls, dither, noise, pca, mean, R)
    y = P.diagonal_shift_inverse(torch.clamp(torch.erfinv(2 * (cls + dither) / R - 1) * 2 ** 0.5, -4, 4).permute(0, 2, 1))
    want = torch.nn.functional.conv1d(torch.cat([y, noise], 1), pca.T.unsqueeze(-1)) + mean[:, None]
    assert rel_l2(z, want) < 1e-12

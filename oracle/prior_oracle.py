"""TEST INFRASTRUCTURE -- restatement of the latent prior (rave/prior/{core,residual_block,model}.py, VariationalPrior) in
plain torch on a {state_dict key: tensor} mapping.  Pinned against the unmodified reference by oracle/make_golden_prior.py
(tests/golden/prior_tiny.pt).  Device- and dtype-agnostic: scripts/time_prior.py runs it on the GPU as the reference's
arithmetic."""
import math

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle.spectral_oracle import seeded_params  # noqa: F401  (re-exported)

# configs/prior/prior_v1.gin
PRIOR_V1 = dict(resolution=32, res_size=512, skp_size=256, kernel_size=3, cycle_size=4, n_layers=10)


def dilations(cfg):
    return [2 ** (i % cfg["cycle_size"]) for i in range(cfg["n_layers"])]


def post_process_latent(z: Tensor, eps: Tensor, latent_mean: Tensor, latent_pca: Tensor, D: int) -> Tensor:
    """VariationalPrior.post_process_latent (rave/prior/model.py:206-211) with the noise of reparametrize injected."""
    mean, scale = z.chunk(2, 1)
    zs = eps * (F.softplus(scale) + 1e-4) + mean
    zs = zs - latent_mean.unsqueeze(-1)
    return F.conv1d(zs, latent_pca.unsqueeze(-1))[:, :D]


def diagonal_shift(x: Tensor) -> Tensor:
    """DiagonalShift.forward (rave/prior/core.py:54-77, groups = 1): dimension c advanced by D - 1 - c frames."""
    D, T = x.shape[1], x.shape[-1]
    Tp = T - D + 1
    return torch.cat([x[:, c:c + 1, D - 1 - c:D - 1 - c + Tp] for c in range(D)], 1)


def diagonal_shift_inverse(x: Tensor) -> Tensor:
    return diagonal_shift(x.flip(1)).flip(1)


def quantize(x: Tensor, R: int) -> Tensor:
    """QuantizedNormal.encode before the one-hot: class indices (long)."""
    u = .5 * (1 + torch.erf(x / math.sqrt(2)))
    return torch.clamp(torch.floor(u * R), 0, R - 1).long()


def dequantize(cls: Tensor, R: int, clamp: float = 4.0) -> Tensor:
    """QuantizedNormal.decode of a one-hot with dither off."""
    u = cls.to(torch.get_default_dtype()) / R
    return torch.clamp(torch.erfinv(2 * u - 1) * math.sqrt(2), -clamp, clamp)


def stack_one_hot(cls: Tensor, R: int) -> Tensor:
    """classes [B, D, T] -> the stacked one-hot [B, D·R, T] (channel d·R + r) of QuantizedNormal.to_stack_one_hot."""
    B, D, T = cls.shape
    return F.one_hot(cls, R).permute(0, 1, 3, 2).reshape(B, D * R, T).to(torch.get_default_dtype())


def latent_classes(z, eps, latent_mean, latent_pca, D, R) -> Tensor:
    """Classes [B, D, T - D + 1] of the training step (rave/prior/model.py:155-156)."""
    return quantize(diagonal_shift(post_process_latent(z, eps, latent_mean, latent_pca, D)), R)


def forward(x: Tensor, sd, cfg, D: int) -> Tensor:
    """Prior.forward (rave/prior/model.py:104-110) on a dense [B, R·D, T] input -> logits [B, R·D, T]."""
    K = cfg["kernel_size"]
    res = F.leaky_relu(F.conv1d(F.pad(x, (K - 1, 0)), sd["pre_net.0.weight"], sd["pre_net.0.bias"], groups=D), .2)
    skp = 0.
    for i, dil in enumerate(dilations(cfg)):
        p = f"residuals.{i}."
        h = F.conv1d(F.pad(res, ((K - 1) * dil, 0)), sd[p + "dconv.weight"], sd[p + "dconv.bias"], dilation=dil)
        a, b = h.chunk(2, 1)
        g = torch.sigmoid(a) * torch.tanh(b)
        res = res + F.conv1d(g, sd[p + "rconv.weight"], sd[p + "rconv.bias"])
        skp = skp + F.conv1d(g, sd[p + "sconv.weight"], sd[p + "sconv.bias"])
    y = F.leaky_relu(F.conv1d(skp, sd["post_net.0.weight"], sd["post_net.0.bias"]), .2)
    return F.conv1d(y, sd["post_net.2.weight"], sd["post_net.2.bias"], groups=D)


def loss(cls: Tensor, sd, cfg, D: int, taps=None) -> Tensor:
    """The cross-entropy of training_step (rave/prior/model.py:157-166) from classes [B, D, T']."""
    R = cfg["resolution"]
    pred = forward(stack_one_hot(cls, R), sd, cfg, D)
    if taps is not None:
        taps["logits"] = pred
    B, _, T = pred.shape
    logits = pred[..., :-1].reshape(B, D, R, T - 1).permute(0, 1, 3, 2)       # split_classes: channel d·R + r
    return F.cross_entropy(logits.reshape(-1, R), cls[..., 1:].reshape(-1))


def generate(x: Tensor, sd, cfg, D: int) -> Tensor:
    """Prior.generate(x, argmax=True) without cached convs: forward on the prefix at each step."""
    R = cfg["resolution"]
    x = x.clone()
    for i in range(x.shape[-1] - 1):
        pred = forward(x[..., :i + 1], sd, cfg, D)[..., -1:]
        cls = pred.reshape(x.shape[0], D, R, 1).argmax(2)
        x[..., i + 1:i + 2] = stack_one_hot(cls, R)
    return x


def model_ratio(n_band: int, ratios) -> int:
    """Samples per latent frame of a pqmf-input RAVE."""
    return n_band * math.prod(ratios)


def min_receptive_field(cfg, ratio: int) -> int:
    rf = (cfg["kernel_size"] - 1) * sum(dilations(cfg)) + 1
    return 2 ** math.ceil(math.log2(rf * ratio))

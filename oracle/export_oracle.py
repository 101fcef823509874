"""TEST INFRASTRUCTURE -- float64 restatement of the exported model's latent arithmetic (scripts/export.py:351-408, the
post / pre-processing of the four ScriptedRAVE subclasses; rave/blocks.py:933-963) and of its `channels` rules (export.py:
272-301).  Pinned against the unmodified reference by oracle/make_golden_export.py (tests/golden/export_latent.pt).
Device-agnostic: scripts/time_export.py runs it on the GPU, in float32, as the reference's arithmetic."""
import math

import numpy as np
import torch
import torch.nn.functional as F
from torch import Tensor


def latent_size(kind: str, fidelity: Tensor = None, f: float = .95, full: int = None, num_quantizers: int = None):
    """ScriptedRAVE.__init__ (export.py:119-137)."""
    if kind == "variational":
        size = max(int(np.argmax(fidelity.numpy() > f)), 1)
        return 2 ** math.ceil(math.log2(size))
    if kind == "discrete":
        return num_quantizers
    if kind == "wasserstein":
        return full
    if kind == "spherical":
        return full - 1
    raise ValueError(kind)


# ------------------------------------------------------------------ variational
def variational_post(z: Tensor, eps: Tensor, latent_mean: Tensor, latent_pca: Tensor, l: int) -> Tensor:
    mean, scale = z.chunk(2, 1)
    zs = eps * (F.softplus(scale) + 1e-4) + mean
    zs = zs - latent_mean.unsqueeze(-1)
    return torch.einsum("ic,bct->bit", latent_pca[:l], zs)


def variational_pre(z: Tensor, noise: Tensor, latent_mean: Tensor, latent_pca: Tensor) -> Tensor:
    y = torch.cat([z, noise], 1)
    return torch.einsum("jc,bjt->bct", latent_pca, y) + latent_mean.unsqueeze(-1)


# ------------------------------------------------------------------ discrete
def rvq_distances(r: Tensor, codebook: Tensor) -> Tensor:
    """|r|^2 - 2 r.c + |c|^2 of rows r [N, D] against codebook [K, D] -> [N, K]."""
    return r.pow(2).sum(1, keepdim=True) - 2 * r @ codebook.t() + codebook.pow(2).sum(1)[None]


def rvq_encode(x: Tensor, codebooks: Tensor, return_gaps: bool = False, residual_dtype=None):
    """ResidualVectorQuantization.encode: x [B, D, T], codebooks [Q, K, D] -> codes [B, Q, T] (long), lowest index on
    ties.  With return_gaps, also the gap between the best and second-best distance of every (b, q, t) [B, Q, T],
    relative to |r|^2 + max_k |c_k|^2, the scale of the rounding error of a distance in the expanded form.
    `residual_dtype` rounds each stage's residual to that type (the subtraction of a float32 run, which is exact in
    float64 before the rounding), so that only the distances are evaluated in x's precision."""
    B, D, T = x.shape
    r = x.permute(0, 2, 1).reshape(-1, D)
    codes, gaps = [], []
    for cb in codebooks:
        d2 = rvq_distances(r, cb)
        k = d2.argmin(1)
        if return_gaps:
            two = d2.topk(2, dim=1, largest=False).values
            scale = r.pow(2).sum(1) + cb.pow(2).sum(1).max()
            gaps.append(((two[:, 1] - two[:, 0]) / scale).reshape(B, T))
        r = r - cb[k]
        if residual_dtype is not None:
            r = r.to(residual_dtype).to(x.dtype)
        codes.append(k.reshape(B, T))
    codes = torch.stack(codes, 1)
    return (codes, torch.stack(gaps, 1)) if return_gaps else codes


def rvq_decode(codes: Tensor, codebooks: Tensor, noise: Tensor = None) -> Tensor:
    """DiscreteScriptedRAVE.pre_process_latent: clamp, truncate, sum the codebook rows, append the noise."""
    K = codebooks.shape[1]
    k = torch.clamp(codes, 0, K - 1).long()
    total = torch.zeros((), dtype=codebooks.dtype, device=codebooks.device)
    for q in range(codebooks.shape[0]):
        total = total + codebooks[q][k[:, q]].permute(0, 2, 1)
    return total if noise is None else torch.cat([total, noise], 1)


# ------------------------------------------------------------------ wasserstein
def wasserstein_pre(z: Tensor, noise: Tensor = None) -> Tensor:
    return z if noise is None else torch.cat([z, noise], 1)


# ------------------------------------------------------------------ spherical
def sphere_to_angles(x: Tensor) -> Tensor:
    """unit_norm_vector_to_angles: tail norms with the last two squares merged, arccos clamped to [-1, 1] (NaN kept),
    the last angle reflected when x[-1] < 0, mapped to [-1, 1)."""
    sq = x.flip(1).pow(2)
    sq[:, 1] += sq[:, 0]
    norms = sq[:, 1:].cumsum(1).flip(1).sqrt()
    angles = torch.arccos(torch.clamp(x[:, :-1] / norms, -1, 1))
    angles[:, -1] = torch.where(x[:, -1] >= 0, angles[:, -1], 2 * np.pi - angles[:, -1])
    angles[:, :-1] = angles[:, :-1] / np.pi
    angles[:, -1] = angles[:, -1] / (2 * np.pi)
    return 2 * (angles - .5)


def angles_to_sphere(angles: Tensor) -> Tensor:
    """angles_to_unit_norm_vector (floor modulo, as torch's %)."""
    a = (angles / 2 + .5) % 1
    a[:, :-1] = a[:, :-1] * np.pi
    a[:, -1] = a[:, -1] * (2 * np.pi)
    ones = torch.ones_like(a[:, :1])
    return torch.cat([a.cos(), ones], 1) * torch.cat([ones, a.sin().cumprod(1)], 1)


# ------------------------------------------------------------------ channels
def decode_rows(z: Tensor, n_channels: int, target_channels: int) -> Tensor:
    """The latent rows decode runs on: each example ceil(tc / nc) times when target_channels > n_channels (row b r + i
    is decode i of example b)."""
    if target_channels > n_channels:
        return z.repeat_interleave(math.ceil(target_channels / n_channels), 0)
    return z


def assemble_channels(y: Tensor, batch: int, n_channels: int, target_channels: int) -> Tensor:
    """Decoded rows [B r, nc, N] -> [B, target_channels, N]: the r decodes of an example stacked on the channel axis,
    then the first target_channels kept."""
    return y.reshape(batch, -1, y.shape[-1])[:, :target_channels]

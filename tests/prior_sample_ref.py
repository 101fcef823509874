"""TEST INFRASTRUCTURE -- float64 restatement of the prior's sampling (Prior.sample, csrc/prior_sample.cu) and of the
decode of its classes (Prior.decode_classes), built on oracle/prior_oracle.py's dense `forward`.  Device-agnostic."""
import math

import torch

from oracle import prior_oracle as P


def inverse_cdf(logits, u):
    """Class of each row of logits [..., R] at the uniform u [...]: the first r whose running softmax probability
    (max subtracted, classes in order) exceeds u, else the last r of non-zero probability."""
    p = torch.softmax(logits - logits.amax(-1, keepdim=True), -1)
    cum = p.cumsum(-1)
    over = cum > u.unsqueeze(-1)
    R = logits.shape[-1]
    first = over.to(torch.int8).argmax(-1)
    last_nz = (R - 1) - (p > 0).flip(-1).to(torch.int8).argmax(-1)
    return torch.where(over.any(-1), first, last_nz)


def cdf_edge_distance(logits, u):
    """Distance of u [...] to the nearest edge of the float64 CDF of softmax(logits [..., R])."""
    cum = torch.softmax(logits - logits.amax(-1, keepdim=True), -1).cumsum(-1)
    return (cum - u.unsqueeze(-1)).abs().amin(-1)


def _pick(lg, u, argmax):
    return lg.argmax(-1) if argmax else inverse_cdf(lg, u)


def teacher_logits(cls, sd, cfg, D):
    """Logits [B, T - 1, D, R] of every step given the whole class sequence cls [B, T, D] (one dense forward)."""
    R = cfg["resolution"]
    B, T, _ = cls.shape
    x = P.stack_one_hot(cls.permute(0, 2, 1).long(), R).to(sd["pre_net.0.weight"].dtype)
    pred = P.forward(x, sd, cfg, D)
    return pred[..., :-1].reshape(B, D, R, T - 1).permute(0, 3, 1, 2)


def sample(prefix, u, sd, cfg, D, n_frames, argmax=False):
    """Prior.sample: classes [B, n_frames, D] (long) continuing prefix [B, P, D] at the uniforms u [B, n_frames, D], and
    the logits [B, n_frames - 1, D, R] of every step; the dense forward over the whole prefix per step."""
    R = cfg["resolution"]
    B, Pn, _ = prefix.shape
    cls = torch.zeros(B, n_frames, D, dtype=torch.long, device=prefix.device)
    cls[:, :Pn] = prefix.long()
    logits = []
    for i in range(n_frames - 1):
        x = P.stack_one_hot(cls[:, :i + 1].permute(0, 2, 1), R).to(sd["pre_net.0.weight"].dtype)
        pred = P.forward(x, sd, cfg, D)[..., -1]
        lg = pred.reshape(B, D, R)
        logits.append(lg)
        if i + 1 >= Pn:
            cls[:, i + 1] = _pick(lg, u[:, i + 1] if u is not None else None, argmax)
    return cls, torch.stack(logits, 1) if logits else None


def classes_to_latent(cls, dither, noise, latent_pca, latent_mean, R):
    """pre_process_latent ∘ DiagonalShift.inverse ∘ QuantizedNormal.decode of classes [B, T, D] with the dither
    [B, T, D] and the noise [B, L - D, T - D + 1] given -> z [B, L, T - D + 1]."""
    x = cls.to(dither.dtype) / R + dither / R
    y = torch.clamp(torch.erfinv(2 * x - 1) * math.sqrt(2), -4, 4).permute(0, 2, 1)
    y = P.diagonal_shift_inverse(y)
    z = torch.cat([y, noise], 1)
    return torch.einsum("cl,bct->blt", latent_pca.to(z.dtype), z) + latent_mean.to(z.dtype)[:, None]

"""Restatement of the reference's EMA callback (scripts/train.py:81-119) in float32 torch ops on the CPU, and the seeded
parameter snapshots of the EMA fixture (tests/golden/ema.pt, written by oracle/make_golden_ema.py).

update: the first call for a name clones the parameter; later calls compute `w * factor + p * (1 - factor)` on float32
tensors, i.e. rn(rn(w * f) + rn(p * g)) with f = float32(factor), g = float32(1 - factor), 1 - factor in double."""
import hashlib
from typing import Dict, List, Sequence, Tuple

import torch

FACTORS = (.999, .9, .5)
N_CALLS = 4
SNAPSHOT_SEED = 2024


def update(weights: Dict[str, torch.Tensor], named_params: Sequence[Tuple[str, torch.Tensor]], factor: float) -> None:
    for n, p in named_params:
        if n not in weights:
            weights[n] = p.detach().clone()
            continue
        weights[n] = weights[n] * factor + p.detach() * (1 - factor)


def swap(weights: Dict[str, torch.Tensor], named_params: Sequence[Tuple[str, torch.Tensor]]) -> None:
    with torch.no_grad():
        for n, p in named_params:
            current = p.detach().clone()
            p.copy_(weights[n])
            weights[n] = current


def snapshots(shapes: Sequence[Tuple[int, ...]], n: int = N_CALLS, seed: int = SNAPSHOT_SEED) -> List[List[torch.Tensor]]:
    """n + 1 parameter snapshots: a N(0, .1) start, then n seeded steps of N(0, 1e-3) per element, like optimiser steps
    of a model that is training.  Float32 on the CPU; the same on every machine with the same torch."""
    g = torch.Generator().manual_seed(seed)
    cur = [torch.randn(s, generator=g) * .1 for s in shapes]
    out = [[t.clone() for t in cur]]
    for _ in range(n):
        cur = [t + torch.randn(t.shape, generator=g) * 1e-3 for t in cur]
        out.append([t.clone() for t in cur])
    return out


def digest(tensors: Sequence[torch.Tensor]) -> str:
    """sha256 of the float32 bytes of the tensors, in order: a bit-exact fingerprint."""
    h = hashlib.sha256()
    for t in tensors:
        h.update(t.detach().to(torch.float32).contiguous().cpu().numpy().tobytes())
    return h.hexdigest()

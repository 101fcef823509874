"""TEST INFRASTRUCTURE -- generates the EMA fixture by EXECUTING THE REFERENCE'S OWN `EMA` class: scripts/train.py is
parsed and only its `class EMA` definition is executed, with a stub `pl.Callback` (the script's flags, imports and main
never run).  Writes a new file only:

    python -m oracle.make_golden_ema

  tests/golden/ema.pt   the parameter names and shapes of a tiny v2 RAVE (capacity 4, discriminator capacity 2: 226
                        tensors, 157016 values); per factor in ema_oracle.FACTORS, the sha256 of the averages after each
                        of N_CALLS + 1 `on_train_batch_end` calls (the first clones), then of the parameters and of the
                        averages after `swap_weights` and after the swap back; the full averages after the last call for
                        factor .999; and the fraction of elements whose fused (FMA) evaluation would round differently.
                        The parameter snapshots are regenerated from their seed by ema_oracle.snapshots.

The oracle (oracle/ema_oracle.py) must reproduce every digest; the script checks it.
"""
import ast
import os
import types

import numpy as np
import torch
import torch.nn as nn

from oracle import ema_oracle as E
from oracle.make_golden import GOLDEN
from oracle.ref_loader import REFERENCE_ROOT


def reference_ema_class():
    """`class EMA` of the reference's scripts/train.py, executed alone over a stub `pl.Callback`."""
    path = os.path.join(REFERENCE_ROOT, "scripts", "train.py")
    tree = ast.parse(open(path).read(), path)
    cls = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "EMA"]
    assert len(cls) == 1
    from typing import Any, Dict
    pl = types.SimpleNamespace(Callback=type("Callback", (), {}))
    ns = {"pl": pl, "torch": torch, "Any": Any, "Dict": Dict}
    exec(compile(ast.Module(body=cls, type_ignores=[]), path, "exec"), ns)
    return ns["EMA"]


def tiny_v2_shapes():
    from rave_b200 import configs
    m = configs.build_rave("v2", capacity=4, disc_capacity=2)
    return [(n, tuple(p.shape)) for n, p in m.named_parameters()]


class Holder(nn.Module):
    """A module whose named_parameters() yields the given (dotted) names in the given order."""

    def __init__(self, names_shapes):
        super().__init__()
        self._order = [n for n, _ in names_shapes]
        self.flat = nn.ParameterDict({n.replace(".", "__"): nn.Parameter(torch.zeros(s)) for n, s in names_shapes})

    def named_parameters(self, *a, **k):
        for n in self._order:
            yield n, self.flat[n.replace(".", "__")]

    def set(self, values):
        with torch.no_grad():
            for (_, p), v in zip(self.named_parameters(), values):
                p.copy_(v)


def fma_fraction(w, p, factor):
    """Fraction of elements where ema * f + rn(p * g) rounded once (what an FMA computes) differs from the
    reference's two roundings."""
    f, g = np.float32(factor), np.float32(1 - factor)
    w, p = w.numpy(), p.numpy()
    two = (w * f) + (p * g)
    fused = (w.astype(np.float64) * np.float64(f) + (p * g).astype(np.float64)).astype(np.float32)
    return float((two != fused).mean())


def run(EMA, names_shapes, factor):
    snaps = E.snapshots([s for _, s in names_shapes])
    mod = Holder(names_shapes)
    ema = EMA(factor)
    digests = []
    for k in range(len(snaps)):
        mod.set(snaps[k])
        ema.on_train_batch_end(None, mod, None, None, k)
        digests.append(E.digest(ema.state_dict()[n] for n, _ in names_shapes))
    last = {n: ema.state_dict()[n].clone() for n, _ in names_shapes}
    before = [p.detach().clone() for _, p in mod.named_parameters()]
    frac = fma_fraction(torch.cat([last[n].flatten() for n, _ in names_shapes]),
                        torch.cat([t.flatten() for t in before]), factor)
    ema.swap_weights(mod)
    swapped = (E.digest(p for _, p in mod.named_parameters()), E.digest(ema.state_dict()[n] for n, _ in names_shapes))
    ema.swap_weights(mod)
    back = (E.digest(p for _, p in mod.named_parameters()), E.digest(ema.state_dict()[n] for n, _ in names_shapes))
    assert back == (E.digest(before), digests[-1])
    return {"digests": digests, "swapped": swapped, "swapped_back": back, "fma_fraction": frac}, last


def oracle_digests(names_shapes, factor):
    snaps = E.snapshots([s for _, s in names_shapes])
    w = {}
    out = []
    for k in range(len(snaps)):
        E.update(w, list(zip([n for n, _ in names_shapes], snaps[k])), factor)
        out.append(E.digest(w[n] for n, _ in names_shapes))
    return out


def main():
    EMA = reference_ema_class()
    names_shapes = tiny_v2_shapes()
    cases = {}
    full = None
    for factor in E.FACTORS:
        rec, last = run(EMA, names_shapes, factor)
        assert oracle_digests(names_shapes, factor) == rec["digests"], factor
        # with factor .5 both products are exact (powers of two), so only the other factors separate FMA from two roundings
        assert factor == .5 or rec["fma_fraction"] > .05, rec["fma_fraction"]
        cases[factor] = rec
        if factor == .999:
            full = last
        print(f"factor {factor}: {len(rec['digests'])} calls, FMA would change {rec['fma_fraction']:.1%} of the "
              f"elements of the last update")
    out = os.path.join(GOLDEN, "ema.pt")
    torch.save({"names_shapes": names_shapes, "seed": E.SNAPSHOT_SEED, "n_calls": E.N_CALLS, "cases": cases,
                "last_999": full}, out)
    print("wrote", out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()

"""TEST INFRASTRUCTURE -- generates the fixtures of the validation pass by EXECUTING THE UNMODIFIED REFERENCE
(`RAVE.validation_step` / `RAVE.validation_epoch_end`, rave/model.py:426-495, and `core.get_rave_receptive_field`,
rave/core.py:180-217) under the stubs of oracle/ref_loader.py, and asserts that oracle/validation_oracle.py reproduces the
latent PCA.  Writes new files only:

    python -m oracle.make_golden_validation

  tests/golden/validation_v2_tiny.pt    v2 at capacity 8, latent 16, in eval mode, encoder / decoder parameters from
                                        spectral_oracle.seeded_params (the fixture keeps their shapes and the seed):
                                        per batch the seeds of the input (spectral_oracle.step_batch) and of the
                                        reparametrisation noise the reference drew (global RNG re-seeded before the
                                        call; randn_like is the first draw: spectral_oracle.step_eps), the logged
                                        `validation` and the posterior mean; then the epoch end's buffers
                                        (latent_mean, latent_pca, fidelity), logged fidelities and probed receptive
                                        field; the full-size probes of v2 and v2_small; the sklearn version
  tests/golden/validation_hybrid_tiny.pt  the probe of v2 + hybrid (mel input, GRU head) at capacity 4, latent 16, from
                                        seeded encoder / decoder parameters

Inputs and parameters are regenerated from their seeds, so the fixtures hold only what the reference computed.

The stub trainer provides `state.stage` (validation, not the sanity check) and a no-op `logger.experiment.add_audio`;
`log` is captured.
"""
import os
import sys
import types
from functools import partial

import numpy as np
import torch
import torch.nn as nn

from oracle import rave_oracle as O
from oracle import validation_oracle as V
from oracle.make_golden import GOLDEN, build_ref_rave
from oracle.make_golden_hybrid import build_ref_rave_hybrid
from oracle.ref_loader import load_reference, set_padding_mode
from oracle.spectral_oracle import seeded_params, step_batch, step_eps


def _stub_lightning(m, logs):
    m.trainer = types.SimpleNamespace(state=types.SimpleNamespace(stage="validate"))
    m.logger = types.SimpleNamespace(experiment=types.SimpleNamespace(add_audio=lambda *a, **k: None))
    m.log = lambda k, v, *a, **kw: logs.__setitem__(k, torch.as_tensor(np.asarray(v)).detach().clone().float())


def build_ref_v2_small(R, disc_capacity=4):
    """rave.RAVE of configs/v2_small.gin at full size (capacity 48, ratios 4 2 2 2, NoiseGeneratorV2)."""
    blocks = R.blocks
    orig = blocks.GeneratorV2
    noise = partial(blocks.NoiseGeneratorV2, hidden_size=64, data_size=16, ratios=[2, 2, 2], noise_bands=32)
    blocks.GeneratorV2 = partial(orig, noise_module=noise)
    try:
        return build_ref_rave(R, O.ArchConfig(capacity=48, ratios=(4, 2, 2, 2)), disc_capacity=disc_capacity)
    finally:
        blocks.GeneratorV2 = orig


def _seed_autoencoder(m, seed):
    shapes = [(k, tuple(v.shape)) for k, v in m.named_parameters() if k.startswith(("encoder.", "decoder."))]
    m.load_state_dict(seeded_params(shapes, seed), strict=False)
    return shapes


def golden_validation_v2(R, n_batches=6, B=2, T=32768, full_size=True, param_seed=71):
    print("RAVE.validation_step / validation_epoch_end v2 (tiny)")
    set_padding_mode("centered")
    cfg = O.ArchConfig(capacity=8, latent_size=16)
    torch.manual_seed(0)
    m = build_ref_rave(R, cfg)
    shapes = _seed_autoencoder(m, param_seed)
    logs = {}
    _stub_lightning(m, logs)
    m.eval()
    batches = []
    out = []
    for i in range(n_batches):
        x = step_batch(B, T, 400 + i)
        torch.manual_seed(1000 + i)
        assert torch.equal(torch.randn(B, cfg.latent_size, T // 2048), step_eps(B, cfg.latent_size, T // 2048, 1000 + i))
        torch.manual_seed(1000 + i)
        logs.clear()
        with torch.no_grad():
            o = m.validation_step(x, i)
        out.append(o)
        batches.append(dict(x_seed=400 + i, eps_seed=1000 + i, validation=logs["validation"].clone(),
                            mean=o[1].detach().clone()))
        print(f"  batch {i}: validation {float(logs['validation']):.6f}")
    logs.clear()
    m.validation_epoch_end(out)
    rf = tuple(int(v) for v in m.receptive_field)
    print(f"  receptive field {rf}, fidelity {m.fidelity.tolist()}")
    mean, comps, ev, fid = V.latent_analysis([b["mean"] for b in batches])
    assert np.abs(fid - m.fidelity.double().numpy()).max() <= 1e-5, np.abs(fid - m.fidelity.double().numpy()).max()
    for i in V.separated(ev):
        c = float(np.dot(comps[i], m.latent_pca[i].double().numpy()))
        assert c >= 0.9999, (i, c)
    assert np.abs(mean - m.latent_mean.double().numpy()).max() <= 1e-5
    assert V.fidelity_logs(fid) == {k: float(v) for k, v in logs.items() if k.startswith("fidelity_")}
    import sklearn
    fx = dict(cfg=vars(cfg), disc_capacity=4, B=B, T=T, param_shapes=shapes, param_seed=param_seed, batches=batches,
              receptive_field=rf,
              latent_mean=m.latent_mean.clone(), latent_pca=m.latent_pca.clone(), fidelity=m.fidelity.clone(),
              fidelity_logs={k: v.clone() for k, v in logs.items() if k.startswith("fidelity_")},
              sklearn_version=sklearn.__version__)
    if full_size:
        fx["full_size_receptive_field"] = {}
        for name, build in (("v2", lambda: build_ref_rave(R, O.ArchConfig(), disc_capacity=4)),
                            ("v2_small", lambda: build_ref_v2_small(R))):
            torch.manual_seed(0)
            mf = build()
            fx["full_size_receptive_field"][name] = tuple(int(v) for v in R.core.get_rave_receptive_field(mf))
            print(f"  full-size {name}: receptive field {fx['full_size_receptive_field'][name]}")
    torch.save(fx, os.path.join(GOLDEN, "validation_v2_tiny.pt"))


def golden_probe_hybrid(R, param_seed=72):
    print("receptive-field probe v2 + hybrid (tiny)")
    set_padding_mode("centered")
    cfg = O.ArchConfig(capacity=4, latent_size=16)
    torch.manual_seed(0)
    m = build_ref_rave_hybrid(R, cfg)
    shapes = _seed_autoencoder(m, param_seed)
    rf = tuple(int(v) for v in R.core.get_rave_receptive_field(m))
    assert all(getattr(mod, "enabled", True) for mod in m.modules() if hasattr(mod, "gru_state"))
    print(f"  receptive field {rf}")
    torch.save(dict(cfg=vars(cfg), disc_capacity=4, param_shapes=shapes, param_seed=param_seed, receptive_field=rf),
               os.path.join(GOLDEN, "validation_hybrid_tiny.pt"))


def main():
    os.makedirs(GOLDEN, exist_ok=True)
    R = load_reference()
    norm = R.blocks.normalization
    R.blocks.normalization = lambda m, mode="weight_norm": norm(m, mode)  # configs/v1.gin:41
    golden_validation_v2(R, full_size="--no-full-size" not in sys.argv)
    golden_probe_hybrid(R)
    for f in ("validation_v2_tiny.pt", "validation_hybrid_tiny.pt"):
        print(f, os.path.getsize(os.path.join(GOLDEN, f)), "bytes")


if __name__ == "__main__":
    sys.exit(main())

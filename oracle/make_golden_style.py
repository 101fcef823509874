"""TEST INFRASTRUCTURE -- generates the style-transfer fixture by EXECUTING THE UNMODIFIED REFERENCE: the v3 encoder and
generator (rave/blocks.py:514-714) with their AdaptiveInstanceNormalization layers (rave/blocks.py:863-926) in eval mode,
under the stubs of oracle/ref_loader.py, and asserts that oracle/style_oracle.py reproduces it.  Writes a new file only:

    python -m oracle.make_golden_style

  tests/golden/style_v3_tiny.pt   v3 at capacity 16, latent 16, ratios [4, 4, 4, 2], B = 2, T = 16384; parameters from
                                  style_oracle.style_params (the fixture keeps the seed).  Inputs, regenerated from
                                  their seeds by style_oracle.fixture_inputs: the PQMF analysis of two target and one
                                  source audio batch, and a latent of two frames for each.  The sequence
                                  style_oracle.STYLE_SEQUENCE: reset and learn the target over both target batches,
                                  learn the source, transfer, reset the target.  Stored after each step: the encoder
                                  output, the decoder output on the latent of the step's batch, and every AdaIN buffer
                                  (rows [:B] of the statistics, the counters and the flags) packed into one tensor.

`ScriptedRAVE` (scripts/export.py) needs nn_tilde, which is not installable here, so the learn / reset flags are written
exactly as its `update_adain` writes them (scripts/export.py:213-230): both learn flags zeroed, then `learn_y.add_(1)` /
`learn_x.add_(1)`, then `reset_y()` / `reset_x()`.
"""
import os

import torch

from oracle import style_oracle as S
from oracle.make_golden import GOLDEN, build_ref_autoencoder, check
from oracle.ref_loader import load_reference, set_padding_mode

B, T, PARAM_SEED = 2, 16384, 91


def ref_update_adain(R, modules, learn_target=False, learn_source=False, reset_target=False, reset_source=False):
    """scripts/export.py:213-230, statement for statement, on the reference's modules."""
    for m in modules:
        if isinstance(m, R.blocks.AdaptiveInstanceNormalization):
            m.learn_x.zero_()
            m.learn_y.zero_()
            if learn_target:
                m.learn_y.add_(1)
            if learn_source:
                m.learn_x.add_(1)
            if reset_target:
                m.reset_y()
            if reset_source:
                m.reset_x()


def main():
    R = load_reference()
    set_padding_mode("centered")
    cfg = S.style_cfg()
    torch.manual_seed(0)
    pq = R.pqmf.CachedPQMF(attenuation=100, n_band=16)
    norm = R.blocks.normalization
    R.blocks.normalization = lambda m, mode="weight_norm": norm(m, mode)          # configs/v1.gin:41
    try:
        enc, dec = build_ref_autoencoder(R, cfg)
    finally:
        R.blocks.normalization = norm
    holder = torch.nn.Module()
    holder.encoder, holder.decoder = enc, dec
    shapes = [(k, tuple(v.shape)) for k, v in holder.named_parameters()]
    assert all(not k.endswith(".weight") or "conv" in k for k, _ in shapes), "weight norm is not bound"
    holder.load_state_dict(S.style_params(shapes, PARAM_SEED), strict=False)
    holder.eval()
    sd0 = {k: v.detach().clone() for k, v in holder.state_dict().items()}
    for k, v in S.snapshot(sd0, B).items():         # the sequence starts from the buffers as constructed
        assert torch.equal(v, torch.ones_like(v) if k.rsplit(".", 1)[-1].startswith("std") else torch.zeros_like(v)), k
    with torch.no_grad():
        inputs, latents = S.fixture_inputs(B, T, cfg.latent_size)
        for k, (seed, gain) in S.AUDIO.items():
            check(f"PQMF input {k}", inputs[k], R.model._pqmf_encode(pq, S.audio_batch(B, T, seed, gain)), 1e-6)
        steps = []
        mods = list(holder.modules())
        for kw, which in S.STYLE_SEQUENCE:
            ref_update_adain(R, mods, **kw)
            e = enc.encoder(inputs[which])
            y = dec(latents[which])
            layout, bufs = S.pack(S.snapshot(holder.state_dict(), B))
            steps.append(dict(update_adain=kw, input=which, encoder=e.clone(), decoder=y.clone(), buffers=bufs))
    n_adain = sum(isinstance(m, R.blocks.AdaptiveInstanceNormalization) for m in mods)
    print(f"style transfer v3 (tiny): {n_adain} AdaIN layers, {len(steps)} steps")
    for i, ((e, y, bufs), st) in enumerate(zip(S.run_sequence(sd0, inputs, latents, cfg), steps)):
        check(f"step {i} encoder", e, st["encoder"], 1e-4)
        check(f"step {i} decoder", y, st["decoder"], 1e-4)
        for k, v in S.unpack(st["buffers"], layout).items():
            check(f"step {i} {k}", bufs[k], v, 1e-4)
    out = dict(B=B, T=T, param_seed=PARAM_SEED, capacity=cfg.capacity, latent_size=cfg.latent_size,
               ratios=list(cfg.ratios), buffer_layout=layout, steps=steps)
    torch.save(out, os.path.join(GOLDEN, "style_v3_tiny.pt"))


if __name__ == "__main__":
    main()

"""TEST INFRASTRUCTURE -- generates the fixtures of the multi-scale spectral discriminator by EXECUTING THE UNMODIFIED
REFERENCE (configs/spectral_discriminator.gin on top of configs/v2.gin), and asserts that oracle/spectral_oracle.py
reproduces them.  Writes new files only:

    python -m oracle.make_golden_spectral

  tests/golden/discriminator_spectral.pt        tiny MultiScaleSpectralDiscriminator: sampled features, loss terms,
                                                grad_x, parameter gradients
  tests/golden/training_step_v2_spectral_tiny.pt the reference's own RAVE.training_step, a phase-2 D-step and a phase-2
                                                G-step from the same seeded parameters: logged losses, sampled gradients
  tests/golden/state_dict_keys_spectral.pt      keys / shapes / dtypes of the full-size rave.RAVE of this configuration
"""
import os
import sys
from functools import partial

import torch
import torch.nn as nn

from oracle import rave_oracle as O
from oracle import spectral_oracle as S
from oracle.make_golden import GOLDEN, check, make_input
from oracle.ref_loader import load_reference, set_padding_mode

FEATURE_SAMPLE = 512
GRAD_SAMPLE = 8192


def _spectral_disc(R, capacity):
    return partial(R.discriminator.MultiScaleSpectralDiscriminator, scales=list(S.SCALES),
                   convnet=partial(R.discriminator.EncodecConvNet, capacity=capacity))


def golden_discriminator_spectral(R, capacity=2, B=1, T=8192):
    """MultiScaleSpectralDiscriminator(EncodecConvNet) at a tiny capacity: features (seeded samples), the training step's
    feature-matching / hinge terms on them, and the gradients of their sum."""
    print("spectral discriminator (MultiScaleSpectralDiscriminator + EncodecConvNet)")
    torch.manual_seed(6)
    D = R.discriminator
    norm = R.blocks.normalization
    D.normalization = lambda m, mode="weight_norm": norm(m, mode)      # configs/v1.gin:41
    try:
        disc = _spectral_disc(R, capacity)(n_channels=1)
    finally:
        D.normalization = norm
    x = make_input(2 * B, 1, T + 3, seed=12)    # +3: frames do not tile the signal
    sd = {"discriminator." + k: v.detach().clone() for k, v in disc.state_dict().items()}
    xg = x.clone().requires_grad_(True)
    feats = disc(xg)
    feats_o = S.multi_scale_spectral_discriminator(x, sd, "discriminator.")
    assert len(feats) == len(feats_o) == len(S.SCALES)
    for i, (fa, fb) in enumerate(zip(feats_o, feats)):
        for j, (a, b) in enumerate(zip(fa, fb)):
            assert a.shape == b.shape
            check(f"disc {i}.{j} {tuple(b.shape)}", a, b, 1e-6)
    real = [[f[:B] for f in s] for s in feats]
    fake = [[f[B:] for f in s] for s in feats]
    fm_r, ld_r, la_r = 0., 0., 0.
    for sr, sf in zip(real, fake):              # rave/model.py:348-379
        fm_r = fm_r + sum(map(partial(R.core.mean_difference, norm="L1", relative=True),
                              sr[1:], sf[1:])) / len(sr[1:])
        d_, a_ = R.core.hinge_gan(sr[-1], sf[-1])
        ld_r, la_r = ld_r + d_, la_r + a_
    fm_r = fm_r / len(real)
    fm, ld, la = O.gan_losses(feats_o, 1, True)
    check("feature matching", fm, fm_r, 1e-6)
    check("loss_dis", ld, ld_r, 1e-6)
    check("loss_adv", la, la_r, 1e-6)
    pp = dict(disc.named_parameters())
    pn = sorted(pp)
    grads = torch.autograd.grad(fm_r + ld_r + la_r, [xg] + [pp[n] for n in pn])
    params = {k: v for k, v in sd.items() if not k.endswith(".window")}     # the hann windows are rebuilt by the module
    fx = dict(capacity=capacity, scales=list(S.SCALES), params=params, x=x,
              features=[[S.sample(f.detach(), FEATURE_SAMPLE, seed=10 * i + j) for j, f in enumerate(s)]
                        for i, s in enumerate(feats)],
              fm=fm_r.detach(), loss_dis=ld_r.detach(), loss_adv=la_r.detach(),
              grad_x=grads[0].detach(),
              grad_params={"discriminator." + n: g.detach() for n, g in zip(pn, grads[1:])})
    torch.save(fx, os.path.join(GOLDEN, "discriminator_spectral.pt"))


def build_ref_rave_spectral(R, cfg: O.ArchConfig, disc_capacity=4, spectral_capacity=32, update_discriminator_every=2,
                            phase_1_duration=1000):
    """The reference's rave.RAVE bound like configs/v2.gin (53-89) + configs/spectral_discriminator.gin (6-17)."""
    D, blocks, core = R.discriminator, R.blocks, R.core
    norm = blocks.normalization
    D.normalization = lambda m, mode="weight_norm": norm(m, mode)
    act = lambda dim: nn.LeakyReLU(.2)
    scales_net = partial(D.ConvNet, out_size=1, capacity=disc_capacity, n_layers=4, stride=4, conv=nn.Conv1d,
                         kernel_size=15)
    disc = partial(D.CombineDiscriminators, [partial(D.MultiScaleDiscriminator, n_discriminators=3, convnet=scales_net),
                                             _spectral_disc(R, spectral_capacity)])
    enc = partial(blocks.VariationalEncoder,
                  partial(blocks.EncoderV2, data_size=cfg.n_band, capacity=cfg.capacity, ratios=cfg.ratios,
                          latent_size=cfg.latent_size, n_out=2, kernel_size=cfg.kernel_size, dilations=cfg.dilations,
                          activation=act, adain=None))
    dec = partial(blocks.GeneratorV2, data_size=cfg.n_band, capacity=cfg.capacity, ratios=cfg.ratios,
                  latent_size=cfg.latent_size, kernel_size=cfg.kernel_size, dilations=cfg.dilations,
                  amplitude_modulation=True, activation=act, adain=None)
    stft = partial(core.MultiScaleSTFT, scales=[2048, 1024, 512, 256, 128], sample_rate=48000, magnitude=True)
    dist = partial(core.AudioDistanceV1, multiscale_stft=stft, log_epsilon=1e-7)
    try:
        m = R.model.RAVE(latent_size=cfg.latent_size, sampling_rate=48000, encoder=enc, decoder=dec,
                         discriminator=disc, phase_1_duration=phase_1_duration, gan_loss=core.hinge_gan,
                         valid_signal_crop=True,
                         feature_matching_fun=partial(core.mean_difference, norm="L1", relative=True),
                         num_skipped_features=1, audio_distance=dist, multiband_audio_distance=dist,
                         weights={"feature_matching": 20},
                         pqmf=partial(R.pqmf.CachedPQMF, attenuation=100, n_band=cfg.n_band),
                         update_discriminator_every=update_discriminator_every, n_channels=1)
    finally:
        D.normalization = norm
    return m


def golden_training_step_spectral(R, B=2, T=32768, param_seed=31, disc_capacity=4, spectral_capacity=4):
    """The reference's OWN RAVE.training_step (rave/model.py:288-424) in phase 2: a D-step (batch_idx 0) and a G-step
    (batch_idx 1), each from the same seeded parameters.  Commits the logged scalars and a seeded sample of the gradients
    the step's optimiser consumed (discriminator.* after the D-step, decoder.* after the G-step)."""
    print("RAVE.training_step v2 + spectral discriminator (phase-2 D, phase-2 G)")
    set_padding_mode("centered")
    cfg = O.ArchConfig(capacity=8, latent_size=16)
    torch.manual_seed(0)
    m = build_ref_rave_spectral(R, cfg, disc_capacity, spectral_capacity)
    # the PQMF's conv weights are parameters of the reference's module, but fixed by the filter design (rave/pqmf.py)
    shapes = [(k, tuple(v.shape)) for k, v in m.named_parameters() if not k.startswith("pqmf.")]
    m.load_state_dict(S.seeded_params(shapes, param_seed), strict=False)
    m.train()
    m.warmed_up = True
    rf = (1024, 512)
    m.receptive_field[0], m.receptive_field[1] = rf                 # what validation_epoch_end would have measured
    opts = m.configure_optimizers()
    gen_opt, dis_opt = opts[0]["optimizer"], opts[1]["optimizer"]
    logs = {}
    m.optimizers = lambda: (gen_opt, dis_opt)
    m.log = lambda k, v: logs.__setitem__(k, v.detach().clone() if torch.is_tensor(v) else torch.tensor(float(v)))
    m.log_dict = lambda d: [m.log(k, v) for k, v in d.items()]
    sd0 = {k: v.detach().clone() for k, v in m.state_dict().items()}
    Lz = T // cfg.n_band
    for r in cfg.ratios:
        Lz //= r
    steps = []
    for name, batch_idx, seed in (("phase2_dis", 0, 101), ("phase2_gen", 1, 102)):
        m.load_state_dict(sd0)
        x = S.step_batch(B, T, seed)
        assert torch.equal(x, make_input(B, 1, T, seed=500 + seed))
        torch.manual_seed(seed)
        eps = torch.randn(B, cfg.latent_size, Lz)
        assert torch.equal(eps, S.step_eps(B, cfg.latent_size, Lz, seed))
        torch.manual_seed(seed)
        logs.clear()
        m.training_step(x.clone(), batch_idx)
        dis = batch_idx % m.update_discriminator_every == 0
        grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()
                 if p.grad is not None and k.startswith("discriminator.") == dis
                 and not k.startswith(("encoder.", "pqmf."))}
        keys = sorted(grads)
        steps.append(dict(name=name, batch_idx=batch_idx, seed=seed, logs={k: v.clone() for k, v in logs.items()},
                          grad_keys=keys, grad_sample=S.sample(torch.cat([grads[k].reshape(-1) for k in keys]),
                                                               GRAD_SAMPLE, seed=seed)))
        print("  ", name, {k: round(float(v), 6) for k, v in logs.items()})
        losses, ldis = S.train_step_losses(x, sd0, cfg, eps, receptive_field=rf)
        for k, v in losses.items():
            check(f"{name} {k}", v, logs[k], 2e-6)
        check(f"{name} loss_dis", ldis, logs["loss_dis"], 2e-6)
    torch.save(dict(cfg=vars(cfg), B=B, T=T, disc_capacity=disc_capacity, spectral_capacity=spectral_capacity,
                    update_discriminator_every=m.update_discriminator_every, receptive_field=rf,
                    param_shapes=shapes, param_seed=param_seed, hk=sd0["pqmf.hk"], steps=steps),
               os.path.join(GOLDEN, "training_step_v2_spectral_tiny.pt"))


def golden_state_dict_keys_spectral(R):
    """Key list of the full-size rave.RAVE of `--config v2 --config spectral_discriminator`."""
    print("state_dict key contract (v2 + spectral discriminator, full size)")
    torch.manual_seed(0)
    m = build_ref_rave_spectral(R, O.ArchConfig(), disc_capacity=96)
    out = {"rave_v2_spectral": {k: (tuple(v.shape), str(v.dtype)) for k, v in m.state_dict().items()}}
    print(f"  rave_v2_spectral: {len(out['rave_v2_spectral'])} keys")
    torch.save(out, os.path.join(GOLDEN, "state_dict_keys_spectral.pt"))


def main():
    os.makedirs(GOLDEN, exist_ok=True)
    R = load_reference()
    norm = R.blocks.normalization
    R.blocks.normalization = lambda m, mode="weight_norm": norm(m, mode)  # configs/v1.gin:41
    golden_discriminator_spectral(R)
    golden_training_step_spectral(R)
    golden_state_dict_keys_spectral(R)
    for f in ("discriminator_spectral.pt", "training_step_v2_spectral_tiny.pt", "state_dict_keys_spectral.pt"):
        print(f, os.path.getsize(os.path.join(GOLDEN, f)), "bytes")


if __name__ == "__main__":
    sys.exit(main())

"""TEST INFRASTRUCTURE -- generates the fixtures of the v2_nopqmf configuration (rave/configs/v2_nopqmf.gin on top of
v1.gin: raw-waveform generator, PQMF-input encoder) by EXECUTING THE UNMODIFIED REFERENCE, and asserts that
oracle/nopqmf_oracle.py reproduces them.  Writes new files only:

    python -m oracle.make_golden_nopqmf

  tests/golden/autoencoder_v2_nopqmf_tiny.pt     tiny PQMF-in / raw-out autoencoder: forward, grad_x and every
                                                 parameter gradient of a probed output
  tests/golden/training_step_v2_nopqmf_tiny.pt   the reference's own RAVE.training_step, a phase-2 D-step and a phase-2
                                                 G-step from the same seeded parameters: logged losses, sampled gradients
  tests/golden/state_dict_keys_nopqmf.pt         keys / shapes / dtypes of the full-size rave.RAVE of this configuration
"""
import os
import sys
from functools import partial

import torch
import torch.nn as nn

from oracle import nopqmf_oracle as N
from oracle import rave_oracle as O
from oracle.make_golden import GOLDEN, check, make_input
from oracle.ref_loader import load_reference, set_padding_mode

GRAD_SAMPLE = 8192


def build_ref_rave_nopqmf(R, cfg: O.ArchConfig, disc_capacity=4, update_discriminator_every=4, phase_1_duration=1000,
                          gen_ratios=N.GEN_RATIOS):
    """The reference's rave.RAVE bound like configs/v2_nopqmf.gin (44-106) on top of configs/v1.gin."""
    D, blocks, core = R.discriminator, R.blocks, R.core
    norm = blocks.normalization
    D.normalization = lambda m, mode="weight_norm": norm(m, mode)
    act = lambda dim: nn.LeakyReLU(.2)
    periods_net = partial(D.ConvNet, out_size=1, capacity=disc_capacity, n_layers=4, stride=4, conv=nn.Conv2d,
                          kernel_size=(5, 1))
    scales_net = partial(D.ConvNet, out_size=1, capacity=disc_capacity, n_layers=4, stride=4, conv=nn.Conv1d,
                         kernel_size=15)
    disc = partial(D.CombineDiscriminators, [
        partial(D.MultiPeriodDiscriminator, periods=[2, 3, 5, 7, 11], convnet=periods_net),
        partial(D.MultiScaleDiscriminator, n_discriminators=3, convnet=scales_net)])
    enc = partial(blocks.VariationalEncoder,
                  partial(blocks.EncoderV2, data_size=cfg.n_band, capacity=cfg.capacity, ratios=cfg.ratios,
                          latent_size=cfg.latent_size, n_out=2, kernel_size=cfg.kernel_size, dilations=cfg.dilations,
                          activation=act, adain=None))
    dec = partial(blocks.GeneratorV2, capacity=cfg.capacity, ratios=list(gen_ratios), latent_size=cfg.latent_size,
                  kernel_size=cfg.kernel_size, dilations=cfg.dilations, amplitude_modulation=True, activation=act,
                  adain=None)
    stft = partial(core.MultiScaleSTFT, scales=[2048, 1024, 512, 256, 128], sample_rate=48000, magnitude=True)
    dist = partial(core.AudioDistanceV1, multiscale_stft=stft, log_epsilon=1e-7)
    try:
        m = R.model.RAVE(latent_size=cfg.latent_size, sampling_rate=48000, encoder=enc, decoder=dec,
                         discriminator=disc, phase_1_duration=phase_1_duration, gan_loss=core.hinge_gan,
                         valid_signal_crop=True,
                         feature_matching_fun=partial(core.mean_difference, norm="L1", relative=True),
                         num_skipped_features=1, audio_distance=dist, multiband_audio_distance=dist,
                         weights={"feature_matching": 20}, n_bands=cfg.n_band,
                         pqmf=partial(R.pqmf.CachedPQMF, attenuation=100, n_band=cfg.n_band),
                         update_discriminator_every=update_discriminator_every, n_channels=1, output_mode="raw")
    finally:
        D.normalization = norm
    return m


def golden_autoencoder_nopqmf(R, capacity=2, latent_size=16, B=1, T=8192):
    """PQMF analysis -> EncoderV2 -> reparametrisation -> raw GeneratorV2 at a tiny capacity; the gradients of
    sum(y * probe) with respect to x and every encoder / decoder parameter."""
    print("autoencoder v2_nopqmf (tiny)")
    set_padding_mode("centered")
    cfg = O.ArchConfig(capacity=capacity, latent_size=latent_size)
    gcfg = N.generator_config(cfg)
    torch.manual_seed(0)
    m = build_ref_rave_nopqmf(R, cfg)
    pq, enc, dec = m.pqmf, m.encoder, m.decoder
    enc.train(), dec.train()
    x = make_input(B, 1, T, seed=21)
    sd = {"pqmf." + k: v for k, v in pq.state_dict().items()}
    sd.update({"encoder." + k: v for k, v in enc.state_dict().items()})
    sd.update({"decoder." + k: v for k, v in dec.state_dict().items()})
    sd = {k: v.detach().clone() for k, v in sd.items()}
    xg = x.clone().requires_grad_(True)
    z = enc(R.model._pqmf_encode(pq, xg))
    g = torch.Generator().manual_seed(4321)
    eps = torch.randn(z.shape[0], z.shape[1] // 2, z.shape[2], generator=g)
    mean, scale = z.chunk(2, 1)
    zs = eps * (nn.functional.softplus(scale) + 1e-4) + mean
    y = dec(zs)
    y_o = N.rave_forward_raw(x, sd, cfg, gcfg, eps)
    assert y.shape == y_o.shape == x.shape, (y.shape, x.shape)
    check("y", y_o, y, 1e-6)
    probe = torch.randn(y.shape, generator=torch.Generator().manual_seed(777))
    params = dict(enc.named_parameters(prefix="encoder"))
    params.update(dict(dec.named_parameters(prefix="decoder")))
    names = sorted(params)
    grads = torch.autograd.grad((y * probe).sum(), [xg] + [params[n] for n in names])
    po = {k: v.clone().requires_grad_(v.is_floating_point() and not k.startswith("pqmf.")) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    go = torch.autograd.grad((N.rave_forward_raw(xo, po, cfg, gcfg, eps) * probe).sum(), [xo] + [po[n] for n in names])
    check("grad_x", go[0], grads[0], 1e-5)
    for n, a, b in zip(names, go[1:], grads[1:]):
        check(f"grad {n}", a, b, 1e-5)
    fx = dict(cfg=vars(cfg), gen_ratios=list(N.GEN_RATIOS), state_dict=sd, x=x, eps=eps, y=y.detach(), probe=probe,
              grad_x=grads[0].detach(), grad_params={n: g_.detach().clone() for n, g_ in zip(names, grads[1:])})
    torch.save(fx, os.path.join(GOLDEN, "autoencoder_v2_nopqmf_tiny.pt"))


def golden_training_step_nopqmf(R, B=2, T=32768, param_seed=41, disc_capacity=4):
    """The reference's OWN RAVE.training_step (rave/model.py:288-424) in phase 2 with output_mode "raw": a D-step
    (batch_idx 0) and a G-step (batch_idx 1), each from the same seeded parameters.  Commits the logged scalars and a
    seeded sample of the gradients the step's optimiser consumed (discriminator.* after the D-step, decoder.* after the
    G-step)."""
    print("RAVE.training_step v2_nopqmf (phase-2 D, phase-2 G)")
    set_padding_mode("centered")
    cfg = O.ArchConfig(capacity=8, latent_size=16)
    gcfg = N.generator_config(cfg)
    torch.manual_seed(0)
    m = build_ref_rave_nopqmf(R, cfg, disc_capacity, update_discriminator_every=2)
    shapes = [(k, tuple(v.shape)) for k, v in m.named_parameters() if not k.startswith("pqmf.")]
    m.load_state_dict(N.seeded_params(shapes, param_seed), strict=False)
    m.train()
    m.warmed_up = True
    rf = (1024, 512)
    m.receptive_field[0], m.receptive_field[1] = rf
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
    for name, batch_idx, seed in (("phase2_dis", 0, 111), ("phase2_gen", 1, 112)):
        m.load_state_dict(sd0)
        x = N.step_batch(B, T, seed)
        torch.manual_seed(seed)
        eps = torch.randn(B, cfg.latent_size, Lz)
        assert torch.equal(eps, N.step_eps(B, cfg.latent_size, Lz, seed))
        torch.manual_seed(seed)
        logs.clear()
        m.training_step(x.clone(), batch_idx)
        dis = batch_idx % m.update_discriminator_every == 0
        grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()
                 if p.grad is not None and k.startswith("discriminator.") == dis
                 and not k.startswith(("encoder.", "pqmf."))}
        keys = sorted(grads)
        steps.append(dict(name=name, batch_idx=batch_idx, seed=seed, logs={k: v.clone() for k, v in logs.items()},
                          grad_keys=keys, grad_sample=N.sample(torch.cat([grads[k].reshape(-1) for k in keys]),
                                                               GRAD_SAMPLE, seed=seed)))
        print("  ", name, {k: round(float(v), 6) for k, v in logs.items()})
        losses, ldis = N.train_step_losses(x, sd0, cfg, gcfg, eps, receptive_field=rf)
        for k, v in losses.items():
            check(f"{name} {k}", v, logs[k], 2e-6)
        check(f"{name} loss_dis", ldis, logs["loss_dis"], 2e-6)
    torch.save(dict(cfg=vars(cfg), gen_ratios=list(N.GEN_RATIOS), B=B, T=T, disc_capacity=disc_capacity,
                    update_discriminator_every=m.update_discriminator_every, receptive_field=rf,
                    param_shapes=shapes, param_seed=param_seed, hk=sd0["pqmf.hk"], steps=steps),
               os.path.join(GOLDEN, "training_step_v2_nopqmf_tiny.pt"))


def golden_state_dict_keys_nopqmf(R):
    """Key list of the full-size rave.RAVE of `--config v2_nopqmf`."""
    print("state_dict key contract (v2_nopqmf, full size)")
    torch.manual_seed(0)
    m = build_ref_rave_nopqmf(R, O.ArchConfig(capacity=N.CAPACITY), disc_capacity=N.CAPACITY)
    out = {"rave_v2_nopqmf": {k: (tuple(v.shape), str(v.dtype)) for k, v in m.state_dict().items()}}
    print(f"  rave_v2_nopqmf: {len(out['rave_v2_nopqmf'])} keys")
    torch.save(out, os.path.join(GOLDEN, "state_dict_keys_nopqmf.pt"))


def main():
    os.makedirs(GOLDEN, exist_ok=True)
    R = load_reference()
    norm = R.blocks.normalization
    R.blocks.normalization = lambda m, mode="weight_norm": norm(m, mode)  # configs/v1.gin:41
    golden_autoencoder_nopqmf(R)
    golden_training_step_nopqmf(R)
    golden_state_dict_keys_nopqmf(R)
    for f in ("autoencoder_v2_nopqmf_tiny.pt", "training_step_v2_nopqmf_tiny.pt", "state_dict_keys_nopqmf.pt"):
        print(f, os.path.getsize(os.path.join(GOLDEN, f)), "bytes")


if __name__ == "__main__":
    sys.exit(main())

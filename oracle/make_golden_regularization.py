"""TEST INFRASTRUCTURE -- generates the fixtures of the two v2 regularisation options (`--config v2 --config
wasserstein`, `--config v2 --config spherical`) by EXECUTING THE UNMODIFIED REFERENCE, and asserts that
oracle/regularization_oracle.py reproduces them.  Writes new files only:

    python -m oracle.make_golden_regularization

  tests/golden/autoencoder_v2_wasserstein_tiny.pt     tiny WAE autoencoder, prior sample and noise injected: forward,
                                                      MMD (and its three kernel means), grad_x and every parameter
                                                      gradient of sum(y * probe) + 100 * MMD
  tests/golden/training_step_v2_wasserstein_tiny.pt   the reference's own RAVE.training_step (beta_factor 100): a
                                                      phase-1 G-step, a phase-2 D-step and a phase-2 G-step from the same
                                                      seeded parameters: logged losses, sampled gradients
  tests/golden/training_step_v2_spherical_tiny.pt     the same for the spherical configuration: phase-1 G and phase-2 G
  tests/golden/state_dict_keys_regularization.pt      keys / shapes / dtypes of the full-size rave.RAVE of both
"""
import os
import sys
from functools import partial

import torch
import torch.nn as nn

from oracle import rave_oracle as O
from oracle import regularization_oracle as G
from oracle.make_golden import GOLDEN, check, make_input
from oracle.ref_loader import load_reference, set_padding_mode

GRAD_SAMPLE = 8192
FILES = ("autoencoder_v2_wasserstein_tiny.pt", "training_step_v2_wasserstein_tiny.pt",
         "training_step_v2_spherical_tiny.pt", "state_dict_keys_regularization.pt")


_REF_DEFAULT_WEIGHTS = {"audio_distance": 1., "multiband_audio_distance": 1., "adversarial": 1., "feature_matching": 20}


def build_ref_rave_reg(R, kind: str, cfg: O.ArchConfig, disc_capacity=4, update_discriminator_every=2,
                       phase_1_duration=1000):
    """The reference's rave.RAVE bound like configs/v2.gin + configs/{wasserstein,spherical}.gin."""
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
    enc_v2 = partial(blocks.EncoderV2, data_size=cfg.n_band, capacity=cfg.capacity, ratios=cfg.ratios,
                     latent_size=cfg.latent_size, n_out=1, kernel_size=cfg.kernel_size, dilations=cfg.dilations,
                     activation=act, adain=None)
    if kind == "wasserstein":
        enc = partial(blocks.WasserteinEncoder, encoder_cls=enc_v2, noise_augmentation=G.NOISE_AUGMENTATION)
        weights = {k: v for k, v in G.WAE_WEIGHTS.items() if k != "feature_matching"}
    else:
        enc = partial(blocks.SphericalEncoder, encoder_cls=enc_v2)
        weights = dict(G.DEFAULT_WEIGHTS)
    dec = partial(blocks.GeneratorV2, data_size=cfg.n_band, capacity=cfg.capacity, ratios=cfg.ratios,
                  latent_size=cfg.generator_latent, kernel_size=cfg.kernel_size, dilations=cfg.dilations,
                  amplitude_modulation=True, activation=act, adain=None)
    stft = partial(core.MultiScaleSTFT, scales=[2048, 1024, 512, 256, 128], sample_rate=48000, magnitude=True)
    dist = partial(core.AudioDistanceV1, multiscale_stft=stft, log_epsilon=1e-7)
    # RAVE.__init__ updates the module-global default dict in place (quirk D1): restore it so that one configuration's
    # weights do not leak into the next model built in this process, as they would not across two training runs
    R.model._default_loss_weights.clear()
    R.model._default_loss_weights.update(_REF_DEFAULT_WEIGHTS)
    try:
        m = R.model.RAVE(latent_size=cfg.latent_size, sampling_rate=48000, encoder=enc, decoder=dec,
                         discriminator=disc, phase_1_duration=phase_1_duration, gan_loss=core.hinge_gan,
                         valid_signal_crop=True,
                         feature_matching_fun=partial(core.mean_difference, norm="L1", relative=True),
                         num_skipped_features=1, audio_distance=dist, multiband_audio_distance=dist,
                         weights=weights, n_bands=cfg.n_band,
                         pqmf=partial(R.pqmf.CachedPQMF, attenuation=100, n_band=cfg.n_band),
                         update_discriminator_every=update_discriminator_every, n_channels=1)
    finally:
        D.normalization = norm
    return m


def check_loss(name, got, want, tol=2e-6, floor=1e-2):
    """Relative error of a logged loss, its scale floored at `floor`: the adversarial term is a mean of scores that
    cancel (|value| ~ 2e-3 here), where the two sides' fp32 summation orders alone differ by a few 1e-6 relatively."""
    err = abs(float(got) - float(want)) / max(abs(float(want)), floor)
    status = "ok" if err <= tol else "FAIL"
    print(f"  [{status}] {name}: {err:.3e} (tol {tol:g})")
    assert err <= tol, name


def spy_reparametrize(enc):
    """Records (z, output, reg) of every reparametrize call of the reference encoder."""
    calls = []
    orig = enc.reparametrize

    def spy(z):
        out, reg = orig(z)
        calls.append((z.detach().clone(), out.detach().clone(), reg.detach().clone()))
        return out, reg
    enc.reparametrize = spy
    return calls


def check_draws(enc, call, prior, noise):
    """The reference's own draws equal the reconstruction: the appended noise bit for bit, and its MMD computed with
    the reconstructed prior sample bit for bit."""
    z, out, reg = call
    assert torch.equal(out[:, z.shape[1]:], noise)
    assert torch.equal(enc.compute_mmd(G.rows(z), prior), reg)


def golden_autoencoder_wae(R, capacity=2, B=2, T=8192, seed=77):
    print("autoencoder v2_wasserstein (tiny)")
    set_padding_mode("centered")
    cfg = G.config("wasserstein", capacity)
    torch.manual_seed(0)
    m = build_ref_rave_reg(R, "wasserstein", cfg)
    pq, enc, dec = m.pqmf, m.encoder, m.decoder
    enc.train(), dec.train()
    x = make_input(B, 1, T, seed=31)
    sd = {"pqmf." + k: v for k, v in pq.state_dict().items()}
    sd.update({"encoder." + k: v for k, v in enc.state_dict().items()})
    sd.update({"decoder." + k: v for k, v in dec.state_dict().items()})
    sd = {k: v.detach().clone() for k, v in sd.items()}
    calls = spy_reparametrize(enc)
    xg = x.clone().requires_grad_(True)
    z = enc(R.model._pqmf_encode(pq, xg))
    torch.manual_seed(seed)
    zs, reg = enc.reparametrize(z)
    prior, noise = G.draws(B, cfg.latent_size, z.shape[-1], seed)
    check_draws(enc, calls[0], prior, noise)
    y = R.model._pqmf_decode(pq, dec(zs), batch_size=x.shape[:-2], n_channels=1)
    y_o, reg_o = G.rave_forward(x, sd, cfg, "wasserstein", prior, noise)
    check("y", y_o, y, 1e-6)
    check("mmd", reg_o, reg, 1e-6)
    probe = torch.randn(y.shape, generator=torch.Generator().manual_seed(778))
    params = dict(enc.named_parameters(prefix="encoder"))
    params.update(dict(dec.named_parameters(prefix="decoder")))
    names = sorted(params)
    grads = torch.autograd.grad((y * probe).sum() + G.BETA * reg, [xg] + [params[n] for n in names])
    po = {k: v.clone().requires_grad_(v.is_floating_point() and not k.startswith("pqmf.")) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    yo, rego = G.rave_forward(xo, po, cfg, "wasserstein", prior, noise)
    go = torch.autograd.grad((yo * probe).sum() + G.BETA * rego, [xo] + [po[n] for n in names])
    check("grad_x", go[0], grads[0], 1e-5)
    for n, a, b in zip(names, go[1:], grads[1:]):
        check(f"grad {n}", a, b, 1e-5)
    terms = torch.stack(G.mmd_terms(calls[0][0], prior))
    fx = dict(cfg=vars(cfg), state_dict=sd, x=x, prior=prior, noise=noise, z=calls[0][0], y=y.detach(),
              mmd=reg.detach(), mmd_terms=terms, probe=probe, beta=G.BETA, grad_x=grads[0].detach(),
              grad_params={n: g_.detach().clone() for n, g_ in zip(names, grads[1:])})
    torch.save(fx, os.path.join(GOLDEN, "autoencoder_v2_wasserstein_tiny.pt"))


def golden_training_step(R, kind, steps_spec, B=2, T=32768, param_seed=43, disc_capacity=4):
    """The reference's OWN RAVE.training_step (rave/model.py:288-424), each step from the same seeded parameters.
    Commits the logged scalars and seeded samples of the gradients the step's optimiser consumed: discriminator.*
    after a D-step; encoder.* (when it has a gradient) and decoder.* separately after a G-step."""
    print(f"RAVE.training_step v2_{kind} ({', '.join(s[0] for s in steps_spec)})")
    set_padding_mode("centered")
    cfg = G.config(kind, 8)
    beta = G.BETA if kind == "wasserstein" else 1.0
    torch.manual_seed(0)
    m = build_ref_rave_reg(R, kind, cfg, disc_capacity, update_discriminator_every=2)
    shapes = [(k, tuple(v.shape)) for k, v in m.named_parameters() if not k.startswith("pqmf.")]
    m.load_state_dict(G.seeded_params(shapes, param_seed), strict=False)
    m.train()
    m.beta_factor = beta
    rf = (1024, 512)
    m.receptive_field[0], m.receptive_field[1] = rf
    opts = m.configure_optimizers()
    gen_opt, dis_opt = opts[0]["optimizer"], opts[1]["optimizer"]
    logs = {}
    m.optimizers = lambda: (gen_opt, dis_opt)
    m.log = lambda k, v: logs.__setitem__(k, v.detach().clone() if torch.is_tensor(v) else torch.tensor(float(v)))
    m.log_dict = lambda d: [m.log(k, v) for k, v in d.items()]
    sd0 = {k: v.detach().clone() for k, v in m.state_dict().items()}
    calls = spy_reparametrize(m.encoder)
    Lz = T // cfg.n_band
    for r in cfg.ratios:
        Lz //= r
    steps = []
    for name, warmed, batch_idx, seed in steps_spec:
        m.load_state_dict(sd0)
        for p in m.parameters():
            p.grad = None
        m.warmed_up = warmed
        x = G.step_batch(B, T, seed)
        prior, noise = G.draws(B, cfg.latent_size, Lz, seed) if kind == "wasserstein" else (None, None)
        torch.manual_seed(seed)
        logs.clear()
        n_calls = len(calls)
        m.training_step(x.clone(), batch_idx)
        assert len(calls) == n_calls + 1
        if kind == "wasserstein":
            check_draws(m.encoder, calls[-1], prior, noise)
        dis = warmed and batch_idx % m.update_discriminator_every == 0
        grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()
                 if p.grad is not None and k.startswith("discriminator.") == dis and not k.startswith("pqmf.")}
        st = dict(name=name, warmed_up=warmed, batch_idx=batch_idx, seed=seed,
                  logs={k: v.clone() for k, v in logs.items()})
        groups = ("discriminator.",) if dis else ("encoder.", "decoder.")
        for gname in groups:
            keys = sorted(k for k in grads if k.startswith(gname))
            tag = gname[:-1]
            st[f"{tag}_keys"] = keys
            st[f"{tag}_sample"] = (G.sample(torch.cat([grads[k].reshape(-1) for k in keys]), GRAD_SAMPLE, seed=seed)
                                   if keys else None)
        steps.append(st)
        print("  ", name, {k: round(float(v), 6) for k, v in logs.items()},
              {k[:-5]: len(v) for k, v in st.items() if k.endswith("_keys")})
        losses, ldis, _ = G.train_step_losses(x, sd0, cfg, kind, warmed, prior, noise, beta, receptive_field=rf)
        for k, v in losses.items():
            if k == "regularization" and k not in logs:
                assert float(v) == 0.0            # `if reg.item():` (rave/model.py:388) skips a zero regulariser
                continue
            check_loss(f"{name} {k}", v, logs[k])
        if warmed:
            check_loss(f"{name} loss_dis", ldis, logs["loss_dis"])
    torch.save(dict(kind=kind, cfg=vars(cfg), B=B, T=T, beta_factor=beta, disc_capacity=disc_capacity,
                    update_discriminator_every=m.update_discriminator_every, receptive_field=rf,
                    param_shapes=shapes, param_seed=param_seed, hk=sd0["pqmf.hk"], steps=steps),
               os.path.join(GOLDEN, f"training_step_v2_{kind}_tiny.pt"))


def golden_state_dict_keys(R):
    """Key lists of the full-size rave.RAVE of both configurations."""
    print("state_dict key contract (v2_wasserstein, v2_spherical, full size)")
    out = {}
    for kind in ("wasserstein", "spherical"):
        torch.manual_seed(0)
        m = build_ref_rave_reg(R, kind, G.config(kind, 96), disc_capacity=96)
        out[f"rave_v2_{kind}"] = {k: (tuple(v.shape), str(v.dtype)) for k, v in m.state_dict().items()}
        print(f"  rave_v2_{kind}: {len(out[f'rave_v2_{kind}'])} keys")
    torch.save(out, os.path.join(GOLDEN, "state_dict_keys_regularization.pt"))


def main():
    os.makedirs(GOLDEN, exist_ok=True)
    R = load_reference()
    norm = R.blocks.normalization
    R.blocks.normalization = lambda m, mode="weight_norm": norm(m, mode)  # configs/v1.gin:41
    golden_autoencoder_wae(R)
    golden_training_step(R, "wasserstein", (("phase1_gen", False, 0, 200), ("phase2_dis", True, 0, 201),
                                            ("phase2_gen", True, 1, 202)))
    golden_training_step(R, "spherical", (("phase1_gen", False, 0, 210), ("phase2_gen", True, 1, 212)))
    golden_state_dict_keys(R)
    for f in FILES:
        print(f, os.path.getsize(os.path.join(GOLDEN, f)), "bytes")


if __name__ == "__main__":
    sys.exit(main())

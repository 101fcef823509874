"""TEST INFRASTRUCTURE -- generates the fixtures of the hybrid configuration (rave/configs/hybrid.gin on top of v2.gin:
mel-spectrogram encoder input, GRU generator head) by EXECUTING THE UNMODIFIED REFERENCE (torchaudio's MelSpectrogram,
rave.blocks.GRU, rave.RAVE), and asserts that oracle/hybrid_oracle.py reproduces them.  Writes new files only:

    python -m oracle.make_golden_hybrid

  tests/golden/mel_filterbanks.pt               torchaudio's MelScale.fb at 44.1 and 48 kHz (n_fft 2048, 128 bands), as
                                                its nonzero entries
  tests/golden/state_dict_keys_hybrid.pt        keys / shapes / dtypes of the full-size rave.RAVE of v2 + hybrid (mono
                                                and stereo) and v3 + hybrid
  tests/golden/autoencoder_v2_hybrid_tiny.pt    mel front end -> encoder -> GRU -> generator -> PQMF synthesis at
                                                capacity 4 from seeded parameters: forward, every encoder / decoder
                                                parameter gradient (a seeded sample of the large ones)
  tests/golden/training_step_v2_hybrid_tiny.pt  the reference's own RAVE.training_step: phase-1 G-step, phase-2 D-step,
                                                phase-2 G-step from the same seeded parameters

The reference's training step cannot run in mel mode as written (quirk D9, SURVEY.md): `encode(x, return_mb=True)`
applies PQMF analysis to the mel spectrogram, whose shape AudioDistanceV1 rejects.  For the training-step fixture ONLY,
the reference's `encode` is replaced by the same method with `x_multiband = PQMF(x)`, the waveform's analysis -- the
one substitution this script makes.
"""
import os
import sys
from functools import partial

import torch
import torch.nn as nn

from oracle import hybrid_oracle as Hy
from oracle import rave_oracle as O
from oracle.make_golden import GOLDEN, check, make_input
from oracle.ref_loader import load_reference, set_padding_mode

GRAD_SAMPLE = 8192


def build_ref_rave_hybrid(R, cfg: O.ArchConfig, disc_capacity=4, update_discriminator_every=4, phase_1_duration=1000,
                          kind="v2", n_channels=1, sr=48000):
    """rave.RAVE bound like configs/hybrid.gin on top of configs/v2.gin (or v3.gin: snake, AdaIN, Descript)."""
    import torchaudio
    D, blocks, core = R.discriminator, R.blocks, R.core
    norm = blocks.normalization
    D.normalization = lambda m, mode="weight_norm": norm(m, mode)
    v3 = kind == "v3"
    act = (lambda dim: blocks.Snake(dim)) if v3 else (lambda dim: nn.LeakyReLU(.2))
    adain = (lambda dim: blocks.AdaptiveInstanceNormalization(dim)) if v3 else None
    if v3:
        disc = R.descript_discriminator.DescriptDiscriminator
    else:
        periods_net = partial(D.ConvNet, out_size=1, capacity=disc_capacity, n_layers=4, stride=4, conv=nn.Conv2d,
                              kernel_size=(5, 1))
        scales_net = partial(D.ConvNet, out_size=1, capacity=disc_capacity, n_layers=4, stride=4, conv=nn.Conv1d,
                             kernel_size=15)
        disc = partial(D.CombineDiscriminators, [
            partial(D.MultiPeriodDiscriminator, periods=[2, 3, 5, 7, 11], convnet=periods_net),
            partial(D.MultiScaleDiscriminator, n_discriminators=3, convnet=scales_net)])
    enc = partial(blocks.VariationalEncoder,
                  partial(blocks.EncoderV2, data_size=Hy.N_MELS, capacity=cfg.capacity, ratios=list(Hy.ENC_RATIOS),
                          latent_size=cfg.latent_size, n_out=2, kernel_size=cfg.kernel_size,
                          dilations=list(Hy.ENC_DILATIONS), activation=act, adain=adain))
    dec = partial(blocks.GeneratorV2, data_size=cfg.n_band, capacity=cfg.capacity, ratios=cfg.ratios,
                  latent_size=cfg.latent_size, kernel_size=cfg.kernel_size, dilations=cfg.dilations,
                  amplitude_modulation=True, activation=act, adain=adain,
                  recurrent_layer=partial(blocks.GRU, num_layers=Hy.NUM_GRU_LAYERS))
    stft = partial(core.MultiScaleSTFT, scales=[2048, 1024, 512, 256, 128], sample_rate=sr, magnitude=True)
    dist = partial(core.AudioDistanceV1, multiscale_stft=stft, log_epsilon=1e-7)
    mel = torchaudio.transforms.MelSpectrogram(sample_rate=sr, n_fft=Hy.N_FFT, win_length=Hy.N_FFT,
                                               hop_length=Hy.HOP, normalized=True, n_mels=Hy.N_MELS)
    orig_du = blocks.DilatedUnit
    blocks.DilatedUnit = partial(orig_du, activation=act)
    try:
        m = R.model.RAVE(latent_size=cfg.latent_size, sampling_rate=sr, encoder=enc, decoder=dec, discriminator=disc,
                         phase_1_duration=phase_1_duration, gan_loss=core.hinge_gan, valid_signal_crop=True,
                         feature_matching_fun=partial(core.mean_difference, norm="L1", relative=True),
                         num_skipped_features=1, audio_distance=dist, multiband_audio_distance=dist,
                         weights={"feature_matching": 20}, n_bands=cfg.n_band,
                         pqmf=partial(R.pqmf.CachedPQMF, attenuation=100, n_band=cfg.n_band),
                         update_discriminator_every=update_discriminator_every, n_channels=n_channels,
                         spectrogram=mel, input_mode="mel")
    finally:
        blocks.DilatedUnit = orig_du
        D.normalization = norm
    return m


def golden_filterbanks():
    """Stored as nonzero entries (hybrid_oracle.pack_filterbank): 2019 of 1025 x 128 at 48 kHz."""
    import torchaudio
    print("mel filter banks")
    out = {}
    for sr in (44100, 48000):
        fb = torchaudio.transforms.MelSpectrogram(sample_rate=sr, n_fft=Hy.N_FFT, win_length=Hy.N_FFT, hop_length=Hy.HOP,
                                                  normalized=True, n_mels=Hy.N_MELS).mel_scale.fb
        out[sr] = Hy.pack_filterbank(fb)
        assert torch.equal(Hy.dense_filterbank(out[sr]), fb)
        print(f"  {sr}: {tuple(fb.shape)}, {out[sr]['value'].numel()} nonzeros")
    torch.save(out, os.path.join(GOLDEN, "mel_filterbanks.pt"))


def golden_state_dict_keys(R):
    print("state_dict key contract (hybrid, full size)")
    out = {}
    for name, kind, C in (("rave_v2_hybrid", "v2", 1), ("rave_v2_hybrid_stereo", "v2", 2), ("rave_v3_hybrid", "v3", 1)):
        torch.manual_seed(0)
        cfg = O.ArchConfig(activation="snake" if kind == "v3" else "leaky", adain=kind == "v3")
        m = build_ref_rave_hybrid(R, cfg, disc_capacity=96, kind=kind, n_channels=C)
        out[name] = {k: (tuple(v.shape), str(v.dtype)) for k, v in m.state_dict().items()}
        print(f"  {name}: {len(out[name])} keys")
    torch.save(out, os.path.join(GOLDEN, "state_dict_keys_hybrid.pt"))


def golden_autoencoder(R, capacity=4, latent_size=128, B=2, T=8192, param_seed=61):
    """Parameters drawn by hybrid_oracle.seeded_params (the fixture keeps their shapes and the seed), buffers except the
    filter bank (in mel_filterbanks.pt), and the parameter gradients as hybrid_oracle.grad_record stores them."""
    print("autoencoder v2 + hybrid (tiny)")
    set_padding_mode("centered")
    cfg = O.ArchConfig(capacity=capacity, latent_size=latent_size)
    torch.manual_seed(0)
    m = build_ref_rave_hybrid(R, cfg)
    shapes = [(k, tuple(v.shape)) for k, v in m.named_parameters() if k.startswith(("encoder.", "decoder."))]
    m.load_state_dict(Hy.seeded_params(shapes, param_seed), strict=False)
    m.train()
    x = make_input(B, 1, T, seed=31)
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()
          if k.startswith(("pqmf.", "spectrogram.", "encoder.", "decoder."))}
    fb = sd["spectrogram.mel_scale.fb"]
    z = m.encoder(m._mel_encode(x))
    g = torch.Generator().manual_seed(4321)
    eps = torch.randn(z.shape[0], z.shape[1] // 2, z.shape[2], generator=g)
    mean, scale = z.chunk(2, 1)
    zs = eps * (nn.functional.softplus(scale) + 1e-4) + mean
    y = m.decode(zs)
    taps = {}
    y_o = Hy.rave_forward_hybrid(x, sd, cfg, eps, taps)
    check("x_mel", taps["x_mel"], m._mel_encode(x), 1e-5)
    check("y", y_o, y, 1e-5)
    probe = torch.randn(y.shape, generator=torch.Generator().manual_seed(777))
    params = dict(m.encoder.named_parameters(prefix="encoder"))
    params.update(dict(m.decoder.named_parameters(prefix="decoder")))
    names = sorted(params)
    grads = torch.autograd.grad((y * probe).sum(), [params[n] for n in names])
    po = {k: v.clone().requires_grad_(k in params) for k, v in sd.items()}
    go = torch.autograd.grad((Hy.rave_forward_hybrid(x, po, cfg, eps) * probe).sum(), [po[n] for n in names])
    for n, a, b in zip(names, go, grads):
        check(f"grad {n}", a, b, 1e-4)
    params_keys = {k for k, _ in shapes}
    buffers = {k: v for k, v in sd.items() if k not in params_keys and k != "spectrogram.mel_scale.fb"}
    fx = dict(cfg=vars(cfg), param_shapes=shapes, param_seed=param_seed, buffers=buffers, x=x, eps=eps,
              x_mel=taps["x_mel"].detach(), y=y.detach(), probe_seed=777,
              grad_params={n: Hy.grad_record(g_, i) for i, (n, g_) in enumerate(zip(names, grads))})
    assert all(torch.equal(v, sd[k]) for k, v in Hy.autoencoder_state(fx, fb).items())
    torch.save(fx, os.path.join(GOLDEN, "autoencoder_v2_hybrid_tiny.pt"))


def _encode_waveform_multiband(R, m):
    """rave/model.py:244-258 with the one substitution of quirk D9: the multiband target is the waveform's analysis."""
    def encode(x, return_mb: bool = False):
        z = m.encoder(m._mel_encode(x))
        if return_mb:
            return z, R.model._pqmf_encode(m.pqmf, x)
        return z
    return encode


def golden_training_step(R, B=2, T=32768, param_seed=51, disc_capacity=4):
    print("RAVE.training_step v2 + hybrid (phase-1 G, phase-2 D, phase-2 G)")
    set_padding_mode("centered")
    cfg = O.ArchConfig(capacity=16, latent_size=128)
    torch.manual_seed(0)
    m = build_ref_rave_hybrid(R, cfg, disc_capacity, update_discriminator_every=2)
    m.encode = _encode_waveform_multiband(R, m)
    shapes = [(k, tuple(v.shape)) for k, v in m.named_parameters() if not k.startswith("pqmf.")]
    m.load_state_dict(Hy.seeded_params(shapes, param_seed), strict=False)
    m.train()
    rf = (1024, 512)
    m.receptive_field[0], m.receptive_field[1] = rf
    opts = m.configure_optimizers()
    gen_opt, dis_opt = opts[0]["optimizer"], opts[1]["optimizer"]
    logs = {}
    m.optimizers = lambda: (gen_opt, dis_opt)
    m.log = lambda k, v: logs.__setitem__(k, v.detach().clone() if torch.is_tensor(v) else torch.tensor(float(v)))
    m.log_dict = lambda d: [m.log(k, v) for k, v in d.items()]
    sd0 = {k: v.detach().clone() for k, v in m.state_dict().items()}
    Lz = T // 2048
    steps = []
    for name, batch_idx, seed, warm in (("phase1_gen", 1, 110, False), ("phase2_dis", 0, 111, True),
                                        ("phase2_gen", 1, 112, True)):
        m.load_state_dict(sd0)
        m.warmed_up = warm
        x = Hy.step_batch(B, T, seed)
        torch.manual_seed(seed)
        eps = torch.randn(B, cfg.latent_size, Lz)
        assert torch.equal(eps, Hy.step_eps(B, cfg.latent_size, Lz, seed))
        torch.manual_seed(seed)
        logs.clear()
        for p in m.parameters():
            p.grad = None
        m.training_step(x.clone(), batch_idx)
        dis = warm and batch_idx % m.update_discriminator_every == 0
        grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()
                 if p.grad is not None and k.startswith("discriminator.") == dis and not k.startswith("pqmf.")}
        keys = sorted(grads)
        steps.append(dict(name=name, batch_idx=batch_idx, seed=seed, warmed_up=warm,
                          logs={k: v.clone() for k, v in logs.items()}, grad_keys=keys,
                          grad_sample=Hy.sample(torch.cat([grads[k].reshape(-1) for k in keys]), GRAD_SAMPLE,
                                                seed=seed)))
        print("  ", name, {k: round(float(v), 6) for k, v in logs.items()})
        losses, ldis = Hy.train_step_losses(x, sd0, cfg, eps, warm, receptive_field=rf)
        for k, v in losses.items():
            check(f"{name} {k}", v, logs[k], 2e-5)
        if ldis is not None:
            check(f"{name} loss_dis", ldis, logs["loss_dis"], 2e-5)
    torch.save(dict(cfg=vars(cfg), B=B, T=T, disc_capacity=disc_capacity,
                    update_discriminator_every=m.update_discriminator_every, receptive_field=rf, param_shapes=shapes,
                    param_seed=param_seed, steps=steps),
               os.path.join(GOLDEN, "training_step_v2_hybrid_tiny.pt"))


def main():
    os.makedirs(GOLDEN, exist_ok=True)
    R = load_reference()
    norm = R.blocks.normalization
    R.blocks.normalization = lambda m, mode="weight_norm": norm(m, mode)  # configs/v1.gin:41
    golden_filterbanks()
    golden_autoencoder(R)
    golden_training_step(R)
    golden_state_dict_keys(R)
    for f in ("mel_filterbanks.pt", "autoencoder_v2_hybrid_tiny.pt", "training_step_v2_hybrid_tiny.pt",
              "state_dict_keys_hybrid.pt"):
        print(f, os.path.getsize(os.path.join(GOLDEN, f)), "bytes")


if __name__ == "__main__":
    sys.exit(main())

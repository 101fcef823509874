"""gin-free instantiation of the reference's configurations (gin-config is not installable
here; SURVEY.md App. B.1 lists the effective bindings with file:line provenance).

`build_rave("v2", sampling_rate=48000)` returns the same module tree (same `state_dict` keys and
shapes) that `scripts/train.py --config v2 --override SAMPLING_RATE=48000` would build through
`rave.RAVE()` (scripts/train.py:139-159).
"""
from contextlib import contextmanager
from functools import partial

import torch.nn as nn

from . import blocks, cc, core, discriminator, pqmf, quantization
from .model import RAVE

V2_DILATIONS = [[1, 3, 9], [1, 3, 9], [1, 3, 9], [1, 3]]          # configs/v2.gin:13-18

ARCH = {
    # name: capacity, ratios, activation, adain, discriminator, update_discriminator_every, phase_1
    "v2": dict(capacity=96, ratios=[4, 4, 4, 2], activation="leaky", adain=False,     # v2.gin:12-21
               disc="v2", update_discriminator_every=4, phase_1_duration=1000000),
    "v2_small": dict(capacity=48, ratios=[4, 2, 2, 2], activation="leaky", adain=False,  # v2_small.gin:12-21
                     disc="v2", update_discriminator_every=2, phase_1_duration=1000000),
    "v3": dict(capacity=96, ratios=[4, 4, 4, 2], activation="snake", adain=True,       # v3.gin:3-13
               disc="descript", update_discriminator_every=4, phase_1_duration=1000000),
    # discrete.gin:13-49 (EnCodec-style RVQ head; generator latent = 128 + 128 noise channels)
    "discrete": dict(capacity=96, ratios=[4, 4, 2, 2], activation="leaky", adain=False, disc="v2",
                     update_discriminator_every=4, phase_1_duration=200000, discrete=True,
                     noise_augmentation=128, log_epsilon=1.0, num_skipped_features=0),
    # `--config v2 --config spectral_discriminator`: v2 with the MPD replaced by the multi-scale spectral discriminator
    "v2_spectral": dict(capacity=96, ratios=[4, 4, 4, 2], activation="leaky", adain=False,
                        disc="v2_spectral", update_discriminator_every=4, phase_1_duration=1000000),
    # v2_nopqmf.gin on top of v1.gin: the generator writes the waveform itself (output_mode "raw", v2_nopqmf.gin:106;
    # GeneratorV2.data_size unbound -> 64 -> 2 output conv with amplitude modulation, v2_nopqmf.gin:58-64) with its own
    # ratios [8, 8, 8, 4] (v2_nopqmf.gin:60); the encoder keeps its PQMF input and ratios [4, 4, 4, 2] (v2_nopqmf.gin:45-52);
    # CombineDiscriminators[MPD, MSD] at CAPACITY = 64 (v2_nopqmf.gin:22, 84-89; v1.gin:75-88)
    "v2_nopqmf": dict(capacity=64, ratios=[4, 4, 4, 2], gen_ratios=[8, 8, 8, 4], raw_output=True,   # v2_nopqmf.gin:15-23
                      activation="leaky", adain=False, disc="v2",
                      update_discriminator_every=4, phase_1_duration=1000000),              # v2_nopqmf.gin:95-106
    # `--config v2 --config hybrid`: mel-spectrogram encoder input and a GRU generator head (HYBRID below)
    "v2_hybrid": dict(capacity=96, ratios=[4, 4, 4, 2], activation="leaky", adain=False, disc="v2",
                      update_discriminator_every=4, phase_1_duration=1000000, hybrid=True),
    # `--config v2 --config wasserstein`: Wasserstein auto-encoder (MMD regulariser), 16 latent channels extended by 128
    # noise channels for the generator; gin replaces v2.gin's weight dict (feature_matching 20 stays, from
    # rave/model.py's defaults).  configs/wasserstein.gin also binds BetaWarmupCallback(100, 100, 1): beta_factor = 100.
    "v2_wasserstein": dict(capacity=96, ratios=[4, 4, 4, 2], activation="leaky", adain=False, disc="v2",
                           update_discriminator_every=4, phase_1_duration=200000, regularization="wasserstein",
                           latent_size=16, n_out=1, noise_augmentation=128,
                           weights={"fullband_spectral_distance": 2, "multiband_spectral_distance": 2,
                                    "adversarial": 2}),
    # `--config v2 --config spherical`: latent projected on the unit sphere, no regulariser; the encoder keeps training
    # in phase 2 (SphericalEncoder.set_warmed_up does nothing)
    "v2_spherical": dict(capacity=96, ratios=[4, 4, 4, 2], activation="leaky", adain=False, disc="v2",
                         update_discriminator_every=4, phase_1_duration=200000, regularization="spherical",
                         latent_size=16, n_out=1),
}

# configs/hybrid.gin on top of any v2-style configuration: EncoderV2(data_size=N_MELS, ratios=[2, 2, 2], dilations=[1])
# fed log1p(MelSpectrogram(n_fft=2048, hop=256, normalized=True, n_mels=128)) (input_mode "mel"), and
# GeneratorV2.recurrent_layer = GRU(LATENT_SIZE, num_layers=2)
HYBRID = dict(n_mels=128, n_fft=2048, hop_length=256, encoder_ratios=[2, 2, 2], encoder_dilations=[1],
              num_gru_layers=2)


def _hybrid_parts(hybrid):
    """(encoder overrides, generator recurrent_layer) of the hybrid switch."""
    if not hybrid:
        return None, None
    enc = dict(data_size=HYBRID["n_mels"], ratios=HYBRID["encoder_ratios"], dilations=HYBRID["encoder_dilations"])
    return enc, partial(blocks.GRU, num_layers=HYBRID["num_gru_layers"])


def mel_spectrogram(sampling_rate):
    """The hybrid configuration's transforms.MelSpectrogram binding (configs/hybrid.gin:19-25)."""
    return core.MelSpectrogram(sampling_rate, n_fft=HYBRID["n_fft"], win_length=HYBRID["n_fft"],
                               hop_length=HYBRID["hop_length"], normalized=True, n_mels=HYBRID["n_mels"])


def _activation_factory(kind):
    if kind == "snake":
        return lambda dim: blocks.Snake(dim)          # configs/snake.gin:5-23
    return lambda dim: nn.LeakyReLU(.2)


def make_autoencoder(name="v2", capacity=None, latent_size=128, n_band=16, n_channels=1,
                     padding_mode="centered", ratios=None, activation=None, adain=None, with_noise=False,
                     gen_ratios=None, hybrid=None):
    """(pqmf, encoder, decoder) factories -> constructed modules for one architecture.  `gen_ratios`: the generator's
    own ratios (v2_nopqmf; defaults to the configuration's, else `ratios`).  `hybrid` (default: the configuration's):
    mel-input encoder (its input is core.MelSpectrogram.encode_log1p of the waveform) and GRU generator head."""
    a = ARCH[name]
    hyb_enc, recurrent = _hybrid_parts(a.get("hybrid", False) if hybrid is None else hybrid)
    capacity = capacity or a["capacity"]
    ratios = ratios or a["ratios"]
    gen_ratios = gen_ratios or a.get("gen_ratios") or ratios
    enc_kw = {**dict(data_size=n_band, ratios=ratios, dilations=V2_DILATIONS), **(hyb_enc or {})}
    raw = a.get("raw_output", False)
    act = _activation_factory(activation or a["activation"])
    use_adain = a["adain"] if adain is None else adain
    adain_f = (lambda dim: blocks.AdaptiveInstanceNormalization(dim)) if use_adain else None
    with cc.configure(conv_bias=False, padding_mode=padding_mode):       # v1.gin:33-34, causal.gin:5
        pq = pqmf.CachedPQMF(attenuation=100, n_band=n_band, n_channels=n_channels)  # v1.gin:37-39
        enc = blocks.VariationalEncoder(                                  # v2.gin:30-40
            partial(blocks.EncoderV2, capacity=capacity, latent_size=latent_size, n_out=2, kernel_size=3,
                    activation=act, adain=adain_f, **enc_kw),
            n_channels=n_channels)
        noise = None
        if name == "v2_small" and with_noise:                                  # v2_small.gin:42-57
            noise = partial(blocks.NoiseGeneratorV2, hidden_size=64, data_size=n_band, ratios=[2, 2, 2],
                            noise_bands=32, activation=act)
        dec = blocks.GeneratorV2(data_size=None if raw else n_band, capacity=capacity, ratios=gen_ratios,  # v2.gin:43-50
                                 latent_size=latent_size, kernel_size=3, dilations=V2_DILATIONS,
                                 amplitude_modulation=True, activation=act, adain=adain_f,
                                 n_channels=n_channels, noise_module=noise, recurrent_layer=recurrent)
    return pq, enc, dec


def make_discriminator_v2(capacity=96, n_channels=1):
    """CombineDiscriminators[MPD(2,3,5,7,11), MSD(3)] (configs/v2.gin:53-75, v1.gin:75-88)."""
    periods_net = partial(discriminator.ConvNet, out_size=1, capacity=capacity, n_layers=4, stride=4,
                          conv=nn.Conv2d, kernel_size=(5, 1))
    scales_net = partial(discriminator.ConvNet, out_size=1, capacity=capacity, n_layers=4, stride=4,
                         conv=nn.Conv1d, kernel_size=15)
    return discriminator.CombineDiscriminators([
        partial(discriminator.MultiPeriodDiscriminator, periods=[2, 3, 5, 7, 11], convnet=periods_net),
        partial(discriminator.MultiScaleDiscriminator, n_discriminators=3, convnet=scales_net),
    ], n_channels=n_channels)


def make_discriminator_v2_spectral(capacity=96, n_channels=1, spectral_capacity=32,
                                   scales=(4096, 2048, 1024, 512, 256)):
    """CombineDiscriminators[MSD(3), MultiScaleSpectralDiscriminator(EncodecConvNet)] (configs/spectral_discriminator.gin:
    6-17 on top of configs/v2.gin)."""
    scales_net = partial(discriminator.ConvNet, out_size=1, capacity=capacity, n_layers=4, stride=4,
                         conv=nn.Conv1d, kernel_size=15)
    return discriminator.CombineDiscriminators([
        partial(discriminator.MultiScaleDiscriminator, n_discriminators=3, convnet=scales_net),
        partial(discriminator.MultiScaleSpectralDiscriminator, scales=list(scales),
                convnet=partial(discriminator.EncodecConvNet, capacity=spectral_capacity)),
    ], n_channels=n_channels)


def build_rave(name="v2", sampling_rate=48000, capacity=None, latent_size=None, n_channels=1,
               padding_mode="centered", phase_1_duration=None, disc_capacity=None, ratios=None, spectral_capacity=32,
               hybrid=None):
    """The full `RAVE` model of a named configuration (`spectral_capacity`: EncodecConvNet capacity of "v2_spectral",
    configs/spectral_discriminator.gin:11).  `hybrid=True` adds `--config hybrid` to any configuration with a
    VariationalEncoder (default: the configuration's own, True for "v2_hybrid").  `latent_size` defaults to the
    configuration's (128 unless it sets one)."""
    a = ARCH[name]
    hyb_enc, recurrent = _hybrid_parts(a.get("hybrid", False) if hybrid is None else hybrid)
    if hyb_enc is not None and (a.get("discrete") or a.get("regularization")):
        raise NotImplementedError("hybrid: the mel-input encoder is built for VariationalEncoder configurations")
    latent_size = latent_size if latent_size is not None else a.get("latent_size", 128)
    cap = capacity or a["capacity"]
    act = _activation_factory(a["activation"])
    adain_f = (lambda dim: blocks.AdaptiveInstanceNormalization(dim)) if a["adain"] else None
    rat = ratios or a["ratios"]
    gen_rat = a.get("gen_ratios") or rat
    raw = a.get("raw_output", False)
    stft = partial(core.MultiScaleSTFT, scales=[2048, 1024, 512, 256, 128],        # v1.gin:21-28
                   sample_rate=sampling_rate, magnitude=True)
    distance = partial(core.AudioDistanceV1, multiscale_stft=stft, log_epsilon=a.get("log_epsilon", 1e-7))
    if a["disc"] == "v2":
        disc = lambda n_channels=1: make_discriminator_v2(disc_capacity or cap, n_channels)
    elif a["disc"] == "v2_spectral":
        disc = lambda n_channels=1: make_discriminator_v2_spectral(disc_capacity or cap, n_channels, spectral_capacity)
    else:
        from .descript_discriminator import DescriptDiscriminator
        disc = lambda n_channels=1: DescriptDiscriminator(n_channels=n_channels)
    noise_aug = a.get("noise_augmentation", 0)
    if a.get("discrete"):
        encoder = partial(blocks.DiscreteEncoder,                                # discrete.gin:26-38
                          encoder_cls=partial(blocks.EncoderV2, data_size=16, capacity=cap, ratios=rat,
                                              latent_size=latent_size, n_out=1, kernel_size=3,
                                              dilations=V2_DILATIONS, activation=act, adain=adain_f),
                          vq_cls=partial(quantization.ResidualVectorQuantization, num_quantizers=16,
                                         dim=latent_size, codebook_size=1024),
                          num_quantizers=16, noise_augmentation=noise_aug)
    else:
        enc_kw = {**dict(data_size=16, ratios=rat, dilations=V2_DILATIONS), **(hyb_enc or {})}
        enc_cls = partial(blocks.EncoderV2, capacity=cap, latent_size=latent_size, n_out=a.get("n_out", 2),
                          kernel_size=3, activation=act, adain=adain_f, **enc_kw)
        reg = a.get("regularization")
        if reg == "wasserstein":                                                 # wasserstein.gin:10-16
            encoder = partial(blocks.WasserteinEncoder, encoder_cls=enc_cls, noise_augmentation=noise_aug)
        elif reg == "spherical":                                                 # spherical.gin:8-13
            encoder = partial(blocks.SphericalEncoder, encoder_cls=enc_cls)
        else:
            encoder = partial(blocks.VariationalEncoder, enc_cls)
    noise = None
    if name == "v2_small":                                                       # v2_small.gin:42-57
        noise = partial(blocks.NoiseGeneratorV2, hidden_size=64, data_size=16, ratios=[2, 2, 2],
                        noise_bands=32, activation=act)
    with cc.configure(conv_bias=False, padding_mode=padding_mode):
        model = RAVE(
            latent_size=latent_size, sampling_rate=sampling_rate,
            pqmf=partial(pqmf.CachedPQMF, attenuation=100, n_band=16),
            encoder=encoder,
            decoder=partial(blocks.GeneratorV2, data_size=None if raw else 16, capacity=cap, ratios=gen_rat,
                            latent_size=core.get_augmented_latent_size(latent_size, noise_aug), kernel_size=3,
                            dilations=V2_DILATIONS, amplitude_modulation=True, activation=act, adain=adain_f,
                            noise_module=noise, recurrent_layer=recurrent),
            discriminator=disc,
            phase_1_duration=phase_1_duration if phase_1_duration is not None else a["phase_1_duration"],
            gan_loss=core.hinge_gan, valid_signal_crop=True,                  # v2.gin:81-83
            feature_matching_fun=partial(core.mean_difference, norm="L1", relative=True),
            num_skipped_features=a.get("num_skipped_features", 1),
            audio_distance=distance, multiband_audio_distance=distance,
            weights=a.get("weights", {"feature_matching": 20}),               # v2.gin:87-89
            update_discriminator_every=a["update_discriminator_every"], n_channels=n_channels,
            output_mode="raw" if raw else "pqmf",
            spectrogram=mel_spectrogram(sampling_rate) if hyb_enc is not None else None,
            input_mode="mel" if hyb_enc is not None else "pqmf")
    return model


# configs/prior/prior_v1.gin (scripts/train_prior.py's default prior configuration)
PRIOR_V1 = dict(resolution=32, res_size=512, skp_size=256, kernel_size=3, cycle_size=4, n_layers=10)


def build_prior(rave_model, latent_size=None, fidelity=None, **overrides):
    """`VariationalPrior(pretrained_vae=rave_model)` at the prior_v1.gin bindings (`sr` = the RAVE's sampling rate), as
    `scripts/train_prior.py` builds it; `overrides` rebind any of them.  One of latent_size / fidelity is required."""
    from .prior import VariationalPrior
    kw = dict(PRIOR_V1, sr=rave_model.sr)
    kw.update(overrides)
    return VariationalPrior(pretrained_vae=rave_model, latent_size=latent_size, fidelity=fidelity, **kw)

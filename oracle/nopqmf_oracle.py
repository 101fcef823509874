"""TEST INFRASTRUCTURE -- restatement of the v2_nopqmf configuration (rave/configs/v2_nopqmf.gin on top of v1.gin) in
plain torch, built on oracle/rave_oracle.py: the raw-waveform generator (GeneratorV2 with `data_size` unbound: the last
conv writes 2 channels, waveform + amplitude, for one mono output) and the raw-output training step, whose multiband
target comes from PQMF ANALYSIS of the generator's output (rave/model.py:307-312).  Pinned against the unmodified
reference by oracle/make_golden_nopqmf.py (tests/golden/*nopqmf*.pt)."""
import torch
from torch import Tensor

from oracle import rave_oracle as O
from oracle.spectral_oracle import sample, seeded_params, step_batch, step_eps  # noqa: F401  (re-exported)

GEN_RATIOS = (8, 8, 8, 4)            # v2_nopqmf.gin:60
ENC_RATIOS = (4, 4, 4, 2)            # v2_nopqmf.gin:48
CAPACITY = 64                        # v2_nopqmf.gin:22


def generator_config(cfg: O.ArchConfig, gen_ratios=GEN_RATIOS) -> O.ArchConfig:
    """The generator-side ArchConfig: O.generator_v2 reads cfg.ratios, which are the encoder's in cfg."""
    return O.ArchConfig(capacity=cfg.capacity, ratios=tuple(gen_ratios), latent_size=cfg.latent_size, n_out=cfg.n_out,
                        kernel_size=cfg.kernel_size, dilations=cfg.dilations, n_band=cfg.n_band,
                        n_channels=cfg.n_channels, activation=cfg.activation, adain=cfg.adain,
                        amplitude_modulation=cfg.amplitude_modulation, pad_mode=cfg.pad_mode, keep_dim=cfg.keep_dim,
                        generator_latent=cfg.generator_latent)


def generator_raw(z: Tensor, sd, prefix: str, gcfg: O.ArchConfig, taps=None) -> Tensor:
    """GeneratorV2 with data_size=None, amplitude_modulation=True (rave/blocks.py:599-714): [B, latent, Lz] ->
    [B, 1, Lz * prod(ratios)]; the output conv's weights carry the 2 channels."""
    return O.generator_v2(z, sd, prefix, gcfg, taps)


def rave_forward_raw(x: Tensor, sd, cfg: O.ArchConfig, gcfg: O.ArchConfig, eps: Tensor, taps=None) -> Tensor:
    """RAVE.forward with output_mode "raw" (rave/model.py:267-270): PQMF analysis -> encoder -> reparametrisation
    (noise injected) -> raw generator; no PQMF synthesis."""
    x_mb = O.pqmf_encode(x, sd["pqmf.hk"], cfg.pad_mode)
    z = O.encoder_v2(x_mb, sd, "encoder.encoder.", cfg)
    zs, _ = O.reparametrize(z, eps)
    y = generator_raw(zs, sd, "decoder.", gcfg)
    if taps is not None:
        taps.update(x_mb=x_mb, z=z, zs=zs)
    return y


def train_step_losses(x: Tensor, sd, cfg: O.ArchConfig, gcfg: O.ArchConfig, eps: Tensor, receptive_field=(0, 0),
                      fm_weight: float = 20.0):
    """Phase-2 forward arithmetic of RAVE.training_step (rave/model.py:292-399) with output_mode "raw": y_multiband =
    PQMF analysis of the generator output (307-312), both crops as the reference orders them, the v2 discriminator
    (MPD + MSD).  Returns (logged loss_gen terms, loss_dis)."""
    hk = sd["pqmf.hk"]
    x_mb = O.pqmf_encode(x, hk, cfg.pad_mode)
    z = O.encoder_v2(x_mb, sd, "encoder.encoder.", cfg).detach()       # warmed up: blocks.py:743-744
    zs, reg = O.reparametrize(z, eps)
    y = generator_raw(zs, sd, "decoder.", gcfg)
    y_mb = O.pqmf_encode(y, hk, cfg.pad_mode)
    y = y[..., :x.shape[-1]]
    y_mb = y_mb[..., :x_mb.shape[-1]]
    x_mb_c, y_mb_c = x_mb, y_mb
    if receptive_field[0] + receptive_field[1]:
        x_mb_c = O.valid_signal_crop(x_mb, *receptive_field)
        y_mb_c = O.valid_signal_crop(y_mb, *receptive_field)
    fm, loss_dis, loss_adv = O.gan_losses(O.combine_discriminators_v2(torch.cat([x, y], 0), sd), 1, True)
    losses = {
        "multiband_spectral_distance": O.audio_distance_v1(x_mb_c, y_mb_c),
        "fullband_spectral_distance": O.audio_distance_v1(x, y),
        "regularization": reg,
        "feature_matching": fm_weight * fm,
        "adversarial": loss_adv,
    }
    return losses, loss_dis

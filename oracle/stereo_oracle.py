"""TEST INFRASTRUCTURE -- the phase-2 training-step arithmetic of RAVE.training_step (rave/model.py:292-399) for a
multichannel model (`n_channels` > 1, scripts/train.py --channels), v2 (MPD + MSD) or v3 (Descript discriminator), in
plain torch on top of oracle/rave_oracle.py, whose restatements already carry the channel axis (pqmf_encode /
pqmf_decode, mpd_fold, the conv stacks, the MRD's "b c f t p -> b (c p) t f", audio_distance_v1).  Pinned against the
unmodified reference by oracle/make_golden_stereo.py (tests/golden/*stereo*.pt)."""
import torch
from torch import Tensor

from oracle import rave_oracle as O
from oracle import spectral_oracle as S
from oracle.spectral_oracle import sample, step_eps  # noqa: F401  (re-exported)

N_CHANNELS = 2


def train_step_losses(x: Tensor, sd, cfg: O.ArchConfig, eps: Tensor, kind: str = "v2", receptive_field=(0, 0),
                      fm_weight: float = 20.0):
    """(logged loss_gen terms, loss_dis) of a phase-2 step; kind "v2" = CombineDiscriminators(MPD, MSD), "v3" =
    DescriptDiscriminator (with Snake / AdaIN in cfg)."""
    hk = sd["pqmf.hk"]
    x_mb = O.pqmf_encode(x, hk, cfg.pad_mode)
    z = O.encoder_v2(x_mb, sd, "encoder.encoder.", cfg).detach()      # warmed up: blocks.py:743-744
    zs, reg = O.reparametrize(z, eps)
    y_mb = O.generator_v2(zs, sd, "decoder.", cfg)
    y = O.pqmf_decode(y_mb, hk, cfg.n_channels, cfg.pad_mode)[..., :x.shape[-1]]
    y_mb = y_mb[..., :x_mb.shape[-1]]
    x_mb_c, y_mb_c = x_mb, y_mb
    if receptive_field[0] + receptive_field[1]:
        x_mb_c = O.valid_signal_crop(x_mb, *receptive_field)
        y_mb_c = O.valid_signal_crop(y_mb, *receptive_field)
    disc = O.combine_discriminators_v2 if kind == "v2" else O.descript_discriminator
    fm, loss_dis, loss_adv = O.gan_losses(disc(torch.cat([x, y], 0), sd), 1, True)
    losses = {
        "multiband_spectral_distance": O.audio_distance_v1(x_mb_c, y_mb_c),
        "fullband_spectral_distance": O.audio_distance_v1(x, y),
        "regularization": reg,
        "feature_matching": fm_weight * fm,
        "adversarial": loss_adv,
    }
    return losses, loss_dis


def step_batch(B: int, T: int, seed: int, n_channels: int = N_CHANNELS) -> Tensor:
    """The training-step fixture's multichannel batch [B, n_channels, T]."""
    g = torch.Generator(device="cpu").manual_seed(500 + seed)
    return (0.5 * torch.randn(B, n_channels, T, generator=g)).clamp(-1, 1)


def seeded_params(shapes, seed):
    """spectral_oracle.seeded_params at the standard deviation of PyTorch's default conv initialisation (kaiming-uniform,
    1 / sqrt(3 fan_in)), with every Snake `alpha` at its initial value 1 (rave/blocks.py Snake).  At unit gain the tiny
    Snake encoder of v3 grows its activations layer by layer and its losses reach 1e2-1e3, where float32 round-off alone
    exceeds the fixture's tolerances."""
    out = S.seeded_params(shapes, seed)
    for k in out:
        if k.endswith(".alpha"):
            out[k] = torch.ones_like(out[k])
        elif out[k].dim() > 1:
            out[k] = out[k] / 3 ** 0.5
    for k in out:
        if k.endswith("weight_g"):
            v = out[k[:-1] + "v"]
            out[k] = v.reshape(v.shape[0], -1).norm(dim=1).reshape(out[k].shape)
    return out

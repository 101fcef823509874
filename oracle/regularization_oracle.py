"""TEST INFRASTRUCTURE -- restatement of the two v2 regularisation options in plain torch, built on
oracle/rave_oracle.py: the Wasserstein auto-encoder (rave/configs/wasserstein.gin, WasserteinEncoder: MMD regulariser,
128 noise channels appended to the latent) and the spherical auto-encoder (rave/configs/spherical.gin, SphericalEncoder:
the latent projected on the unit sphere).  Pinned against the unmodified reference by
oracle/make_golden_regularization.py (tests/golden/*_v2_wasserstein_* and *_v2_spherical_*)."""
import torch
from torch import Tensor

from oracle import rave_oracle as O
from oracle.spectral_oracle import sample, seeded_params, step_batch  # noqa: F401  (re-exported)

LATENT_SIZE = 16                    # wasserstein.gin:6, spherical.gin:6
NOISE_AUGMENTATION = 128            # wasserstein.gin:7
BETA = 100.0                        # wasserstein.gin:25-28: BetaWarmupCallback(100, 100, 1)
# wasserstein.gin:20-24 replaces v2.gin's dict; feature_matching 20 comes from rave/model.py's defaults
WAE_WEIGHTS = {"fullband_spectral_distance": 2, "multiband_spectral_distance": 2, "adversarial": 2,
               "feature_matching": 20}
DEFAULT_WEIGHTS = {"feature_matching": 20}


def mean_kernel(x: Tensor, y: Tensor) -> Tensor:
    """WasserteinEncoder.compute_mean_kernel (rave/blocks.py:761-763): mean over pairs of exp(-mean_d (x - y)^2 / D)."""
    return torch.exp(-((x[:, None] - y[None]).pow(2).mean(2) / x.shape[-1])).mean()


def rows(z: Tensor) -> Tensor:
    """z [B, D, L] -> [B·L, D], row b·L + t = z[b, :, t] (rave/blocks.py:773)."""
    return z.permute(0, 2, 1).reshape(-1, z.shape[1])


def mmd_terms(z: Tensor, prior: Tensor):
    """(mean k(x, x), mean k(y, y), mean k(x, y)) of the latent rows x and the prior sample y."""
    x = rows(z)
    return mean_kernel(x, x), mean_kernel(prior, prior), mean_kernel(x, prior)


def mmd(z: Tensor, prior: Tensor) -> Tensor:
    """WasserteinEncoder.compute_mmd (rave/blocks.py:765-770)."""
    kxx, kyy, kxy = mmd_terms(z, prior)
    return kxx + kyy - 2 * kxy


def draws(B: int, D: int, L: int, seed: int, noise_augmentation: int = NOISE_AUGMENTATION):
    """The two draws WasserteinEncoder.reparametrize makes after torch.manual_seed(seed) (no earlier draw in the step):
    the prior sample randn_like of the [B·L, D] rows, then the noise randn(B, noise_augmentation, L)."""
    g = torch.Generator().manual_seed(seed)
    prior = torch.randn(B * L, D, generator=g)
    noise = torch.randn(B, noise_augmentation, L, generator=g) if noise_augmentation else None
    return prior, noise


def reparametrize(z: Tensor, kind: str, prior=None, noise=None):
    """(latent fed to the generator, regulariser) of WasserteinEncoder (rave/blocks.py:772-781) or SphericalEncoder
    (839-842)."""
    if kind == "wasserstein":
        reg = mmd(z, prior)
        if noise is not None:
            z = torch.cat([z, noise], 1)
        return z, reg
    return z / torch.norm(z, p=2, dim=1, keepdim=True), torch.zeros_like(z).mean()


def config(kind: str, capacity: int, latent_size: int = LATENT_SIZE) -> O.ArchConfig:
    """The ArchConfig of either configuration: EncoderV2.n_out = 1; the generator reads 16 + 128 channels for the WAE."""
    extra = NOISE_AUGMENTATION if kind == "wasserstein" else 0
    return O.ArchConfig(capacity=capacity, latent_size=latent_size, n_out=1, generator_latent=latent_size + extra)


def rave_forward(x: Tensor, sd, cfg: O.ArchConfig, kind: str, prior=None, noise=None, taps=None):
    """PQMF analysis -> EncoderV2 -> regulariser -> GeneratorV2 -> PQMF synthesis; returns (y, reg)."""
    hk = sd["pqmf.hk"]
    z = O.encoder_v2(O.pqmf_encode(x, hk, cfg.pad_mode), sd, "encoder.encoder.", cfg)
    zs, reg = reparametrize(z, kind, prior, noise)
    y = O.pqmf_decode(O.generator_v2(zs, sd, "decoder.", cfg), hk, cfg.n_channels, cfg.pad_mode)
    if taps is not None:
        taps.update(z=z, zs=zs)
    return y, reg


def train_step_losses(x: Tensor, sd, cfg: O.ArchConfig, kind: str, warmed_up: bool, prior=None, noise=None,
                      beta: float = BETA, receptive_field=(0, 0)):
    """Forward arithmetic of RAVE.training_step (rave/model.py:292-399) for either configuration.  Returns (logged
    loss_gen terms, loss_dis, the generator's total loss with the weights applied as train_step applies them).  The
    WAE's encoder output is detached in phase 2 (rave/blocks.py:789-790); the spherical encoder's never is."""
    weights = WAE_WEIGHTS if kind == "wasserstein" else DEFAULT_WEIGHTS
    hk = sd["pqmf.hk"]
    x_mb = O.pqmf_encode(x, hk, cfg.pad_mode)
    z = O.encoder_v2(x_mb, sd, "encoder.encoder.", cfg)
    if warmed_up and kind == "wasserstein":
        z = z.detach()
    zs, reg = reparametrize(z, kind, prior, noise)
    y_mb = O.generator_v2(zs, sd, "decoder.", cfg)
    y = O.pqmf_decode(y_mb, hk, cfg.n_channels, cfg.pad_mode)[..., :x.shape[-1]]
    y_mb = y_mb[..., :x_mb.shape[-1]]
    x_mb_c, y_mb_c = x_mb, y_mb
    if receptive_field[0] + receptive_field[1]:
        x_mb_c = O.valid_signal_crop(x_mb, *receptive_field)
        y_mb_c = O.valid_signal_crop(y_mb, *receptive_field)
    losses = {
        "multiband_spectral_distance": O.audio_distance_v1(x_mb_c, y_mb_c),
        "fullband_spectral_distance": O.audio_distance_v1(x, y),
        "regularization": reg * beta,
    }
    loss_dis = torch.zeros(())
    if warmed_up:
        fm, loss_dis, loss_adv = O.gan_losses(O.combine_discriminators_v2(torch.cat([x, y], 0), sd), 1, True)
        losses["feature_matching"] = weights["feature_matching"] * fm
        losses["adversarial"] = weights.get("adversarial", 1) * loss_adv
    total = sum(v * weights.get(k, 1) for k, v in losses.items())
    return losses, loss_dis, total

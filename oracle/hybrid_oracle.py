"""TEST INFRASTRUCTURE -- restatement of the hybrid configuration (rave/configs/hybrid.gin on top of v2.gin) in plain
torch, built on oracle/rave_oracle.py: the mel front end of RAVE._mel_encode (rave/model.py:238-242 with
torchaudio.transforms.MelSpectrogram(normalized=True)), the GRU generator head (rave/blocks.py:295-319, nn.GRU's
documented cell) and the training-step arithmetic in mel mode.  Pinned against the unmodified reference by
oracle/make_golden_hybrid.py (tests/golden/*hybrid*.pt)."""
import torch
import torch.nn.functional as F
from torch import Tensor

from oracle import rave_oracle as O
from oracle.spectral_oracle import sample, seeded_params, step_batch, step_eps  # noqa: F401  (re-exported)

N_FFT, HOP, N_MELS = 2048, 256, 128              # hybrid.gin:10-12
ENC_RATIOS, ENC_DILATIONS = (2, 2, 2), (1,)      # hybrid.gin:13, 18-20
NUM_GRU_LAYERS = 2                               # hybrid.gin:14


def encoder_config(cfg: O.ArchConfig) -> O.ArchConfig:
    """The encoder side of hybrid.gin: EncoderV2(data_size=N_MELS, ratios=[2, 2, 2], dilations=[1])."""
    return O.ArchConfig(capacity=cfg.capacity, ratios=ENC_RATIOS, latent_size=cfg.latent_size, n_out=cfg.n_out,
                        kernel_size=cfg.kernel_size, dilations=ENC_DILATIONS, n_band=N_MELS, n_channels=cfg.n_channels,
                        activation=cfg.activation, adain=cfg.adain, pad_mode=cfg.pad_mode)


def mel_log1p(x: Tensor, window: Tensor, fb: Tensor, n_fft: int = N_FFT, hop: int = HOP) -> Tensor:
    """log1p(MelSpectrogram(x)[..., :-1]) reshaped to [B, C * n_mels, frames - 1] (rave/model.py:238-242).
    torchaudio.functional.spectrogram: centred reflect-padded frames, periodic hann window, |X|^2 / sum(w^2)
    (normalized=True, power 2); MelScale: spec^T @ fb."""
    B, C, T = x.shape
    xp = F.pad(x.reshape(B * C, 1, T), (n_fft // 2, n_fft // 2), mode="reflect").reshape(B * C, -1)
    frames = xp.unfold(-1, n_fft, hop) * window                      # [N, F, n_fft]
    X = torch.fft.rfft(frames)
    spec = (X.real ** 2 + X.imag ** 2) / window.pow(2).sum()
    mel = spec @ fb                                                  # [N, F, n_mels]
    mel = mel.transpose(1, 2)[..., :-1]
    return torch.log1p(mel).reshape(B, C * fb.shape[1], -1)


def gru(x: Tensor, sd, prefix: str, num_layers: int = NUM_GRU_LAYERS) -> Tensor:
    """blocks.GRU.forward (rave/blocks.py:308-313): nn.GRU(batch_first=True) over the time axis of [B, H, T], h0 = 0,
    the cell of torch.nn.GRU's documentation:
        r = sigmoid(W_ir x + b_ir + W_hr h + b_hr)    z = sigmoid(W_iz x + b_iz + W_hz h + b_hz)
        n = tanh(W_in x + b_in + r * (W_hn h + b_hn))  h' = (1 - z) * n + z * h"""
    h_seq = x.transpose(1, 2)                                        # [B, T, I]
    for l in range(num_layers):
        w_ih, w_hh = sd[f"{prefix}gru.weight_ih_l{l}"], sd[f"{prefix}gru.weight_hh_l{l}"]
        b_ih, b_hh = sd[f"{prefix}gru.bias_ih_l{l}"], sd[f"{prefix}gru.bias_hh_l{l}"]
        H = w_hh.shape[1]
        gi_all = h_seq @ w_ih.t() + b_ih
        h = h_seq.new_zeros(h_seq.shape[0], H)
        outs = []
        for t in range(h_seq.shape[1]):
            gi = gi_all[:, t]
            gh = h @ w_hh.t() + b_hh
            r = torch.sigmoid(gi[:, :H] + gh[:, :H])
            z = torch.sigmoid(gi[:, H:2 * H] + gh[:, H:2 * H])
            n = torch.tanh(gi[:, 2 * H:] + r * gh[:, 2 * H:])
            h = (1 - z) * n + z * h
            outs.append(h)
        h_seq = torch.stack(outs, 1)
    return h_seq.transpose(1, 2)


def _generator_sd(sd, prefix: str = "decoder."):
    """GeneratorV2 with recurrent_layer: the GRU is net.0, every later index shifted by one (rave/blocks.py:626-629);
    the view O.generator_v2 reads (indices back to the recurrent-free numbering)."""
    out = {}
    p = prefix + "net."
    for k, v in sd.items():
        if k.startswith(p):
            i, rest = k[len(p):].split(".", 1)
            if int(i) > 0:
                out[f"{p}{int(i) - 1}.{rest}"] = v
    return out


def generator_hybrid(z: Tensor, sd, gcfg: O.ArchConfig, prefix: str = "decoder.") -> Tensor:
    return O.generator_v2(gru(z, sd, prefix + "net.0."), _generator_sd(sd, prefix), prefix, gcfg)


def rave_forward_hybrid(x: Tensor, sd, cfg: O.ArchConfig, eps: Tensor, taps=None) -> Tensor:
    """RAVE.forward in mel mode with the GRU head: mel front end -> encoder -> reparametrisation (noise injected) ->
    GRU -> generator -> PQMF synthesis."""
    ecfg = encoder_config(cfg)
    x_mel = mel_log1p(x, sd["spectrogram.spectrogram.window"], sd["spectrogram.mel_scale.fb"])
    z = O.encoder_v2(x_mel, sd, "encoder.encoder.", ecfg)
    zs, _ = O.reparametrize(z, eps)
    y = generator_hybrid(zs, sd, cfg)
    if taps is not None:
        taps.update(x_mel=x_mel, z=z, zs=zs)
    return O.pqmf_decode(y, sd["pqmf.hk"], cfg.n_channels, cfg.pad_mode)


def train_step_losses(x: Tensor, sd, cfg: O.ArchConfig, eps: Tensor, warmed_up: bool, receptive_field=(0, 0),
                      fm_weight: float = 20.0):
    """Forward arithmetic of RAVE.training_step (rave/model.py:292-399) in mel mode with the multiband target taken as
    the PQMF analysis of the waveform (quirk D9, SURVEY.md).  Returns (logged loss_gen terms, loss_dis or None)."""
    hk = sd["pqmf.hk"]
    ecfg = encoder_config(cfg)
    x_mel = mel_log1p(x, sd["spectrogram.spectrogram.window"], sd["spectrogram.mel_scale.fb"])
    z = O.encoder_v2(x_mel, sd, "encoder.encoder.", ecfg)
    if warmed_up:
        z = z.detach()                                              # rave/blocks.py:743-744
    x_mb = O.pqmf_encode(x, hk, cfg.pad_mode)
    zs, reg = O.reparametrize(z, eps)
    y_mb = generator_hybrid(zs, sd, cfg)
    y = O.pqmf_decode(y_mb, hk, cfg.n_channels, cfg.pad_mode)[..., :x.shape[-1]]
    y_mb = y_mb[..., :x_mb.shape[-1]]
    x_mb_c, y_mb_c = x_mb, y_mb
    if receptive_field[0] + receptive_field[1]:
        x_mb_c = O.valid_signal_crop(x_mb, *receptive_field)
        y_mb_c = O.valid_signal_crop(y_mb, *receptive_field)
    losses = {
        "multiband_spectral_distance": O.audio_distance_v1(x_mb_c, y_mb_c),
        "fullband_spectral_distance": O.audio_distance_v1(x, y),
        "regularization": reg,
    }
    if not warmed_up:
        return losses, None
    fm, loss_dis, loss_adv = O.gan_losses(O.combine_discriminators_v2(torch.cat([x, y], 0), sd), 1, True)
    losses.update(feature_matching=fm_weight * fm, adversarial=loss_adv)
    return losses, loss_dis


# ----------------------------------------------------------------------------------
# compact fixture forms (tests/golden/*hybrid*.pt, mel_filterbanks.pt)
# ----------------------------------------------------------------------------------

def pack_filterbank(fb: Tensor) -> dict:
    """The banded filter bank as its nonzero entries: (index [2, nnz] int32, value [nnz], shape)."""
    nz = (fb != 0).nonzero().t()
    return dict(index=nz.to(torch.int32), value=fb[nz[0], nz[1]].clone(), shape=tuple(fb.shape))


def dense_filterbank(packed: dict) -> Tensor:
    fb = torch.zeros(packed["shape"], dtype=packed["value"].dtype)
    idx = packed["index"].long()
    fb[idx[0], idx[1]] = packed["value"]
    return fb


GRAD_SAMPLE_PER_TENSOR = 2048


def grad_record(g: Tensor, seed: int):
    """A gradient as stored in a fixture: the whole tensor when small, else (indices, values) of a seeded sample."""
    flat = g.detach().reshape(-1)
    if flat.numel() <= GRAD_SAMPLE_PER_TENSOR:
        return flat.clone()
    idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(seed))[:GRAD_SAMPLE_PER_TENSOR]
    idx = idx.sort().values
    return (idx.to(torch.int32), flat[idx].clone())


def grad_pair(g: Tensor, rec):
    """(this gradient at the recorded entries, the recorded values)."""
    flat = g.detach().reshape(-1).cpu()
    if torch.is_tensor(rec):
        return flat, rec
    return flat[rec[0].long()], rec[1]


def autoencoder_state(fx: dict, fb: Tensor) -> dict:
    """The tiny autoencoder's state_dict from its fixture: seeded parameters, the stored buffers and the 48 kHz filter
    bank (torchaudio's, from mel_filterbanks.pt)."""
    sd = dict(fx["buffers"])
    sd.update(seeded_params(fx["param_shapes"], fx["param_seed"]))
    sd["spectrogram.mel_scale.fb"] = fb
    return sd

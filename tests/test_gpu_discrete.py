"""GPU: the `discrete` configuration (BASELINE config 5: EnCodec-style RVQ head, causal padding) on the device --
DiscreteEncoder + ResidualVectorQuantization against the same modules on CPU (bit-exact on CPU against the reference:
tests/test_quantization_cpu.py), the causal encoder / generator chains of the wgmma engine against the oracle, and the
whole training step of the configuration."""
import pytest
import torch
import torch.nn as nn

from oracle import rave_oracle as O
from tests.conftest import rel_l2

pytestmark = pytest.mark.gpu


def _trained_rvq(dim=32, codes=64, nq=4, seed=0):
    """An RVQ whose codebooks went through k-means init + a few EMA steps ON CPU (deterministic, reference-exact)."""
    from rave_b200 import quantization as Q
    torch.manual_seed(seed)
    rvq = Q.ResidualVectorQuantization(num_quantizers=nq, dim=dim, codebook_size=codes)
    rvq.train()
    for step in range(3):
        rvq(torch.randn(6, dim, 50) * (1 + 0.3 * step))
    return rvq


def test_rvq_device_matches_cpu():
    """Index work must agree: the device picks the same codes as the CPU wherever the two best codes are separated by
    more than fp32 rounding of the distance (|d1 - d2| > 1e-4 |d1|), and then the quantised tensors agree to 1e-6."""
    import copy
    rvq = _trained_rvq()
    rvq.eval()
    x = torch.randn(5, 32, 77, generator=torch.Generator().manual_seed(9))
    idx_c = rvq.encode(x)
    q_c, loss_c, idx_c2 = rvq(x)
    assert torch.equal(idx_c, idx_c2)
    dev = copy.deepcopy(rvq).cuda()
    idx_g = dev.encode(x.cuda())
    q_g, loss_g, _ = dev(x.cuda())
    assert idx_g.dtype == torch.int64 and idx_g.shape == idx_c.shape
    same = idx_g.cpu() == idx_c
    # every disagreement must be a numerical tie of the first stage that differs
    residual = x.clone()
    for qi, vq in enumerate(rvq.layers):
        rows = residual.permute(0, 2, 1).reshape(-1, 32)
        d = torch.cdist(rows.double(), vq.codebook.double()) ** 2
        best2 = d.topk(2, largest=False).values
        tie = ((best2[:, 1] - best2[:, 0]) <= 1e-4 * best2[:, 0].abs().clamp_min(1e-12)).reshape(5, 77)
        bad = ~same[:, qi] & ~tie
        assert not bad.any(), (qi, int(bad.sum()))
        if not same[:, qi].all():
            break                                   # later stages quantise different residuals at the tied rows
        residual = residual - vq.decode(idx_c[:, qi])
    if same.all():
        assert rel_l2(q_g, q_c) < 1e-6
        assert abs(float(loss_g) - float(loss_c)) < 1e-6


def test_rvq_training_step_on_device_updates_buffers_like_cpu():
    """One EMA update (training mode) from identical state and input: same indices (modulo exact ties), same
    cluster_size / embed_avg / embed buffers to fp32 rounding; dead-code revival needs no random draw here (all codes
    alive)."""
    import copy
    rvq = _trained_rvq(codes=8, nq=2, seed=1)
    for vq in rvq.layers:
        vq._codebook.threshold_ema_dead_code = 0
    rvq.train()
    dev = copy.deepcopy(rvq).cuda()
    x = torch.randn(6, 32, 64, generator=torch.Generator().manual_seed(4))
    q_c, l_c, i_c = rvq(x)
    q_g, l_g, i_g = dev(x.cuda())
    if torch.equal(i_c, i_g.cpu()):
        for (k, a), b in zip(rvq.state_dict().items(), dev.state_dict().values()):
            assert rel_l2(b, a) < 1e-5 or float((b.cpu() - a).abs().max()) < 1e-6, k
        assert rel_l2(q_g, q_c) < 1e-6


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_discrete_causal_autoencoder_vs_oracle(precision):
    """configs/discrete.gin + causal.gin: EncoderV2(n_out=1) -> DiscreteEncoder (RVQ bypassed: quirk D3, `enabled` is
    never switched on by the reference's training code) -> GeneratorV2 with 128 noise channels (injected), causal
    padding everywhere.  Tiny capacity, ratios [4,4,2,2]."""
    import rave_b200
    from rave_b200 import configs
    from rave_b200.model import _pqmf_decode, _pqmf_encode
    torch.manual_seed(2)
    m = configs.build_rave("discrete", capacity=16, latent_size=16, disc_capacity=8, padding_mode="causal")
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    cfg = O.ArchConfig(capacity=16, latent_size=16, ratios=(4, 4, 2, 2), n_out=1, pad_mode="causal",
                       generator_latent=16 + 128)
    B, T = 2, 16384
    x = (0.5 * torch.randn(B, 1, T, generator=torch.Generator().manual_seed(3))).clamp(-1, 1)
    Lz = T // 16 // 64
    noise = torch.randn(B, 128, Lz, generator=torch.Generator().manual_seed(8))     # NOISE_AUGMENTATION = 128
    hk = sd["pqmf.hk"]
    x_mb = O.pqmf_encode(x, hk, "causal")
    z_o = O.encoder_v2(x_mb, sd, "encoder.encoder.", cfg)
    y_mb_o = O.generator_v2(torch.cat([z_o, noise], 1), sd, "decoder.", cfg)
    y_o = O.pqmf_decode(y_mb_o, hk, 1, "causal")
    m.cuda().train()
    rave_b200.set_precision(precision)
    try:
        with torch.no_grad():
            z = m.encoder(_pqmf_encode(m.pqmf, x.cuda()))
            y = _pqmf_decode(m.pqmf, m.decoder(torch.cat([z, noise.cuda()], 1)), batch_size=x.shape[:-2], n_channels=1)
    finally:
        rave_b200.set_precision("fp32")
    tol = 1e-4 if precision == "fp32" else 3e-2
    assert z.shape == z_o.shape and y.shape == y_o.shape
    assert rel_l2(z, z_o) < tol and rel_l2(y, y_o) < tol, (rel_l2(z, z_o), rel_l2(y, y_o))


def test_discrete_training_steps_run_in_bf16_and_graphs():
    """Config 5 end to end: phase-1 / phase-2 steps of the discrete + causal model on the engine, eager and replayed from
    CUDA graphs (no host sync on the `enabled` / `warmed_up` buffers)."""
    import rave_b200
    from rave_b200 import configs
    from rave_b200.graphs import GraphedTrainer
    torch.manual_seed(0)
    m = configs.build_rave("discrete", capacity=16, latent_size=16, disc_capacity=8, padding_mode="causal").cuda().train()
    x = (0.5 * torch.randn(2, 1, 65536, device="cuda")).clamp(-1, 1)
    rave_b200.set_precision("bf16")
    try:
        logs = m.training_step(x, 1)
        assert torch.isfinite(logs["fullband_spectral_distance"])
        m.warmed_up = True
        for i in range(2):
            logs = m.training_step(x, i)
        for k in ("loss_dis", "feature_matching", "adversarial"):
            assert torch.isfinite(logs[k]), k
        tr = GraphedTrainer(m, x, warmup_steps=1)
        for i in range(4):
            logs = tr.step(x, i)
        torch.cuda.synchronize()
        assert torch.isfinite(logs["fullband_spectral_distance"]) and torch.isfinite(logs["feature_matching"])
    finally:
        rave_b200.set_precision("fp32")

"""GPU: the v2_nopqmf configuration (raw-waveform generator, rave/configs/v2_nopqmf.gin) -- the fused dilated unit at
C = 64 / 128 / 256 (weight-stationary and batched-tile paths), the r = 8 transposed conv on the wgmma engine, the fp32
and bf16 models against the reference's fixtures and the oracle, both training steps, and CUDA-graph replays."""
import copy
import math
import os

import pytest
import torch

from oracle import nopqmf_oracle as N
from oracle import rave_oracle as O
from tests.conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu


def load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def cos(a, b):
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    return float(a @ b / (a.norm() * b.norm()).clamp_min(1e-30))


# (B, L): L >= 128 with one batch per tile runs the weight-stationary kernel at C = 64; L < 128 packs several batches
# into one 128-row tile (the batched-tile path of dilated_unit_tc_kernel)
UNIT_CASES = [(C, B, L, dil, keep_a1) for C in (64, 128, 256) for (B, L) in ((2, 1000), (3, 40))
              for dil in (1, 3, 9) for keep_a1 in (False, True)]


@pytest.mark.parametrize("case", UNIT_CASES)
def test_fused_unit_narrow_widths_vs_two_launches_and_oracle(case):
    """rave_dilated_unit_tc_fwd at the widths of the raw-waveform generator against the two per-layer launches it
    replaces (<= 1e-6) and the fp32 oracle of Residual(DilatedUnit) (bf16 tolerance)."""
    from rave_b200 import ops
    C, B, L, dil, keep_a1 = case
    assert ops.dilated_unit_tc_supported(C, L)
    g = torch.Generator().manual_seed(1000 * C + 10 * dil + L)
    x = torch.randn(B, C, L, generator=g)
    w3 = torch.randn(C, C, 3, generator=g) / (3 * C) ** 0.5
    w1 = torch.randn(C, C, 1, generator=g) / C ** 0.5
    pad_l = dil
    pad = (pad_l, 2 * dil - pad_l)
    y_ref = x + O.conv1d(O.leaky_relu(O.conv1d(O.leaky_relu(x, 0.2), w3, None, 1, dil, pad), 0.2), w1, None, 1, 1, (0, 0))
    xa, _ = ops.ncl_to_cl(x.cuda(), ops.ACT_LEAKY, 0.2)
    w3t = ops.weight_to_tapmajor_bf16(w3.cuda())
    w1t = ops.weight_to_tapmajor_bf16(w1.cuda())
    _, a1_ref = ops.conv1d_tc(xa, w3t, None, None, 1, dil, pad, ops.ACT_LEAKY, 0.2, want_f32=False, want_act=True)
    o_ref, oa_ref = ops.conv1d_tc(a1_ref, w1t, None, None, 1, 1, (0, 0), ops.ACT_LEAKY, 0.2, want_f32=True, want_act=True,
                                  res_act=xa, res_slope=0.2)
    out_f32 = torch.full((B, L, C), float("nan"), device="cuda")
    out_act = torch.empty(B, L, C, device="cuda", dtype=torch.bfloat16)
    a1, _, _ = ops.dilated_unit_tc(xa, w3t, w1t, dil, pad_l, 0.2, 0.2, ops.ACT_LEAKY, 0.2, want_a1=keep_a1,
                                   out_f32=out_f32, out_act=out_act)
    torch.cuda.synchronize()
    if keep_a1:
        assert rel_l2(a1.float(), a1_ref.float()) < 1e-6
    assert rel_l2(out_act.float(), oa_ref.float()) < 1e-6
    assert rel_l2(out_f32, o_ref) < 1e-6
    assert rel_l2(ops.cl_to_ncl(out_f32), y_ref) < 1.5e-2
    assert rel_l2(out_act.float(), O.leaky_relu(y_ref, 0.2).permute(0, 2, 1)) < 1.5e-2


def _no_fp32_convs(monkeypatch):
    from rave_b200 import ops

    def boom(*a, **k):
        raise AssertionError("fp32 conv fallback in bf16 mode")
    monkeypatch.setattr(ops, "conv1d", boom)
    monkeypatch.setattr(ops, "conv_transpose1d", boom)


def test_r8_upconv_forward_dgrad_wgrad_vs_oracle(monkeypatch):
    """conv3 -> LeakyReLU -> ConvTranspose1d(K = 16, stride 8, padding 4) as one bf16 engine chain: the phase-fused
    forward (J = 3, 24 slabs for 16 taps), the stride-8 dgrad and the wide wgrad against the fp32 oracle."""
    import rave_b200
    import torch.nn as nn
    from rave_b200 import blocks, cc
    torch.manual_seed(8)
    with cc.configure(conv_bias=False):
        seq = cc.CachedSequential(blocks.normalization(cc.Conv1d(32, 128, 3, padding=cc.get_padding(3))),
                                  nn.LeakyReLU(.2), blocks.normalization(cc.ConvTranspose1d(128, 64, 16, stride=8,
                                                                                            padding=4)))
    sd = {k: v.detach().clone() for k, v in seq.state_dict().items()}
    x = torch.randn(4, 32, 300)
    po = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    h = O.conv1d(xo, O.wn_weight(po, "0."), None, pad=O.get_padding(3))
    want = O.conv_transpose1d(O.leaky_relu(h, 0.2), O.wn_weight(po, "2."), None, 8, 4)
    probe = torch.randn(want.shape)
    names = sorted(po)
    g_o = torch.autograd.grad((want * probe).sum(), [xo] + [po[k] for k in names])
    seq.cuda().train()
    _no_fp32_convs(monkeypatch)
    rave_b200.set_precision("bf16")
    try:
        assert seq._tc_plan() is not None
        xg = x.cuda().requires_grad_(True)
        y = seq(xg)
        pg = dict(seq.named_parameters())
        g = torch.autograd.grad((y * probe.cuda()).sum(), [xg] + [pg[k] for k in names])
        torch.cuda.synchronize()
    finally:
        rave_b200.set_precision("fp32")
    assert y.shape == want.shape
    assert rel_l2(y, want) < 3e-2
    assert rel_l2(g[0], g_o[0]) < 5e-2
    for k, a, b in zip(names, g[1:], g_o[1:]):
        assert rel_l2(a, b) < 5e-2, (k, rel_l2(a, b))


def _tiny_model_from_fixture(fx):
    from rave_b200 import configs
    cfg = fx["cfg"]
    holder = torch.nn.Module()
    holder.pqmf, holder.encoder, holder.decoder = configs.make_autoencoder("v2_nopqmf", capacity=cfg["capacity"],
                                                                           latent_size=cfg["latent_size"])
    holder.load_state_dict(fx["state_dict"], strict=True)
    return holder


def _forward(holder, x, eps):
    from rave_b200.model import _pqmf_encode
    z = holder.encoder(_pqmf_encode(holder.pqmf, x))
    zs, _ = holder.encoder.reparametrize(z, eps)
    return holder.decoder(zs)


def test_fp32_model_vs_reference_fixture():
    """DESIGN §2 fp32 tolerances: forward <= 2e-5, grad_x <= 1e-4, parameter gradients <= 5e-4."""
    fx = load("autoencoder_v2_nopqmf_tiny.pt")
    holder = _tiny_model_from_fixture(fx).cuda().train()
    x = fx["x"].cuda().requires_grad_(True)
    y = _forward(holder, x, fx["eps"].cuda())
    assert y.shape == fx["y"].shape
    assert rel_l2(y, fx["y"]) < 2e-5
    pp = dict(holder.named_parameters())
    names = sorted(fx["grad_params"])
    g = torch.autograd.grad((y * fx["probe"].cuda()).sum(), [x] + [pp[n] for n in names])
    assert rel_l2(g[0], fx["grad_x"]) < 1e-4
    for n, a in zip(names, g[1:]):
        assert rel_l2(a, fx["grad_params"][n]) < 5e-4, (n, rel_l2(a, fx["grad_params"][n]))


def test_bf16_model_vs_oracle_without_fallback(monkeypatch):
    """Capacity 16 (every conv width a multiple of 16): encoder and raw generator as engine chains, fused units, padded
    output conv; the fp32 conv entry points raise, so a chain that falls back fails the test."""
    import rave_b200
    from rave_b200 import _lib, configs
    torch.manual_seed(3)
    pq, enc, dec = configs.make_autoencoder("v2_nopqmf", capacity=16, latent_size=16)
    holder = torch.nn.Module()
    holder.pqmf, holder.encoder, holder.decoder = pq, enc, dec
    sd = {k: v.detach().clone() for k, v in holder.state_dict().items()}
    cfg = O.ArchConfig(capacity=16, latent_size=16)
    gcfg = N.generator_config(cfg)
    T = 16384
    x = (0.5 * torch.randn(2, 1, T)).clamp(-1, 1)
    eps = torch.randn(2, 16, T // 2048)
    po = {k: v.clone().requires_grad_(v.is_floating_point() and not k.startswith("pqmf.")) for k, v in sd.items()}
    xo = x.clone().requires_grad_(True)
    want = N.rave_forward_raw(xo, po, cfg, gcfg, eps)
    probe = torch.randn(want.shape)
    names = sorted(k for k, p in holder.named_parameters() if p.requires_grad and not k.startswith("pqmf."))
    g_o = torch.autograd.grad((want * probe).sum(), [xo] + [po[k] for k in names])
    holder.cuda().train()
    _no_fp32_convs(monkeypatch)
    rave_b200.set_precision("bf16")
    _lib.PROFILE = []
    try:
        xg = x.cuda().requires_grad_(True)
        y = _forward(holder, xg, eps.cuda())
        pg = dict(holder.named_parameters())
        g = torch.autograd.grad((y * probe.cuda()).sum(), [xg] + [pg[k] for k in names])
        torch.cuda.synchronize()
        launched = {name for name, *_ in _lib.PROFILE}
    finally:
        _lib.PROFILE = None
        rave_b200.set_precision("fp32")
    assert "rave_dilated_unit_tc_fwd" in launched and "rave_conv1d_tc_wgrad" in launched
    assert rel_l2(y, want) < 3e-2, rel_l2(y, want)
    assert cos(g[0], g_o[0]) > 0.98
    ga = torch.cat([a.detach().cpu().reshape(-1) for a in g[1:]])
    gb = torch.cat([b.reshape(-1) for b in g_o[1:]])
    assert cos(ga, gb) > 0.99, cos(ga, gb)


def _run_golden_steps(precision):
    """Replays tests/golden/training_step_v2_nopqmf_tiny.pt (a phase-2 D-step and G-step of the reference's own
    RAVE.training_step with output_mode "raw", both from the same seeded parameters) through
    rave_b200.RAVE.training_step.  Returns per step (logs, the seeded sample of the stepped group's gradients)."""
    import rave_b200
    from rave_b200 import configs
    g = load("training_step_v2_nopqmf_tiny.pt")
    cfg = g["cfg"]
    m = configs.build_rave("v2_nopqmf", capacity=cfg["capacity"], latent_size=cfg["latent_size"],
                           disc_capacity=g["disc_capacity"], phase_1_duration=1000)
    m.update_discriminator_every = g["update_discriminator_every"]
    sd0 = dict(m.state_dict(), **N.seeded_params(g["param_shapes"], g["param_seed"]))
    m.cuda().train()
    Lz = g["T"] // cfg["n_band"] // math.prod(cfg["ratios"])
    rave_b200.set_precision(precision)
    out = []
    try:
        for st in g["steps"]:
            m.load_state_dict(sd0, strict=True)
            m.set_receptive_field(*g["receptive_field"])
            m.warmed_up = True
            for p in m.parameters():
                p.grad = None
            x = N.step_batch(g["B"], g["T"], st["seed"]).cuda()
            eps = N.step_eps(g["B"], cfg["latent_size"], Lz, st["seed"]).cuda()
            logs = m.training_step(x, st["batch_idx"], eps=eps)
            logs = {k: (v.detach().float().cpu() if torch.is_tensor(v) else torch.tensor(float(v))) for k, v in logs.items()}
            pg = dict(m.named_parameters())
            assert all(pg[k].grad is not None for k in st["grad_keys"]), st["name"]
            flat = torch.cat([pg[k].grad.detach().reshape(-1).cpu() for k in st["grad_keys"]])
            shape, idx, _ = st["grad_sample"]
            assert tuple(flat.shape) == tuple(shape)
            out.append((logs, flat[idx]))
    finally:
        rave_b200.set_precision("fp32")
    return g, out


def test_nopqmf_training_step_matches_reference_goldens_fp32():
    """Logged losses <= 1e-4 of the reference's; the sampled gradient of the stepped group in direction (cos > 0.99)."""
    g, out = _run_golden_steps("fp32")
    for st, (logs, gs) in zip(g["steps"], out):
        for k, want in st["logs"].items():
            if k == "beta_factor":
                continue
            assert k in logs, (st["name"], k)
            assert abs(float(logs[k]) - float(want)) <= 1e-4 * max(abs(float(want)), 1e-3), (st["name"], k,
                                                                                              float(logs[k]), float(want))
        c = cos(gs, st["grad_sample"][2])
        print(f"{st['name']} (fp32): gradient sample cos {c:.6f}")
        assert c > 0.99, (st["name"], c)


def test_nopqmf_training_step_matches_reference_goldens_bf16():
    """Within the bounds of test_gpu_parity.py::test_training_step_matches_reference_goldens_bf16.  The tiny model
    (capacity 8) has widths that are not multiples of 16, so its generator runs the fp32 kernels; the engine path of
    the generator is covered at capacity 16 by test_bf16_model_vs_oracle_without_fallback."""
    g, out = _run_golden_steps("bf16")
    for st, (logs, gs) in zip(g["steps"], out):
        for k, want in st["logs"].items():
            if k == "beta_factor":
                continue
            tol = 0.10 if k in ("feature_matching", "adversarial", "pred_fake", "pred_real") else 0.03
            assert abs(float(logs[k]) - float(want)) <= tol * max(abs(float(want)), 1e-3), (st["name"], k,
                                                                                           float(logs[k]), float(want))
        c = cos(gs, st["grad_sample"][2])
        print(f"{st['name']} (bf16): gradient sample cos {c:.4f}")
        assert c > 0.9, (st["name"], c)


def test_nopqmf_graphed_steps_match_eager_and_are_deterministic(monkeypatch):
    """bf16, capacity 16 (the raw generator on the engine): GraphedTrainer replays == eager training_step on the same
    data, and two graphed runs from the same state are bit-identical."""
    import rave_b200
    from rave_b200 import configs, discriminator
    from rave_b200.graphs import GraphedTrainer
    monkeypatch.setattr(discriminator, "DISC_STREAMS", 1)
    torch.manual_seed(0)
    rave_b200.set_precision("bf16")
    try:
        m1 = configs.build_rave("v2_nopqmf", capacity=16, latent_size=16, disc_capacity=16).cuda().train()
        m1.warmed_up = True
        m1.encoder.reparametrize = (lambda z, eps=None, enc=m1.encoder: type(enc).reparametrize(
            enc, z, torch.zeros_like(z[:, :z.shape[1] // 2])))
        m2, m3 = copy.deepcopy(m1), copy.deepcopy(m1)
        x = (0.5 * torch.randn(2, 1, 65536, device="cuda")).clamp(-1, 1)
        assert m1.decoder.net._tc_plan() is not None
        tr2 = GraphedTrainer(m2, x, warmup_steps=2)
        tr3 = GraphedTrainer(m3, x, warmup_steps=2)
        m1.optimizers(capturable=True)
        for i in range(4):
            l2 = tr2.step(x, i)
            l3 = tr3.step(x, i)
            l1 = m1.training_step(x, i)
        torch.cuda.synchronize()
    finally:
        rave_b200.set_precision("fp32")
    for k in ("fullband_spectral_distance", "multiband_spectral_distance", "feature_matching", "adversarial"):
        assert torch.equal(l2[k], l3[k]), k
        assert rel_l2(l2[k], l1[k]) < 2e-2, (k, float(l2[k]), float(l1[k]))
    for (n, p2), p3 in zip(m2.named_parameters(), m3.parameters()):
        assert torch.equal(p2, p3), n
    w = lambda m: m.decoder.net[-1].weight_v
    assert rel_l2(w(m2), w(m1)) < 1e-2

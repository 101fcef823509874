"""GPU: the hybrid configuration (rave/configs/hybrid.gin) -- rave_mel_log1p_fwd, the GRU kernels (rave_gru_fwd /
rave_gru_bwd + rave_gemm_f32) against torch.nn.GRU in float64, the fp32 and bf16 models against the reference's
fixtures and the oracle, the three training steps, and CUDA-graph replays."""
import copy
import os

import pytest
import torch

from oracle import hybrid_oracle as Hy
from oracle import rave_oracle as O
from tests.conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu


def load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def cos(a, b):
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    return float(a @ b / (a.norm() * b.norm()).clamp_min(1e-30))


@pytest.mark.parametrize("B,C,T", [(1, 1, 1100), (2, 1, 5000), (3, 2, 8191), (2, 2, 65536), (4, 1, 16384)])
def test_mel_front_end_vs_oracle(B, C, T):
    from rave_b200 import configs
    torch.manual_seed(B * 100 + T)
    mel = configs.mel_spectrogram(44100 if C == 2 else 48000)
    x = torch.randn(B, C, T)
    want = Hy.mel_log1p(x.double(), mel.spectrogram.window.double(), mel.mel_scale.fb.double())
    got = mel.cuda().encode_log1p(x.cuda())
    torch.cuda.synchronize()
    assert got.shape == want.shape == (B, C * 128, T // 256)
    assert rel_l2(got, want) < 1e-5, rel_l2(got, want)
    try:
        import torchaudio
    except ImportError:
        return
    ta = torchaudio.transforms.MelSpectrogram(sample_rate=44100 if C == 2 else 48000, n_fft=2048, win_length=2048,
                                              hop_length=256, normalized=True, n_mels=128)
    assert rel_l2(got, torch.log1p(ta(x)[..., :-1]).reshape(B, C * 128, -1)) < 1e-5


def _autoencoder_fixture():
    fx = load("autoencoder_v2_hybrid_tiny.pt")
    return fx, Hy.autoencoder_state(fx, Hy.dense_filterbank(load("mel_filterbanks.pt")[48000]))


def test_mel_front_end_vs_fixture():
    from rave_b200 import configs
    fx, sd = _autoencoder_fixture()
    mel = configs.mel_spectrogram(48000)
    mel.load_state_dict({k[len("spectrogram."):]: v for k, v in sd.items() if k.startswith("spectrogram.")})
    got = mel.cuda().encode_log1p(fx["x"].cuda())
    assert rel_l2(got, fx["x_mel"]) < 1e-5


# B = 1, 3, 5, 33: not multiples of the kernel's two rows per CTA
@pytest.mark.parametrize("B,T", [(1, 1), (3, 5), (5, 33), (32, 32), (33, 64), (2, 200)])
def test_gru_forward_and_gradients_vs_torch_float64(B, T):
    from rave_b200 import blocks
    torch.manual_seed(B * 1000 + T)
    g = blocks.GRU(128, 2)
    ref = copy.deepcopy(g.gru).double()
    x = torch.randn(B, 128, T)
    probe = torch.randn(B, 128, T)
    xr = x.double().requires_grad_(True)
    yr = ref(xr.transpose(1, 2))[0].transpose(1, 2)
    pr = list(ref.parameters())
    gr = torch.autograd.grad((yr * probe.double()).sum(), [xr] + pr)
    g = g.cuda()
    xg = x.cuda().requires_grad_(True)
    y = g(xg)
    pg = list(g.gru.parameters())
    gg = torch.autograd.grad((y * probe.cuda()).sum(), [xg] + pg)
    torch.cuda.synchronize()
    assert y.shape == (B, 128, T)
    assert rel_l2(y, yr) < 1e-5, rel_l2(y, yr)
    names = ["x"] + [n for n, _ in ref.named_parameters()]
    for n, a, b in zip(names, gg, gr):
        assert rel_l2(a, b) < 1e-4, (n, rel_l2(a, b))


def test_gru_is_bit_identical_across_runs():
    from rave_b200 import blocks
    torch.manual_seed(0)
    g = blocks.GRU(128, 2).cuda()
    x = torch.randn(32, 128, 32, device="cuda", requires_grad=True)
    outs = []
    for _ in range(2):
        y = g(x)
        grads = torch.autograd.grad(y.square().sum(), [x] + list(g.parameters()))
        outs.append([y.detach()] + [t.detach() for t in grads])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def _tiny_holder(capacity, latent_size, sd=None):
    from rave_b200 import configs
    holder = torch.nn.Module()
    pq, enc, dec = configs.make_autoencoder("v2_hybrid", capacity=capacity, latent_size=latent_size)
    holder.pqmf, holder.spectrogram, holder.encoder, holder.decoder = pq, configs.mel_spectrogram(48000), enc, dec
    if sd is not None:
        holder.load_state_dict(sd, strict=True)
    return holder


def _forward(holder, x, eps):
    from rave_b200.model import _pqmf_decode
    z = holder.encoder(holder.spectrogram.encode_log1p(x))
    zs, _ = holder.encoder.reparametrize(z, eps)
    return _pqmf_decode(holder.pqmf, holder.decoder(zs), batch_size=x.shape[:-2], n_channels=1)


def test_fp32_model_vs_reference_fixture():
    """DESIGN §2 fp32 tolerances: forward <= 2e-5, parameter gradients <= 5e-4."""
    fx, sd = _autoencoder_fixture()
    holder = _tiny_holder(fx["cfg"]["capacity"], fx["cfg"]["latent_size"], sd).cuda().train()
    y = _forward(holder, fx["x"].cuda(), fx["eps"].cuda())
    assert y.shape == fx["y"].shape
    assert rel_l2(y, fx["y"]) < 2e-5, rel_l2(y, fx["y"])
    pp = dict(holder.named_parameters())
    names = sorted(fx["grad_params"])
    probe = torch.randn(y.shape, generator=torch.Generator().manual_seed(fx["probe_seed"]))
    g = torch.autograd.grad((y * probe.cuda()).sum(), [pp[n] for n in names])
    for n, a in zip(names, g):
        got, want = Hy.grad_pair(a, fx["grad_params"][n])
        assert rel_l2(got, want) < 5e-4, (n, rel_l2(got, want))


def _no_fp32_convs(monkeypatch):
    from rave_b200 import ops

    def boom(*a, **k):
        raise AssertionError("fp32 conv fallback in bf16 mode")
    monkeypatch.setattr(ops, "conv1d", boom)
    monkeypatch.setattr(ops, "conv_transpose1d", boom)


def test_bf16_model_vs_oracle_without_fallback(monkeypatch):
    """Capacity 16: the mel encoder and the generator after the GRU as engine chains; the fp32 conv entry points raise,
    and no fp32 conv kernel is launched at all (the GRU's GEMMs are its own)."""
    import rave_b200
    from rave_b200 import _lib
    torch.manual_seed(3)
    holder = _tiny_holder(16, 128)
    sd = {k: v.detach().clone() for k, v in holder.state_dict().items()}
    cfg = O.ArchConfig(capacity=16, latent_size=128)
    T = 16384
    x = (0.5 * torch.randn(2, 1, T)).clamp(-1, 1)
    eps = torch.randn(2, 128, T // 2048)
    names = sorted(k for k, p in holder.named_parameters() if p.requires_grad and not k.startswith("pqmf."))
    po = {k: v.clone().requires_grad_(k in names) for k, v in sd.items()}
    want = Hy.rave_forward_hybrid(x, po, cfg, eps)
    probe = torch.randn(want.shape)
    g_o = torch.autograd.grad((want * probe).sum(), [po[k] for k in names])
    holder.cuda().train()
    _no_fp32_convs(monkeypatch)
    rave_b200.set_precision("bf16")
    _lib.PROFILE = []
    try:
        y = _forward(holder, x.cuda(), eps.cuda())
        pg = dict(holder.named_parameters())
        g = torch.autograd.grad((y * probe.cuda()).sum(), [pg[k] for k in names])
        torch.cuda.synchronize()
        launched = [name for name, *_ in _lib.PROFILE]
    finally:
        _lib.PROFILE = None
        rave_b200.set_precision("fp32")
    assert launched.count("rave_gru_fwd") == 2 and launched.count("rave_gru_bwd") == 2
    assert "rave_mel_log1p_fwd" in launched and "rave_dilated_unit_tc_fwd" in launched
    assert "rave_conv1d_gather_f32" not in launched and "rave_conv1d_scatter_f32" not in launched
    assert rel_l2(y, want) < 3e-2, rel_l2(y, want)
    ga = torch.cat([a.detach().cpu().reshape(-1) for a in g])
    gb = torch.cat([b.reshape(-1) for b in g_o])
    assert cos(ga, gb) > 0.99, cos(ga, gb)
    gru = [i for i, k in enumerate(names) if ".gru." in k]
    assert cos(torch.cat([g[i].cpu().reshape(-1) for i in gru]), torch.cat([g_o[i].reshape(-1) for i in gru])) > 0.99


def _run_golden_steps(precision):
    import rave_b200
    from rave_b200 import configs
    g = load("training_step_v2_hybrid_tiny.pt")
    cfg = g["cfg"]
    m = configs.build_rave("v2_hybrid", capacity=cfg["capacity"], latent_size=cfg["latent_size"],
                           disc_capacity=g["disc_capacity"], phase_1_duration=1000)
    m.update_discriminator_every = g["update_discriminator_every"]
    sd0 = dict(m.state_dict(), **Hy.seeded_params(g["param_shapes"], g["param_seed"]))
    m.cuda().train()
    Lz = g["T"] // 2048
    rave_b200.set_precision(precision)
    out = []
    try:
        for st in g["steps"]:
            m.load_state_dict(sd0, strict=True)
            m.set_receptive_field(*g["receptive_field"])
            m.warmed_up = st["warmed_up"]
            for p in m.parameters():
                p.grad = None
            x = Hy.step_batch(g["B"], g["T"], st["seed"]).cuda()
            eps = Hy.step_eps(g["B"], cfg["latent_size"], Lz, st["seed"]).cuda()
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


# Gradient samples are compared for the D-step only.  In both G-steps the logged losses match the reference's, but the
# gradient its own training_step leaves on the generator does not point the way the gradient of those losses does when
# the oracle restates them on the CPU (phase 1: cos 0.96); the cause is not known, so those samples are not a yardstick.
def _gradient_checked(st):
    return st["warmed_up"] and st["batch_idx"] == 0


def test_hybrid_training_steps_match_reference_goldens_fp32():
    g, out = _run_golden_steps("fp32")
    for st, (logs, gs) in zip(g["steps"], out):
        for k, want in st["logs"].items():
            if k == "beta_factor":
                continue
            assert abs(float(logs[k]) - float(want)) <= 1e-4 * max(abs(float(want)), 1e-3), (st["name"], k,
                                                                                              float(logs[k]), float(want))
        c = cos(gs, st["grad_sample"][2])
        print(f"{st['name']} (fp32): gradient sample cos {c:.6f}")
        if _gradient_checked(st):
            assert c > 0.99, (st["name"], c)


def test_hybrid_training_steps_match_reference_goldens_bf16():
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
        if _gradient_checked(st):
            assert c > 0.9, (st["name"], c)


@pytest.mark.parametrize("n_channels", [1, 2])
def test_hybrid_graphed_steps_match_eager_and_are_deterministic(monkeypatch, n_channels):
    """bf16, capacity 16: GraphedTrainer replays == eager training_step on the same data, and two graphed runs from the
    same state are bit-identical."""
    import rave_b200
    from rave_b200 import configs, discriminator
    from rave_b200.graphs import GraphedTrainer
    monkeypatch.setattr(discriminator, "DISC_STREAMS", 1)
    torch.manual_seed(0)
    rave_b200.set_precision("bf16")
    try:
        m1 = configs.build_rave("v2_hybrid", capacity=16, disc_capacity=16, n_channels=n_channels).cuda().train()
        m1.warmed_up = True
        m1.encoder.reparametrize = (lambda z, eps=None, enc=m1.encoder: type(enc).reparametrize(
            enc, z, torch.zeros_like(z[:, :z.shape[1] // 2])))
        m2, m3 = copy.deepcopy(m1), copy.deepcopy(m1)
        x = (0.5 * torch.randn(2, n_channels, 65536, device="cuda")).clamp(-1, 1)
        assert m1.decoder.net._tc_plan() is not None and m1.encoder.encoder.net._tc_plan() is not None
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
    w = lambda m: m.decoder.net[0].gru.weight_hh_l1
    assert rel_l2(w(m2), w(m1)) < 1e-2

"""CPU: the v2_nopqmf configuration (raw-waveform generator, rave/configs/v2_nopqmf.gin) -- module tree against the
reference's, the oracle restatement against the reference's fixtures, and the engine's plan of the full-size generator
(padded 2-channel output conv, fused units of width 64 / 128 / 256) with the kernels emulated (tests/tc_emulator.py)."""
import os

import pytest
import torch

from oracle import nopqmf_oracle as N
from oracle import rave_oracle as O
from tests import tc_emulator
from tests.conftest import GOLDEN, rel_l2


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def test_state_dict_matches_reference():
    from rave_b200 import configs
    want = _load("state_dict_keys_nopqmf.pt")["rave_v2_nopqmf"]
    m = configs.build_rave("v2_nopqmf")
    got = {k: (tuple(v.shape), str(v.dtype)) for k, v in m.state_dict().items()}
    assert list(got) == list(want)
    assert got == want
    assert m.output_mode == "raw" and m.input_mode == "pqmf"
    assert m.decoder.net[-1].out_channels == 2                   # waveform + amplitude, mono
    assert m.update_discriminator_every == 4


def test_oracle_autoencoder_vs_fixture():
    fx = _load("autoencoder_v2_nopqmf_tiny.pt")
    cfg = O.ArchConfig(**fx["cfg"])
    gcfg = N.generator_config(cfg, fx["gen_ratios"])
    sd = fx["state_dict"]
    po = {k: v.clone().requires_grad_(v.is_floating_point() and not k.startswith("pqmf.")) for k, v in sd.items()}
    x = fx["x"].clone().requires_grad_(True)
    y = N.rave_forward_raw(x, po, cfg, gcfg, fx["eps"])
    assert rel_l2(y, fx["y"]) < 1e-6
    names = sorted(fx["grad_params"])
    g = torch.autograd.grad((y * fx["probe"]).sum(), [x] + [po[n] for n in names])
    assert rel_l2(g[0], fx["grad_x"]) < 1e-5
    for n, a in zip(names, g[1:]):
        assert rel_l2(a, fx["grad_params"][n]) < 1e-5, n


def test_oracle_training_step_vs_fixture():
    fx = _load("training_step_v2_nopqmf_tiny.pt")
    cfg = O.ArchConfig(**fx["cfg"])
    gcfg = N.generator_config(cfg, fx["gen_ratios"])
    sd = N.seeded_params(fx["param_shapes"], fx["param_seed"])
    sd["pqmf.hk"] = fx["hk"]
    B, T = fx["B"], fx["T"]
    Lz = T // cfg.n_band
    for r in cfg.ratios:
        Lz //= r
    for st in fx["steps"]:
        x = N.step_batch(B, T, st["seed"])
        eps = N.step_eps(B, cfg.latent_size, Lz, st["seed"])
        losses, ldis = N.train_step_losses(x, sd, cfg, gcfg, eps, receptive_field=fx["receptive_field"])
        for k, v in losses.items():
            assert rel_l2(v, st["logs"][k]) < 2e-6, (st["name"], k)
        assert rel_l2(ldis, st["logs"]["loss_dis"]) < 2e-6


@pytest.fixture(params=["exact_fp32", "bf16"])
def emu(request, monkeypatch):
    from rave_b200 import engine
    tc_emulator.install(monkeypatch)
    dt = torch.float32 if request.param == "exact_fp32" else torch.bfloat16
    monkeypatch.setattr(tc_emulator, "OPERAND_DTYPE", dt)
    monkeypatch.setattr(engine, "ACT_DTYPE", dt)
    return request.param


def test_full_generator_plans_fused_units_and_matches_the_two_launch_form(emu, monkeypatch):
    """Capacity 64: the whole generator is one engine chain (its 64 -> 2 output conv padded to 16 channels, the chain
    still returning 2); the 9 units of width 64 / 128 / 256 run through ops.dilated_unit_tc (C = 512 keeps two launches),
    and forward and every gradient equal the unfused chain."""
    from rave_b200 import configs, engine, ops
    monkeypatch.setattr(ops, "dilated_unit_tc_supported", lambda C, L: C in (64, 96, 128, 192, 256, 384) and L >= 8)
    calls = []
    real = tc_emulator.dilated_unit_tc

    def spy(*a, **k):
        calls.append(a[0].shape[-1])
        return real(*a, **k)
    monkeypatch.setattr(ops, "dilated_unit_tc", spy)
    torch.manual_seed(5)
    _, _, dec = configs.make_autoencoder("v2_nopqmf")
    dec.train()
    specs = dec.net._tc_plan()
    assert specs is not None and engine.chain_supported(specs)
    assert specs[-1].Cout == 2 and specs[-1].cout_pad == 14
    assert [s.stride for s in specs if s.kind == "convT"] == [4, 8, 8, 8]
    z = torch.randn(1, 128, 1)
    outs = {}
    for fuse in (True, False):
        monkeypatch.setattr(engine, "FUSE_UNITS", fuse)
        zi = z.clone().requires_grad_(True)
        n0 = len(calls)
        (out,) = engine.run_chain(engine.to_channel_last(zi), specs)
        L = engine.chain_lengths(specs, 1)[-1]
        assert L == 2048 and out.shape[-1] == 16
        w = engine.from_channel_last(out[:, :L, :2].contiguous())
        pd = dict(dec.named_parameters())
        names = sorted(pd)
        probe = torch.randn(w.shape, generator=torch.Generator().manual_seed(3))
        g = torch.autograd.grad((w * probe).sum(), [zi] + [pd[k] for k in names])
        outs[fuse] = (w.detach(), [t.detach() for t in g], calls[n0:])
    if emu == "bf16":
        assert sorted(outs[True][2]) == [64] * 3 + [128] * 3 + [256] * 3 and outs[False][2] == []
        assert torch.equal(outs[True][0], outs[False][0])
        for a, b in zip(outs[True][1], outs[False][1]):
            assert torch.equal(a, b)
    else:
        assert outs[True][2] == []               # fp32 operand emulation: the fused kernel is a bf16 kernel


def test_padded_output_conv_vs_oracle(emu):
    """A capacity-16 generator: its padded output conv and r = 8 transposed convs on the emulated engine against the
    fp32 oracle: forward and the gradients of the input and of every parameter (CachedSequential slices the 2 real
    channels; the slice's backward zero-extends the incoming gradient)."""
    from rave_b200 import configs, engine
    torch.manual_seed(6)
    _, _, dec = configs.make_autoencoder("v2_nopqmf", capacity=16, latent_size=16)
    dec.train()
    sd = {"decoder." + k: v.detach().clone() for k, v in dec.state_dict().items()}
    gcfg = N.generator_config(O.ArchConfig(capacity=16, latent_size=16))
    z = torch.randn(2, 16, 2)
    # the oracle runs in float64: its fp32 CPU stride-8 transposed-conv backward is itself ~2e-5 off in grad z here
    po = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    zo = z.double().requires_grad_(True)
    taps = {}
    want = N.generator_raw(zo, po, "decoder.", gcfg, taps)
    specs = dec.net._tc_plan()
    assert specs is not None and specs[-1].cout_pad == 14
    ze = z.clone().requires_grad_(True)
    (out,) = engine.run_chain(engine.to_channel_last(ze), specs)
    L = engine.chain_lengths(specs, 2)[-1]
    wave = engine.from_channel_last(out[:, :L, :2].contiguous())
    assert wave.shape == taps["wave"].shape
    t = tol_of(emu)
    assert rel_l2(wave, taps["wave"]) < t
    probe = torch.randn(wave.shape, generator=torch.Generator().manual_seed(9))
    names = sorted(k for k in sd if k.startswith("decoder."))
    pd = dict(dec.named_parameters(prefix="decoder"))
    ge = torch.autograd.grad((wave * probe).sum(), [ze] + [pd[k] for k in names])
    go = torch.autograd.grad((taps["wave"] * probe.double()).sum(), [zo] + [po[k] for k in names])
    # gradient tolerances of test_engine_cpu.py::test_encoder_generator_chain_vs_oracle
    assert rel_l2(ge[0], go[0]) < tol_of(emu, 1e-5, 0.15)
    for n, a, b in zip(names, ge[1:], go[1:]):
        assert a.shape == b.shape and rel_l2(a, b) < tol_of(emu, 2e-5, 0.2), (n, rel_l2(a, b))


def tol_of(emu, exact=1e-5, loose=3e-2):
    return exact if emu == "exact_fp32" else loose

"""CPU: the hybrid configuration (rave/configs/hybrid.gin) -- the HTK filter bank, the oracle against the reference's
fixtures, the module trees / state_dict keys, and the engine plan that runs the GRU ahead of the generator chain."""
import os

import pytest
import torch

from oracle import hybrid_oracle as Hy
from oracle import rave_oracle as O
from rave_b200 import blocks, configs, core, engine
from tests.conftest import GOLDEN, rel_l2


def load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


@pytest.mark.parametrize("sr", [44100, 48000])
def test_filterbank_matches_torchaudio_fixture(sr):
    fb = core.htk_mel_filterbank(sr, 2048, 128)
    want = Hy.dense_filterbank(load("mel_filterbanks.pt")[sr])
    assert fb.shape == want.shape == (1025, 128)
    assert torch.equal(fb != 0, want != 0)
    assert (fb - want).abs().max() < 3e-5          # float32 rounding of the slopes (torch vs numpy order)
    # banded: each bin feeds at most 2 bands, each band is one contiguous bin range
    assert int((fb != 0).sum(1).max()) <= 2
    for m in range(128):
        nz = torch.nonzero(fb[:, m]).reshape(-1)
        assert int(nz[-1] - nz[0]) + 1 == nz.numel()
    try:
        import torchaudio
    except ImportError:
        return
    ta = torchaudio.functional.melscale_fbanks(1025, 0.0, float(sr // 2), 128, sr, None, "htk")
    assert (fb - ta).abs().max() < 3e-5


def test_band_table_packs_the_filterbank():
    mel = configs.mel_spectrogram(48000)
    band, w = mel.band_table()
    fb = mel.mel_scale.fb
    dense = torch.zeros_like(fb)
    for m, (lo, hi, off) in enumerate(band.tolist()):
        dense[lo:hi, m] = w[off:off + hi - lo]
    assert torch.equal(dense, fb)
    assert w.numel() == int((fb != 0).sum())


def _autoencoder_fixture():
    fx = load("autoencoder_v2_hybrid_tiny.pt")
    return fx, Hy.autoencoder_state(fx, Hy.dense_filterbank(load("mel_filterbanks.pt")[48000]))


def test_oracle_reproduces_autoencoder_fixture():
    fx, sd = _autoencoder_fixture()
    cfg = O.ArchConfig(**{k: v for k, v in fx["cfg"].items() if k != "generator_latent"})
    taps = {}
    y = Hy.rave_forward_hybrid(fx["x"], sd, cfg, fx["eps"], taps)
    assert rel_l2(taps["x_mel"], fx["x_mel"]) < 1e-6
    assert rel_l2(y, fx["y"]) < 1e-6


def test_oracle_gru_matches_torch_gru():
    torch.manual_seed(0)
    g = blocks.GRU(16, 2).double()
    sd = {"m." + k: v for k, v in g.state_dict().items()}
    x = torch.randn(3, 16, 7, dtype=torch.float64)
    want = g.gru(x.transpose(1, 2))[0].transpose(1, 2)
    assert rel_l2(Hy.gru(x, sd, "m."), want) < 1e-12


def test_oracle_mel_matches_torchaudio():
    torchaudio = pytest.importorskip("torchaudio")
    mel = torchaudio.transforms.MelSpectrogram(sample_rate=44100, n_fft=2048, win_length=2048, hop_length=256,
                                               normalized=True, n_mels=128)
    x = torch.randn(2, 2, 5000)
    want = torch.log1p(mel(x)[..., :-1]).reshape(2, 256, -1)
    got = Hy.mel_log1p(x, mel.spectrogram.window, mel.mel_scale.fb)
    assert got.shape == want.shape == (2, 256, 5000 // 256)
    assert rel_l2(got, want) < 1e-6


def test_oracle_reproduces_training_step_fixture():
    g = load("training_step_v2_hybrid_tiny.pt")
    cfg = O.ArchConfig(**{k: v for k, v in g["cfg"].items() if k != "generator_latent"})
    m = configs.build_rave("v2_hybrid", capacity=cfg.capacity, latent_size=cfg.latent_size,
                           disc_capacity=g["disc_capacity"])
    sd = dict(m.state_dict(), **Hy.seeded_params(g["param_shapes"], g["param_seed"]))
    Lz = g["T"] // 2048
    for st in g["steps"]:
        x = Hy.step_batch(g["B"], g["T"], st["seed"])
        eps = Hy.step_eps(g["B"], cfg.latent_size, Lz, st["seed"])
        losses, ldis = Hy.train_step_losses(x, sd, cfg, eps, st["warmed_up"], g["receptive_field"])
        for k, v in losses.items():
            assert abs(float(v) - float(st["logs"][k])) <= 1e-5 * abs(float(st["logs"][k])), (st["name"], k)
        if ldis is not None:
            assert abs(float(ldis) - float(st["logs"]["loss_dis"])) <= 1e-5 * abs(float(st["logs"]["loss_dis"]))


@pytest.mark.parametrize("name,kw", [("rave_v2_hybrid", dict(name="v2_hybrid")),
                                     ("rave_v2_hybrid_stereo", dict(name="v2_hybrid", n_channels=2)),
                                     ("rave_v3_hybrid", dict(name="v3", hybrid=True))])
def test_full_rave_state_dict_contract(name, kw):
    ks = load("state_dict_keys_hybrid.pt")[name]
    m = configs.build_rave(**kw)
    sd = {k: (tuple(v.shape), str(v.dtype)) for k, v in m.state_dict().items()}
    assert set(sd) == set(ks), sorted(set(sd) ^ set(ks))[:20]
    assert sd == ks, [k for k in sd if sd[k] != ks[k]][:20]
    assert m.input_mode == "mel" and isinstance(m.decoder.net[0], blocks.GRU)


def test_make_autoencoder_loads_fixture_strictly():
    fx, sd = _autoencoder_fixture()
    pq, enc, dec = configs.make_autoencoder("v2_hybrid", capacity=fx["cfg"]["capacity"],
                                            latent_size=fx["cfg"]["latent_size"])
    holder = torch.nn.Module()
    holder.pqmf, holder.spectrogram, holder.encoder, holder.decoder = pq, configs.mel_spectrogram(48000), enc, dec
    holder.load_state_dict(sd, strict=True)


def test_plan_splits_off_the_gru_and_plans_the_rest():
    m = configs.build_rave("v2_hybrid", capacity=16)
    mods = list(m.decoder.net)
    lead, rest = engine.split_recurrent(mods)
    assert lead is mods[0] and rest == mods[1:]
    specs = engine.plan_sequential(mods)
    ref = engine.plan_sequential(rest)
    assert specs is not None and engine.chain_supported(specs)
    assert [(s.kind, s.Cin, s.Cout, s.K, s.stride) for s in specs] == [(s.kind, s.Cin, s.Cout, s.K, s.stride) for s in ref]
    assert specs[0].module is mods[1]
    # the plain v2 generator's plan is unchanged by the split
    v2 = configs.build_rave("v2", capacity=16)
    assert engine.split_recurrent(list(v2.decoder.net))[0] is None


@pytest.mark.parametrize("C", [1, 2])
def test_mel_encoder_is_one_engine_chain(C):
    """Stem Cin = 128 * C, units at 96 / 192 / 384, stride-2 downsampling convs: every layer on the engine."""
    m = configs.build_rave("v2_hybrid", n_channels=C)
    specs = engine.plan_sequential(list(m.encoder.encoder.net))
    assert specs is not None and engine.chain_supported(specs)
    assert specs[0].Cin == 128 * C
    convs = [s for s in specs if s.kind == "conv"]
    assert len(convs) == sum(1 for mod in m.encoder.encoder.net.modules() if isinstance(mod, torch.nn.Conv1d))


def test_disabled_gru_is_identity():
    g = blocks.GRU(128, 2)
    g.disable()
    x = torch.randn(1, 128, 4)
    assert g(x) is x
    g.enable()
    assert g.enabled

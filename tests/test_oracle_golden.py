"""CPU: the oracle restatement reproduces every committed golden tensor (the goldens were
produced by executing the unmodified reference, oracle/make_golden.py)."""
import os

import pytest
import torch

from oracle import rave_oracle as O
from tests.conftest import GOLDEN, rel_l2


def load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def test_pqmf_design_and_operators():
    g = load("pqmf.pt")
    h, hk = O.pqmf_design(100, 16)
    assert torch.equal(h, g["h"]) and torch.equal(hk, g["hk"])
    assert h.shape == (377,) and hk.shape == (16, 512)
    hkf, hki = O.cached_pqmf_weights(hk)
    assert torch.equal(hkf, g["forward_conv.weight"]) and torch.equal(hki, g["inverse_conv.weight"])
    for mode in ("centered", "causal"):
        x, y, xr = g[mode]["x"], g[mode]["y"], g[mode]["xr"]
        assert rel_l2(O.pqmf_analysis(x, hk, mode), y) < 1e-7
        assert rel_l2(O.pqmf_synthesis(y, hk, mode), xr) < 1e-7


def test_pqmf_three_formulations_agree():
    """SURVEY 8c: cached / polyphase / classic analysis agree; CachedPQMF.inverse == PQMF.inverse
    delayed by 16 samples."""
    g = load("pqmf.pt")
    hk = g["hk"]
    x, y = g["centered"]["x"], g["centered"]["y"]
    assert rel_l2(O.polyphase_forward(x, hk), y) < 4e-7
    assert rel_l2(O.classic_forward(x, hk), y) < 4e-7
    inv_poly = O.polyphase_inverse(y, hk)
    assert rel_l2(inv_poly, g["polyphase_inverse"]) < 1e-7
    inv_cached = O.pqmf_synthesis(y, hk)
    assert (inv_cached[..., 16:] - inv_poly[..., :-16]).abs().max() < 1e-5


def test_pqmf_roundtrip_config1():
    """BASELINE config 1: 16-band analysis->synthesis on 1 x 131072 @48 kHz, CPU.  Near-perfect
    reconstruction only: rel-L2 ~ 1.0e-3 (100 dB pseudo-QMF), 16-sample delay."""
    g = load("pqmf.pt")
    hk = g["hk"]
    gen = torch.Generator().manual_seed(7)
    x = (0.5 * torch.randn(1, 1, 131072, generator=gen)).clamp(-1, 1)
    xr = O.pqmf_synthesis(O.pqmf_analysis(x, hk), hk)
    assert xr.shape == x.shape
    r = rel_l2(xr[..., 16 + 1024:-1024], x[..., 1024:-1024 - 16])
    assert abs(r - g["roundtrip_rel_l2"]) < 1e-6
    assert 0.9e-3 < r < 1.1e-3


@pytest.mark.parametrize("name", ["v2_tiny", "v2_tiny_causal", "v3_tiny", "v2_small_tiny"])
def test_autoencoder_golden(name):
    g = load(f"autoencoder_{name}.pt")
    cfg = O.ArchConfig(**{k: v for k, v in g["cfg"].items()})
    taps = {}
    y = O.rave_forward(g["x"], g["state_dict"], cfg, g["eps"], taps)
    assert rel_l2(taps["x_mb"], g["x_mb"]) < 1e-7
    assert rel_l2(taps["z"], g["z"]) < 2e-6
    assert rel_l2(taps["y_mb"], g["y_mb"]) < 2e-6
    assert rel_l2(y, g["y"]) < 2e-6
    assert y.shape == g["x"].shape                      # tests/test_configs.py:69 contract


def test_discriminator_golden():
    g = load("discriminator_v2.pt")
    feats = O.combine_discriminators_v2(g["x"], g["state_dict"])
    assert len(feats) == 8 and all(len(f) == 5 for f in feats)
    for fa, fb in zip(feats, g["features"]):
        for a, b in zip(fa, fb):
            assert a.shape == b.shape and rel_l2(a, b) < 1e-6
    fm, ld, la = O.gan_losses(feats, 1, True)
    assert rel_l2(fm, g["fm"]) < 1e-6 and rel_l2(ld, g["loss_dis"]) < 1e-6 and rel_l2(la, g["loss_adv"]) < 1e-5


def test_audio_distance_golden():
    g = load("audio_distance.pt")
    assert rel_l2(O.audio_distance_v1(g["x"], g["y"]), g["distance"]) < 1e-6


def _pins(name):
    """tests/golden/reference_pins.pt (oracle/make_reference_pins.py): outputs of the unmodified reference, with the
    module parameters regenerated from their seed."""
    from oracle.make_reference_pins import seeded_state_dict
    g = load("reference_pins.pt")[name]
    sd = dict(seeded_state_dict(g["shapes"], g["seed"]), **g["buffers"]) if "shapes" in g else None
    return g, sd


def _check_sampled(got, want, tol):
    assert len(got) == len(want)
    for a, (shape, idx, val) in zip(got, want):
        assert tuple(a.shape) == tuple(shape) and rel_l2(a.reshape(-1)[idx], val) < tol, (shape, rel_l2(a.reshape(-1)[idx], val))


def test_oracle_matches_reference_pqmf():
    """The PQMF restatement against the unmodified reference's CachedPQMF (analysis and synthesis)."""
    g, _ = _pins("pqmf")
    assert torch.equal(O.pqmf_analysis(g["x"], g["hk"]), g["y"])
    assert torch.equal(O.pqmf_synthesis(g["y"], g["hk"]), g["x_rec"])


def test_descript_mpd_oracle_matches_reference():
    """Descript MPD (rave/descript_discriminator.py:30-66) and DescriptDiscriminator.preprocess against the unmodified
    reference (1024-channel layers: seeded parameters, sampled feature maps)."""
    g, sd = _pins("descript_mpd")
    got = O.descript_mpd(g["x"], sd, "", 3)
    assert len(got) == 6
    _check_sampled(got, g["out"], 1e-6)
    assert torch.equal(O.descript_preprocess(g["y"]), g["preprocessed"])


def test_descript_mrd_oracle_matches_reference():
    """Descript MRD (rave/descript_discriminator.py:118-184) against the unmodified reference."""
    g, sd = _pins("descript_mrd")
    got = O.descript_mrd(g["x"], sd, "", 512)
    assert len(got) == 26
    _check_sampled(got, g["out"], 2e-6)


# fp32 conditioning of the training-step gradients, (all tensors, worst tensor) rel-L2: see the comments in the test
GRAD_TOL = {"phase1_gen": (3e-3, 1e-2), "phase2_dis": (2e-5, 1e-3), "phase2_gen": (5e-2, 1e-1)}
# fraction of parameter elements whose Adam update may differ by more than 5 % of lr (same conditioning)
UPD_FRAC = {"phase1_gen": 2e-3, "phase2_dis": 2e-3, "phase2_gen": 6e-2}


def test_training_step_restatement_reproduces_reference_steps():
    """tests/golden/training_step_v2_tiny.pt holds three steps of the reference's OWN RAVE.training_step
    (rave/model.py:288-424; phase-1 G, phase-2 D, phase-2 G).  The restatement (O.train_step_losses / train_step_cpu,
    the CPU arm of bench.py) must give the same logged losses, and its gradients pushed through O.adam_step must land
    on the reference's post-step parameters."""
    g = load("training_step_v2_tiny.pt")
    cfg = O.ArchConfig(**g["cfg"])
    rf = tuple(g["receptive_field"])
    prev = g["state_dict"]
    moments = {}
    steps_taken = {"gen": 0, "dis": 0}
    for st in g["steps"]:
        dis_step = st["warmed_up"] and st["batch_idx"] % g["update_discriminator_every"] == 0
        total, loss_dis, parts = O.train_step_losses(st["x"], prev, cfg, st["eps"], warmed_up=st["warmed_up"],
                                                     receptive_field=rf, return_parts=True)
        for k, v in parts.items():
            assert rel_l2(v, st["logs"][k]) < 2e-6, (st["name"], k)
        if st["warmed_up"]:
            assert rel_l2(loss_dis, st["logs"]["loss_dis"]) < 2e-6
        _, _, grads = O.train_step_cpu(st["x"], prev, cfg, st["eps"], dis_step, warmed_up=st["warmed_up"],
                                       receptive_field=rf, return_named=True)
        group = "dis" if dis_step else "gen"
        steps_taken[group] += 1
        lr = 1e-4 if dis_step else 1e-3
        new = dict(prev)
        n_upd = 0
        assert {k for k, gr in grads.items() if gr is not None} == set(st["grads"]), st["name"]
        for k, gr in grads.items():
            if gr is None:
                continue
            # The gradient of the log-magnitude spectral distance is ill-conditioned in fp32: the reference's OWN fp32
            # gradients sit 5e-4 (rel-L2, all tensors) from an fp64 evaluation of the same step, this restatement's 8e-4
            # (measured in the build container); the losses themselves agree to the last bit.
            # The phase-2 generator step adds the L1 feature-matching term, whose gradient is sign(h_r - h_f): elements
            # at rounding level flip, and the reference's fp32 gradients are 1.1e-2 from fp64 (this restatement's 0.9e-2).
            # The discriminator step (hinge on the scores) is well conditioned: 5e-7.
            if st["grads"][k].abs().max() > 0:
                assert rel_l2(gr, st["grads"][k]) < GRAD_TOL[st["name"]][1], (st["name"], k, rel_l2(gr, st["grads"][k]))
            m, v = moments.get(k, (torch.zeros_like(gr), torch.zeros_like(gr)))
            # per-parameter step count: the encoder is frozen in phase 2 (z.detach()), its Adam state stays behind
            cnt = moments.get(("n", k), 0) + 1
            new[k], m, v = O.adam_step(prev[k], gr, m, v, cnt, lr)
            moments[k], moments[("n", k)] = (m, v), cnt
            n_upd += 1
        assert n_upd > 0
        cat = lambda d: torch.cat([d[k].reshape(-1) for k in sorted(st["grads"])])
        assert rel_l2(cat(grads), cat(st["grads"])) < GRAD_TOL[st["name"]][0], (st["name"],
                                                                                rel_l2(cat(grads), cat(st["grads"])))
        n_bad = n_all = 0
        for k in prev:
            want = st["state_dict"][k]
            if not want.is_floating_point():      # integer buffers (warmed_up flags, receptive_field): module state
                continue
            upd_ref = (want - prev[k]).double()
            upd = (new[k] - prev[k]).double()
            if upd_ref.abs().max() == 0:
                assert upd.abs().max() == 0, (st["name"], k)
            else:
                # a first Adam step is lr * sign(g): an element whose gradient sits at rounding level may flip, so
                # count elements that moved differently instead of taking a norm
                n_bad += int(((upd - upd_ref).abs() > 0.05 * lr).sum())
                n_all += upd.numel()
        assert n_bad <= UPD_FRAC[st["name"]] * n_all, (st["name"], n_bad, n_all)
        prev = st["state_dict"]


def test_noise_generator_oracle_matches_reference():
    """a13: the restatement of NoiseGeneratorV2 (+ mod_sigmoid / amp_to_impulse_response / fft_convolve) against the
    unmodified reference module; the reference's torch.rand_like draw is reproduced by re-seeding."""
    g, sd = _pins("noise_generator_v2")
    sd = {"n." + k: v for k, v in sd.items()}
    torch.manual_seed(77)
    noise = torch.rand(2, 32, 16, 8) * 2 - 1          # rand_like(ir): ir is [B, T/8, 16, 8]
    y = O.noise_generator_v2(g["x"], sd, "n.", (2, 2, 2), 16, 1, noise)
    assert y.shape == g["y"].shape == (2, 16, 256)
    assert rel_l2(y, g["y"]) < 1e-6


def test_v1_restatement_matches_reference_golden():
    """a12: O.encoder_v1 / O.generator_v1 (BatchNorm encoder, ResidualStack generator with loudness and filtered-noise
    branches) against tests/golden/autoencoder_v1_tiny.pt, forward and every gradient."""
    g = load("autoencoder_v1_tiny.pt")
    sd = g["state_dict"]
    po = {k: v.clone().requires_grad_(v.is_floating_point() and "running_" not in k and "target_size" not in k)
          for k, v in sd.items()}
    x = g["x"].clone().requires_grad_(True)
    z = O.encoder_v1(x, po, "encoder.", g["ratios"])
    assert rel_l2(z, g["z"]) < 2e-6
    zin = g["zin"].clone().requires_grad_(True)
    y = O.generator_v1(zin, po, "decoder.", tuple(g["ratios"])[::-1], warmed_up=True, noise=g["noise"])
    assert rel_l2(y, g["y"]) < 2e-6
    names = sorted(g["grads"])
    ge = torch.autograd.grad((z * g["probe_z"]).sum(), [x] + [po[k] for k in names if k.startswith("encoder.")])
    gd = torch.autograd.grad((y * g["probe_y"]).sum(), [zin] + [po[k] for k in names if k.startswith("decoder.")])
    assert rel_l2(ge[0], g["grad_x"]) < 1e-5 and rel_l2(gd[0], g["grad_zin"]) < 1e-5
    for k, a in zip([k for k in names if k.startswith("encoder.")], ge[1:]):
        assert rel_l2(a, g["grads"][k]) < 1e-5, k
    for k, a in zip([k for k in names if k.startswith("decoder.")], gd[1:]):
        assert rel_l2(a, g["grads"][k]) < 1e-5, k

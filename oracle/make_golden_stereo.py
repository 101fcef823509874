"""TEST INFRASTRUCTURE -- generates the fixtures of multichannel (stereo, `n_channels = 2`: scripts/train.py --channels 2)
models by EXECUTING THE UNMODIFIED REFERENCE, and asserts that oracle/rave_oracle.py / oracle/stereo_oracle.py reproduce
them.  Writes new files only:

    python -m oracle.make_golden_stereo

  tests/golden/discriminator_v2_stereo.pt       v2 discriminator (MPD + MSD, capacity 4) on a stereo signal: sampled
                                                features, fm / dis / adv terms, grad_x, a parameter-gradient sample
  tests/golden/training_step_v2_stereo_tiny.pt  the reference's own RAVE.training_step at n_channels = 2, a phase-2
  tests/golden/training_step_v3_stereo_tiny.pt  D-step and a phase-2 G-step from the same seeded parameters: logged
                                                losses, a seeded sample of the stepped group's gradients
  tests/golden/state_dict_keys_stereo.pt        keys / shapes / dtypes of the full-size v2 and v3 rave.RAVE in stereo
"""
import os
import sys
from functools import partial

import torch
import torch.nn as nn

from oracle import rave_oracle as O
from oracle import stereo_oracle as ST
from oracle.make_golden import GOLDEN, build_ref_rave, check, make_input
from oracle.ref_loader import load_reference, set_padding_mode

FEATURE_SAMPLE = 256
GRAD_SAMPLE = 8192
NC = ST.N_CHANNELS


def build_ref_rave_stereo(R, cfg: O.ArchConfig, *args, **kwargs):
    """oracle/make_golden.py::build_ref_rave (the v2 / v3 bindings of the reference's rave.RAVE) at n_channels = 2: the
    bindings are reused as they are, only the RAVE constructor sees n_channels = NC for the duration of the call."""
    rave_cls = R.model.RAVE

    def stereo(*a, **k):
        k["n_channels"] = NC
        return rave_cls(*a, **k)
    R.model.RAVE = stereo
    try:
        m = build_ref_rave(R, cfg, *args, **kwargs)
    finally:
        R.model.RAVE = rave_cls
    assert m.n_channels == NC
    return m


def golden_discriminator_v2_stereo(R, capacity=4, B=2, T=8192):
    """CombineDiscriminators(MPD, MSD) at n_channels = 2 on [2B, 2, T + 3] (+3: MPD remainder padding)."""
    print("v2 discriminator (MPD + MSD), stereo")
    D = R.discriminator
    torch.manual_seed(15)
    norm = R.blocks.normalization
    D.normalization = lambda m, mode="weight_norm": norm(m, mode)
    try:
        periods_net = partial(D.ConvNet, out_size=1, capacity=capacity, n_layers=4, stride=4,
                              conv=nn.Conv2d, kernel_size=(5, 1))
        scales_net = partial(D.ConvNet, out_size=1, capacity=capacity, n_layers=4, stride=4,
                             conv=nn.Conv1d, kernel_size=15)
        disc = D.CombineDiscriminators([
            partial(D.MultiPeriodDiscriminator, periods=[2, 3, 5, 7, 11], convnet=periods_net),
            partial(D.MultiScaleDiscriminator, n_discriminators=3, convnet=scales_net),
        ], n_channels=NC)
    finally:
        D.normalization = norm
    x = make_input(2 * B, NC, T + 3, seed=13)
    sd = {"discriminator." + k: v.detach().clone() for k, v in disc.state_dict().items()}
    xg = x.clone().requires_grad_(True)
    feats = disc(xg)
    feats_o = O.combine_discriminators_v2(x, sd)
    assert len(feats) == len(feats_o) == 8
    for i, (fa, fb) in enumerate(zip(feats_o, feats)):
        for j, (a, b) in enumerate(zip(fa, fb)):
            assert a.shape == b.shape
            check(f"disc {i}.{j} {tuple(b.shape)}", a, b, 1e-6)
    real = [[f[:B] for f in s] for s in feats]
    fake = [[f[B:] for f in s] for s in feats]
    fm_r, ld_r, la_r = 0., 0., 0.
    for sr, sf in zip(real, fake):              # rave/model.py:348-379
        fm_r = fm_r + sum(map(partial(R.core.mean_difference, norm="L1", relative=True),
                              sr[1:], sf[1:])) / len(sr[1:])
        d_, a_ = R.core.hinge_gan(sr[-1], sf[-1])
        ld_r, la_r = ld_r + d_, la_r + a_
    fm_r = fm_r / len(real)
    fm, ld, la = O.gan_losses(feats_o, 1, True)
    check("feature matching", fm, fm_r, 1e-6)
    check("loss_dis", ld, ld_r, 1e-6)
    check("loss_adv", la, la_r, 1e-6)
    pp = dict(disc.named_parameters(prefix="discriminator"))
    names = sorted(pp)
    grads = torch.autograd.grad(fm_r + ld_r + la_r, [xg] + [pp[n] for n in names])
    gflat = torch.cat([g.reshape(-1) for g in grads[1:]])
    fx = dict(capacity=capacity, n_channels=NC, state_dict=sd, x=x,
              features=[[ST.sample(f.detach(), FEATURE_SAMPLE, seed=100 * i + j) for j, f in enumerate(s)]
                        for i, s in enumerate(feats)],
              fm=fm_r.detach(), loss_dis=ld_r.detach(), loss_adv=la_r.detach(), grad_x=grads[0].detach(),
              grad_keys=names, grad_sample=ST.sample(gflat.detach(), GRAD_SAMPLE, seed=7))
    torch.save(fx, os.path.join(GOLDEN, "discriminator_v2_stereo.pt"))


def golden_training_step_stereo(R, kind, B=2, T=32768, param_seed=43, disc_capacity=4):
    """The reference's OWN RAVE.training_step (rave/model.py:288-424) at n_channels = 2 in phase 2: a D-step (batch_idx 0)
    and a G-step (batch_idx 1), each from the same seeded parameters."""
    print(f"RAVE.training_step {kind} stereo (phase-2 D, phase-2 G)")
    set_padding_mode("centered")
    v3 = kind == "v3"
    cfg = O.ArchConfig(capacity=8, latent_size=16, n_channels=NC, activation="snake" if v3 else "leaky", adain=v3)
    torch.manual_seed(0)
    m = build_ref_rave_stereo(R, cfg, disc_capacity, update_discriminator_every=2, kind=kind)
    shapes = [(k, tuple(v.shape)) for k, v in m.named_parameters() if not k.startswith("pqmf.")]
    m.load_state_dict(ST.seeded_params(shapes, param_seed), strict=False)
    m.train()
    m.warmed_up = True
    rf = (1024, 512)
    m.receptive_field[0], m.receptive_field[1] = rf
    opts = m.configure_optimizers()
    gen_opt, dis_opt = opts[0]["optimizer"], opts[1]["optimizer"]
    logs = {}
    m.optimizers = lambda: (gen_opt, dis_opt)
    m.log = lambda k, v: logs.__setitem__(k, v.detach().clone() if torch.is_tensor(v) else torch.tensor(float(v)))
    m.log_dict = lambda d: [m.log(k, v) for k, v in d.items()]
    sd0 = {k: v.detach().clone() for k, v in m.state_dict().items()}
    Lz = T // cfg.n_band
    for r in cfg.ratios:
        Lz //= r
    steps = []
    for name, batch_idx, seed in (("phase2_dis", 0, 121), ("phase2_gen", 1, 122)):
        m.load_state_dict(sd0)
        x = ST.step_batch(B, T, seed)
        torch.manual_seed(seed)
        eps = torch.randn(B, cfg.latent_size, Lz)
        assert torch.equal(eps, ST.step_eps(B, cfg.latent_size, Lz, seed))
        torch.manual_seed(seed)
        logs.clear()
        m.training_step(x.clone(), batch_idx)
        dis = batch_idx % m.update_discriminator_every == 0
        grads = {k: p.grad.detach().clone() for k, p in m.named_parameters()
                 if p.grad is not None and k.startswith("discriminator.") == dis
                 and not k.startswith(("encoder.", "pqmf."))}
        keys = sorted(grads)
        steps.append(dict(name=name, batch_idx=batch_idx, seed=seed, logs={k: v.clone() for k, v in logs.items()},
                          grad_keys=keys, grad_sample=ST.sample(torch.cat([grads[k].reshape(-1) for k in keys]),
                                                                GRAD_SAMPLE, seed=seed)))
        print("  ", name, {k: round(float(v), 6) for k, v in logs.items()})
        losses, ldis = ST.train_step_losses(x, sd0, cfg, eps, kind, receptive_field=rf)
        for k, v in losses.items():
            check(f"{name} {k}", v, logs[k], 2e-6)
        check(f"{name} loss_dis", ldis, logs["loss_dis"], 2e-6)
    torch.save(dict(kind=kind, cfg=vars(cfg), B=B, T=T, disc_capacity=disc_capacity,
                    update_discriminator_every=m.update_discriminator_every, receptive_field=rf,
                    param_shapes=shapes, param_seed=param_seed, hk=sd0["pqmf.hk"], steps=steps),
               os.path.join(GOLDEN, f"training_step_{kind}_stereo_tiny.pt"))


def golden_state_dict_keys_stereo(R):
    """Key lists of the full-size v2 and v3 rave.RAVE at n_channels = 2."""
    print("state_dict key contract (v2 / v3 stereo, full size)")
    out = {}
    for name, cfg, kind in (("rave_v2", O.ArchConfig(n_channels=NC), "v2"),
                            ("rave_v3", O.ArchConfig(activation="snake", adain=True, n_channels=NC), "v3")):
        torch.manual_seed(0)
        m = build_ref_rave_stereo(R, cfg, disc_capacity=cfg.capacity, kind=kind)
        out[name] = {k: (tuple(v.shape), str(v.dtype)) for k, v in m.state_dict().items()}
        print(f"  {name}: {len(out[name])} keys")
        del m
    torch.save(out, os.path.join(GOLDEN, "state_dict_keys_stereo.pt"))


def main():
    os.makedirs(GOLDEN, exist_ok=True)
    R = load_reference()
    norm = R.blocks.normalization
    R.blocks.normalization = lambda m, mode="weight_norm": norm(m, mode)  # configs/v1.gin:41
    golden_discriminator_v2_stereo(R)
    golden_training_step_stereo(R, "v2")
    golden_training_step_stereo(R, "v3")
    golden_state_dict_keys_stereo(R)
    for f in ("discriminator_v2_stereo.pt", "training_step_v2_stereo_tiny.pt", "training_step_v3_stereo_tiny.pt",
              "state_dict_keys_stereo.pt"):
        print(f, os.path.getsize(os.path.join(GOLDEN, f)), "bytes")


if __name__ == "__main__":
    sys.exit(main())

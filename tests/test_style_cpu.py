"""CPU: the v3 style transfer -- `update_adain`'s flag / reset semantics against the reference's fixture
(tests/golden/style_v3_tiny.pt, oracle/make_golden_style.py), the oracle restatement of eval-mode AdaIN against the same
fixture, and which chains the engine plans with AdaIN and which it leaves to the module path."""
import os

import pytest
import torch
import torch.nn as nn

from oracle import style_oracle as S
from rave_b200 import blocks, cc, configs, engine
from tests.conftest import GOLDEN, rel_l2


@pytest.fixture(scope="module")
def fixture():
    return S.load_fixture(os.path.join(GOLDEN, "style_v3_tiny.pt"))


def _tiny_v3(g):
    torch.manual_seed(0)
    _, enc, dec = configs.make_autoencoder("v3", capacity=g["capacity"], latent_size=g["latent_size"],
                                           ratios=g["ratios"])
    holder = nn.Module()
    holder.encoder, holder.decoder = enc, dec
    shapes = [(k, tuple(v.shape)) for k, v in holder.named_parameters()]
    holder.load_state_dict(S.style_params(shapes, g["param_seed"]), strict=False)
    return holder.eval()


def _adain_modules(root):
    return {k + ".": m for k, m in root.named_modules() if isinstance(m, blocks.AdaptiveInstanceNormalization)}


def test_update_adain_matches_the_export_step_for_step(fixture):
    """Before step i the buffers are the reference's after step i-1; blocks.update_adain then writes the flags and
    resets, and the reference's forward of step i can only have advanced the counter of the statistics it learned."""
    g = fixture
    B = g["B"]
    holder = _tiny_v3(g)
    mods = _adain_modules(holder)
    assert len(mods) == 22
    prev = S.snapshot(holder.state_dict(), B)          # as constructed: the reference's sequence starts there too
    for step in g["steps"]:
        for p, m in mods.items():
            for name in S.BUFFERS:
                getattr(m, name)[:B].copy_(prev[p + name])
        kw = step["update_adain"]
        assert blocks.update_adain(holder, **kw) == 22
        after = step["buffers"]
        for p, m in mods.items():
            assert m.learn_y.item() == after[p + "learn_y"].item() == float(kw.get("learn_target", False))
            assert m.learn_x.item() == after[p + "learn_x"].item() == float(kw.get("learn_source", False))
            for s, reset, learned in (("y", kw.get("reset_target"), m.learn_y.item() != 0),
                                      ("x", kw.get("reset_source"), m.learn_y.item() == 0 and m.learn_x.item() != 0)):
                n_ours, n_ref = getattr(m, "num_update_" + s).item(), after[p + "num_update_" + s].item()
                if reset:
                    assert n_ours == 0
                    assert torch.equal(getattr(m, "mean_" + s), torch.zeros_like(getattr(m, "mean_" + s)))
                    assert torch.equal(getattr(m, "std_" + s), torch.ones_like(getattr(m, "std_" + s)))
                assert n_ref == n_ours + (1 if learned else 0), (p, s)
                if not learned:       # the forward left these statistics alone
                    assert torch.equal(getattr(m, "mean_" + s)[:B], after[p + "mean_" + s])
                    assert torch.equal(getattr(m, "std_" + s)[:B], after[p + "std_" + s])
        prev = after


def test_update_adain_on_models_without_adain():
    _, enc, dec = configs.make_autoencoder("v2", capacity=8, latent_size=8)
    assert blocks.update_adain(enc) == 0 and blocks.update_adain(dec) == 0
    m = configs.build_rave("v2", capacity=8, latent_size=8, disc_capacity=4)
    assert m.update_adain(learn_target=True) == 0


def test_rave_update_adain_counts_every_layer():
    m = configs.build_rave("v3", capacity=8, latent_size=8, disc_capacity=4)
    assert m.update_adain(learn_target=True, reset_source=True) == 22
    ads = [x for x in m.modules() if isinstance(x, blocks.AdaptiveInstanceNormalization)]
    assert all(a.learn_y.item() == 1 and a.learn_x.item() == 0 for a in ads)
    assert m.update_adain() == 22
    assert all(a.learn_y.item() == 0 for a in ads)


def test_oracle_reproduces_the_fixture(fixture):
    g = fixture
    holder = _tiny_v3(g)
    sd = {k: v.detach().clone() for k, v in holder.state_dict().items()}
    cfg = S.style_cfg(g["capacity"], g["latent_size"])
    got = S.run_sequence(sd, g["inputs"], g["latents"], cfg)
    for i, ((e, y, bufs), step) in enumerate(zip(got, g["steps"])):
        assert rel_l2(e, step["encoder"]) < 1e-4, i          # fp32 against fp32 in another summation order
        assert rel_l2(y, step["decoder"]) < 1e-4, i
        for k, v in step["buffers"].items():
            if k.rsplit(".", 1)[-1] in ("learn_x", "learn_y", "num_update_x", "num_update_y"):
                assert torch.equal(bufs[k], v), (i, k)
            else:
                assert rel_l2(bufs[k], v) < 1e-4, (i, k)
    # the sequence is not the identity: the transfer moves both outputs, resetting the target undoes it
    steps = g["steps"]
    assert rel_l2(steps[3]["decoder"], steps[4]["decoder"]) > 1e-2
    assert rel_l2(steps[3]["encoder"], steps[4]["encoder"]) > 1e-2
    assert rel_l2(steps[2]["encoder"], steps[4]["encoder"]) > 1e-2      # learn_source already transfers


def _chain_adains(seq):
    specs = engine.plan_sequential(list(seq))
    return None if specs is None else sum(s.adain is not None for s in specs)


def test_plan_attaches_every_adain_of_the_v3_chains():
    _, enc, dec = configs.make_autoencoder("v3", capacity=8, latent_size=8)
    enc.eval(), dec.eval()
    assert _chain_adains(enc.encoder.net) == 11
    assert _chain_adains(dec.net) == 11
    specs = engine.plan_sequential(list(enc.encoder.net))
    for s in specs:
        if s.adain is not None:          # the first conv of a Snake unit: its raw input is the unit's skip
            assert s.pre_act == engine.ops.ACT_SNAKE and s.K == 3
            assert specs[specs.index(s) + 1].res_raw == specs.index(s)
    enc.train(), dec.train()
    assert _chain_adains(enc.encoder.net) == 0
    assert _chain_adains(dec.net) == 0


def test_plan_falls_back_for_leaky_units_with_adain():
    _, enc, dec = configs.make_autoencoder("v2", capacity=8, latent_size=8, adain=True)
    enc.eval(), dec.eval()
    assert engine.plan_sequential(list(enc.encoder.net)) is None
    assert engine.plan_sequential(list(dec.net)) is None
    assert enc.encoder.net._tc_plan() is None
    enc.train()
    assert _chain_adains(enc.encoder.net) == 0


def test_adain_chains_stay_on_the_module_path_under_autograd_x3_and_large_batches():
    _, enc, _ = configs.make_autoencoder("v3", capacity=16, latent_size=16)
    net = enc.encoder.net.eval()
    specs = net._tc_plan()
    x = torch.zeros(2, 16, 64)
    assert not net._adain_ok(specs, x, x3=False)                 # parameters require grad
    with torch.no_grad():
        assert net._adain_ok(specs, x, x3=False)
        assert not net._adain_ok(specs, x, x3=True)
        assert not net._adain_ok(specs, torch.zeros(cc.MAX_BATCH_SIZE + 1, 16, 64), x3=False)
    net.requires_grad_(False)
    assert net._adain_ok(specs, x, x3=False)
    assert not net._adain_ok(specs, x.requires_grad_(True), x3=False)
    # chains without AdaIN are unaffected
    _, enc2, _ = configs.make_autoencoder("v2", capacity=16, latent_size=16)
    assert enc2.encoder.net._adain_ok(enc2.encoder.net.eval()._tc_plan(), x, x3=True)


def test_run_chain_refuses_adain_under_autograd():
    _, enc, _ = configs.make_autoencoder("v3", capacity=16, latent_size=16)
    specs = enc.encoder.net.eval()._tc_plan()
    with pytest.raises(engine._lib.RaveB200Error, match="AdaIN"):
        engine.run_chain(torch.zeros(1, 64, 16), specs)


def test_cached_modules_keep_the_module_path():
    cc.use_cached_conv(True)
    try:
        _, enc, dec = configs.make_autoencoder("v3", capacity=8, latent_size=8)
    finally:
        cc.use_cached_conv(False)
    assert enc.encoder.net._cached and dec.net._cached

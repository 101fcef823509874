"""TEST INFRASTRUCTURE -- generates the latent prior's fixtures by EXECUTING THE UNMODIFIED REFERENCE
(rave/prior/{core,residual_block,model}.py, loaded under oracle/ref_loader.py's stubs) and asserts that
oracle/prior_oracle.py reproduces them.  Writes new files only:

    python -m oracle.make_golden_prior

  tests/golden/prior_tiny.pt             a tiny VariationalPrior on a tiny v2 RAVE, parameters from seeded_params: encoder
                                         output, injected eps, classes, logits, loss and every parameter gradient of the
                                         reference's training_step; QuantizedNormal / DiagonalShift; generate(argmax)
  tests/golden/state_dict_keys_prior.pt  keys / shapes of VariationalPrior at the prior_v1.gin bindings on a full-size v2
                                         RAVE, with latent_size given and with it chosen by `fidelity`

Conv biases: scripts/train_prior.py:90 calls gin.clear_config() after building the pretrained RAVE, so v1.gin's
`cc.Conv1d.bias = False` does not reach the prior, and its cc.Conv1d layers take cached-conv's own default.  That
default is nn.Conv1d's bias=True -- a recalled fact about cached-conv 2.5.0 (not installable here), like the padding
constant of SURVEY App. A.  The loader below builds the prior with the stub's bias default switched to True.
"""
import importlib.util
import os
import sys
import types

import torch

from oracle import prior_oracle as P
from oracle import rave_oracle as O
from oracle.make_golden import GOLDEN, build_ref_rave, check, make_input
from oracle.ref_loader import REFERENCE_ROOT, _CCState, load_reference

TINY = dict(resolution=8, res_size=32, skp_size=16, kernel_size=3, cycle_size=2, n_layers=3)
TINY_D = 4
TINY_VAE = dict(capacity=4, latent_size=8)
PARAM_SEED = 1234


def load_reference_prior():
    """The reference's rave.prior package (core, residual_block, model) on top of load_reference()."""
    R = load_reference()
    if hasattr(R, "prior"):
        return R
    pkg = types.ModuleType("rave.prior")
    pkg.__path__ = [os.path.join(REFERENCE_ROOT, "rave", "prior")]
    sys.modules["rave.prior"] = pkg
    for name in ("core", "residual_block", "model"):
        spec = importlib.util.spec_from_file_location("rave.prior." + name,
                                                      os.path.join(REFERENCE_ROOT, "rave", "prior", name + ".py"))
        mod = importlib.util.module_from_spec(spec)
        sys.modules["rave.prior." + name] = mod
        spec.loader.exec_module(mod)
        setattr(pkg, name, mod)
    R.prior = pkg
    return R


def build_ref_prior(R, vae, **kw):
    old = _CCState.bias
    _CCState.bias = True            # gin.clear_config(): cached-conv's own default (see the module docstring)
    try:
        return R.prior.model.VariationalPrior(pretrained_vae=vae, **kw)
    finally:
        _CCState.bias = old


def prior_param_names(m):
    return [k for k, _ in m.named_parameters() if not k.startswith("synth.")]


def golden_tiny(R, B=2, T=32768, seed=5):
    print("prior (tiny)")
    torch.manual_seed(0)
    cfg = O.v2_config(**TINY_VAE)
    vae = build_ref_rave(R, cfg)
    vae_shapes = [(k, tuple(v.shape)) for k, v in vae.named_parameters()]
    vae.load_state_dict(P.seeded_params(vae_shapes, PARAM_SEED), strict=False)
    g = torch.Generator().manual_seed(11)
    L = TINY_VAE["latent_size"]
    pca = torch.linalg.qr(torch.randn(L, L, generator=g))[0]
    lmean = 0.1 * torch.randn(L, generator=g)
    vae.latent_pca.copy_(pca)
    vae.latent_mean.copy_(lmean)
    prior = build_ref_prior(R, vae, latent_size=TINY_D, sr=48000, **TINY)
    shapes = [(k, tuple(v.shape)) for k, v in prior.named_parameters() if not k.startswith("synth.")]
    psd = P.seeded_params(shapes, PARAM_SEED + 1)
    prior.load_state_dict(psd, strict=False)
    assert all(k in psd for k in prior_param_names(prior))
    x = make_input(B, 1, T, seed=41)

    # the reference's own step, its one random draw (reparametrize's randn_like) reconstructed from the seed
    z_enc = vae.encode(x).detach()
    eps = torch.randn(B, L, z_enc.shape[-1], generator=torch.Generator().manual_seed(seed))
    taps = {}
    orig_fwd = prior.forward

    def spy(xin):
        out = orig_fwd(xin)
        taps["x"], taps["logits"] = xin.detach().clone(), out.detach().clone()
        return out
    prior.forward = spy
    prior.log = lambda *a, **k: None          # LightningModule.log: the stub's LightningModule is nn.Module
    torch.manual_seed(seed)
    loss = prior.training_step(x, 0)
    prior.forward = orig_fwd
    params = dict(prior.named_parameters())
    names = prior_param_names(prior)
    grads = torch.autograd.grad(loss, [params[k] for k in names], allow_unused=True)
    grads = {k: (None if g_ is None else g_.detach().clone()) for k, g_ in zip(names, grads)}

    # the restatement reproduces it
    y = P.post_process_latent(z_enc, eps, lmean, pca, TINY_D)
    cls = P.latent_classes(z_enc, eps, lmean, pca, TINY_D, TINY["resolution"])
    check("one-hot input", P.stack_one_hot(cls, TINY["resolution"]), taps["x"], 0.0)
    # no shifted latent lies near a class edge: classes are stable under fp32 reordering
    u = 0.5 * (1 + torch.erf(P.diagonal_shift(y).double() / 2 ** 0.5)) * TINY["resolution"]
    edge = (u - u.round()).abs().min().item()
    print(f"  closest bin edge distance (in classes): {edge:.3e}")
    assert edge > 1e-4
    psd_r = {k: v.detach().requires_grad_(True) for k, v in psd.items()}
    o_taps = {}
    lo = P.loss(cls, psd_r, TINY, TINY_D, o_taps)
    check("logits", o_taps["logits"], taps["logits"], 1e-6)
    check("loss", lo, loss, 1e-6)
    og = torch.autograd.grad(lo, [psd_r[k] for k in names], allow_unused=True)
    for k, g_ in zip(names, og):
        if grads[k] is None:
            assert g_ is None or g_.abs().max() == 0, k
        else:
            check(f"grad {k}", g_, grads[k], 1e-5)

    # QuantizedNormal (dither off) and DiagonalShift
    qn = R.prior.core.QuantizedNormal(TINY["resolution"], dither=False)
    ds = R.prior.core.DiagonalShift()
    zq = torch.randn(B, TINY_D, 9, generator=g)
    q_enc = qn.encode(zq)
    q_dec = qn.decode(q_enc)
    check("quantize", P.stack_one_hot(P.quantize(zq, TINY["resolution"]), TINY["resolution"]), q_enc, 0.0)
    check("dequantize", P.dequantize(P.quantize(zq, TINY["resolution"]), TINY["resolution"]), q_dec, 1e-7)
    s_fwd, s_inv = ds(zq), ds.inverse(zq)
    check("shift", P.diagonal_shift(zq), s_fwd, 0.0)
    check("shift inverse", P.diagonal_shift_inverse(zq), s_inv, 0.0)

    # generate(argmax=True), 4 steps from a random first frame
    g0 = torch.randint(0, TINY["resolution"], (B, TINY_D, 5), generator=g)
    x_gen = P.stack_one_hot(g0, TINY["resolution"])
    with torch.no_grad():
        out_gen = prior.generate(x_gen.clone(), argmax=True)
        check("generate", P.generate(x_gen, psd, TINY, TINY_D), out_gen, 0.0)

    fx = dict(prior_cfg=TINY, D=TINY_D, vae_cfg=TINY_VAE, B=B, T=T, param_seed=PARAM_SEED,
              vae_param_shapes=vae_shapes, prior_param_shapes=shapes, latent_pca=pca, latent_mean=lmean,
              x=x, z=z_enc, eps=eps, classes=cls, logits=taps["logits"], loss=loss.detach(), grads=grads,
              min_receptive_field=prior.min_receptive_field, model_ratio=prior.get_model_ratio(),
              quant_in=zq, quant_enc=q_enc, quant_dec=q_dec, shift_fwd=s_fwd, shift_inv=s_inv,
              gen_in=x_gen, gen_out=out_gen)
    torch.save(fx, os.path.join(GOLDEN, "prior_tiny.pt"))


def golden_keys(R):
    print("prior state_dict keys (prior_v1 on v2)")
    torch.manual_seed(0)
    vae = build_ref_rave(R, O.v2_config(), disc_capacity=96)
    out = {}
    prior = build_ref_prior(R, vae, latent_size=16, sr=48000, **P.PRIOR_V1)
    out["latent_size_16"] = {k: tuple(v.shape) for k, v in prior.state_dict().items()}
    out["min_receptive_field"] = prior.min_receptive_field
    fid = torch.linspace(0.02, 1.0, 128)
    vae.fidelity.copy_(fid)
    prior_f = build_ref_prior(R, vae, fidelity=0.9, sr=48000, **P.PRIOR_V1)
    out["fidelity"] = dict(buffer=fid, value=0.9, latent_size=prior_f.latent_size,
                           shapes={k: tuple(v.shape) for k, v in prior_f.state_dict().items()})
    print(f"  {len(out['latent_size_16'])} keys; fidelity .9 -> latent_size {prior_f.latent_size}; "
          f"min_receptive_field {prior.min_receptive_field}")
    torch.save(out, os.path.join(GOLDEN, "state_dict_keys_prior.pt"))


def main():
    R = load_reference_prior()
    torch.set_grad_enabled(True)
    golden_tiny(R)
    golden_keys(R)


if __name__ == "__main__":
    main()

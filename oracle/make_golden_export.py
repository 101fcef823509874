"""TEST INFRASTRUCTURE -- generates the fixture of the exported model's latent arithmetic by EXECUTING THE UNMODIFIED
REFERENCE: the post / pre-processing methods of `VariationalScriptedRAVE`, `DiscreteScriptedRAVE`,
`WasserteinScriptedRAVE` and `SphericalScriptedRAVE`, and `ScriptedRAVE.decode`'s `channels` handling
(scripts/export.py:75-409), loaded under the stubs of oracle/ref_loader.py plus stubs for nn_tilde, absl.flags and the
modules export.py imports but these methods never call.  Objects are made with `__new__` and given only the attributes
the methods read.  Everything runs in float64 (the methods follow the input's dtype through `type_as`).  Writes a new
file only:

    python -m oracle.make_golden_export

  tests/golden/export_latent.pt   per case: the inputs, the eps / noise the reference drew (recorded from its
                                  torch.randn_like / torch.randn calls) and the reference's float64 outputs; the
                                  latent_size rule on a few fidelity curves; `channels` decodes at B = 1 through a fixed
                                  transposed-conv stand-in of the decoder.
"""
import importlib.util
import math
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import export_oracle as EO
from oracle.make_golden import GOLDEN
from oracle.ref_loader import REFERENCE_ROOT, load_reference


def _stubs(ns):
    nn_tilde = types.ModuleType("nn_tilde")

    class Module(nn.Module):
        def register_attribute(self, name, value):
            setattr(self, name, (value,))

        def register_method(self, *a, **k):
            pass

    nn_tilde.Module = Module
    absl = types.ModuleType("absl")
    flags = types.ModuleType("absl.flags")
    for name in ("DEFINE_string", "DEFINE_bool", "DEFINE_float", "DEFINE_integer"):
        setattr(flags, name, lambda *a, **k: None)
    flags.FLAGS = types.SimpleNamespace()
    app = types.ModuleType("absl.app")
    app.run = lambda *a, **k: None
    absl.flags, absl.app = flags, app
    gin = sys.modules["gin"]
    gin.get_bindings = lambda *a, **k: {}
    gin.parse_config_file = lambda *a, **k: None
    gin.clear_config = lambda *a, **k: None
    pkg = sys.modules["rave"]
    pkg.RAVE = ns.model.RAVE
    resampler = types.ModuleType("rave.resampler")
    resampler.Resampler = object
    prior_pkg = types.ModuleType("rave.prior")
    prior_model = types.ModuleType("rave.prior.model")
    prior_model.Prior = nn.Module
    prior_pkg.model = prior_model
    pkg.resampler, pkg.prior = resampler, prior_pkg
    sys.modules.update({"nn_tilde": nn_tilde, "absl": absl, "absl.flags": flags, "absl.app": app,
                        "rave.resampler": resampler, "rave.prior": prior_pkg, "rave.prior.model": prior_model})


def load_export():
    ns = load_reference()
    _stubs(ns)
    spec = importlib.util.spec_from_file_location("rave_export_script",
                                                  os.path.join(REFERENCE_ROOT, "scripts", "export.py"))
    mod = importlib.util.module_from_spec(spec)
    grad = torch.is_grad_enabled()
    spec.loader.exec_module(mod)           # export.py switches autograd off at import
    torch.set_grad_enabled(grad)
    return ns, mod


class _Record:
    """Wraps torch.randn / torch.randn_like while the reference runs: the values pass through and are kept."""

    def __init__(self):
        self.draws = []

    def __enter__(self):
        self._randn, self._like = torch.randn, torch.randn_like

        def randn(*a, **k):
            v = self._randn(*a, **k)
            self.draws.append(v.clone())
            return v

        def randn_like(*a, **k):
            v = self._like(*a, **k)
            self.draws.append(v.clone())
            return v
        torch.randn, torch.randn_like = randn, randn_like
        return self

    def __exit__(self, *a):
        torch.randn, torch.randn_like = self._randn, self._like
        return False


def _obj(cls, **attrs):
    o = cls.__new__(cls)
    nn.Module.__init__(o)
    for k, v in attrs.items():
        setattr(o, k, v)
    return o


def _pca(L, g):
    q, _ = torch.linalg.qr(torch.randn(L, L, generator=g, dtype=torch.float64))
    return q


def variational_cases(ns, E):
    out = []
    for name, B, L, T, l, seed in (("v_l4", 2, 8, 5, 4, 1), ("v_full", 1, 6, 7, 6, 2), ("v_l1", 3, 4, 3, 1, 3)):
        g = torch.Generator().manual_seed(seed)
        z = torch.randn(B, 2 * L, T, generator=g, dtype=torch.float64) * 2
        mean = torch.randn(L, generator=g, dtype=torch.float64) * .3
        pca = _pca(L, g)
        enc = ns.blocks.VariationalEncoder(lambda n_channels: nn.Identity())
        o = _obj(E.VariationalScriptedRAVE, encoder=enc, latent_mean=mean, latent_pca=pca, latent_size=l,
                 full_latent_size=L)
        torch.manual_seed(seed)
        with _Record() as r:
            post = o.post_process_latent(z)
        eps = r.draws[0]
        with _Record() as r:
            pre = o.pre_process_latent(post)
        noise = r.draws[0] if l < L else torch.zeros(B, 0, T, dtype=torch.float64)
        assert torch.allclose(EO.variational_post(z, eps, mean, pca, l), post, rtol=1e-12, atol=1e-12), name
        assert torch.allclose(EO.variational_pre(post, noise, mean, pca), pre, rtol=1e-12, atol=1e-12), name
        out.append(dict(name=name, z=z, latent_mean=mean, latent_pca=pca, l=l, eps=eps, post=post, noise=noise,
                        pre=pre))
        print(f"{name:10s} B={B} L={L} T={T} l={l}")
    return out


def discrete_cases(ns, E):
    out = []
    for name, B, D, T, Q, K, n_noise, seed in (("d_small", 2, 8, 6, 3, 16, 4, 11), ("d_odd_k", 1, 12, 9, 4, 37, 0, 12)):
        g = torch.Generator().manual_seed(seed)
        rvq = ns.quantization.ResidualVectorQuantization(num_quantizers=Q, dim=D, codebook_size=K, kmeans_init=False)
        cbs = torch.randn(Q, K, D, generator=g, dtype=torch.float64) / (1 + torch.arange(Q, dtype=torch.float64))[:, None,
                                                                                                                   None]
        for q, layer in enumerate(rvq.layers):
            layer._codebook.embed = cbs[q].clone()
        x = torch.randn(B, D, T, generator=g, dtype=torch.float64) * 1.5
        o = _obj(E.DiscreteScriptedRAVE, encoder=types.SimpleNamespace(rvq=rvq, noise_augmentation=n_noise))
        codes = o.post_process_latent(x)
        # decode input: the codes plus out-of-range and fractional values that the clamp and the truncation handle
        dec_in = codes.clone()
        dec_in[0, 0, 0] = -3.7
        dec_in[0, -1, -1] = K + 5.5
        dec_in[-1, 0, -1] = 2.9
        torch.manual_seed(seed)
        with _Record() as r:
            pre = o.pre_process_latent(dec_in)
        noise = r.draws[0] if n_noise else torch.zeros(B, 0, T, dtype=torch.float64)
        assert torch.equal(EO.rvq_encode(x, cbs).double(), codes), name
        assert torch.allclose(EO.rvq_decode(dec_in, cbs, noise if n_noise else None), pre, rtol=1e-12, atol=1e-12)
        out.append(dict(name=name, x=x, codebooks=cbs, codes=codes, decode_in=dec_in, noise=noise, pre=pre))
        print(f"{name:10s} B={B} D={D} T={T} Q={Q} K={K} noise={n_noise}")
    return out


def wasserstein_cases(E):
    out = []
    for name, B, L, T, n_noise, seed in (("w_noise", 2, 5, 4, 3, 21), ("w_plain", 1, 4, 6, 0, 22)):
        g = torch.Generator().manual_seed(seed)
        z = torch.randn(B, L, T, generator=g, dtype=torch.float64)
        o = _obj(E.WasserteinScriptedRAVE, encoder=types.SimpleNamespace(noise_augmentation=n_noise))
        post = o.post_process_latent(z)
        torch.manual_seed(seed)
        with _Record() as r:
            pre = o.pre_process_latent(post)
        noise = r.draws[0] if n_noise else torch.zeros(B, 0, T, dtype=torch.float64)
        assert torch.equal(post, z) and torch.equal(EO.wasserstein_pre(z, noise if n_noise else None), pre)
        out.append(dict(name=name, z=z, post=post, noise=noise, pre=pre))
    return out


def spherical_cases(E):
    out = []
    for name, B, L, T, seed in (("s_8", 2, 8, 6, 31), ("s_2", 1, 2, 9, 32), ("s_3", 2, 3, 5, 33)):
        g = torch.Generator().manual_seed(seed)
        x = torch.randn(B, L, T, generator=g, dtype=torch.float64)
        x[0, -1, 0] = -abs(x[0, -1, 0])                # reflected last angle
        x[0, -1, 1] = abs(x[0, -1, 1])
        x[-1, :, -1] = 0                               # all-zero frame: NaN angles, in the reference too
        o = _obj(E.SphericalScriptedRAVE)
        angles = o.post_process_latent(x)
        a_in = torch.rand(B, L - 1, T, generator=g, dtype=torch.float64) * 2 - 1
        a_in[0, 0, 0] = 1.75                           # outside [-1, 1): the floor modulo wraps it
        a_in[0, -1, 1] = -1.5
        sphere = o.pre_process_latent(a_in.clone())
        mine = EO.sphere_to_angles(x)
        fin = torch.isfinite(angles)
        assert torch.equal(fin, torch.isfinite(mine)) and torch.allclose(mine[fin], angles[fin], rtol=1e-12,
                                                                         atol=1e-12), name
        assert torch.allclose(EO.angles_to_sphere(a_in), sphere, rtol=1e-12, atol=1e-12), name
        out.append(dict(name=name, x=x, angles=angles, angles_in=a_in, sphere=sphere))
    return out


def fidelity_cases(E):
    """latent_size of VariationalScriptedRAVE.__init__ (export.py:119-123), evaluated by its own two lines."""
    curves = {
        "never_exceeds": (torch.linspace(.1, .9, 16), .95),
        "first_index": (torch.full((16,), .99), .95),
        "non_power_of_two": (torch.linspace(.5, 1., 16), .8),
        "untrained_zero": (torch.zeros(16), .95),
    }
    out = []
    for name, (fid, f) in curves.items():
        size = max(np.argmax(fid.numpy() > f), 1)
        size = 2 ** math.ceil(math.log2(size))
        assert size == EO.latent_size("variational", fid, f), name
        out.append(dict(name=name, fidelity=fid, f=f, latent_size=int(size)))
        print(f"latent_size {name:18s} -> {size}")
    return out


def channels_cases(E):
    """ScriptedRAVE.decode at B = 1 (no pqmf, no resampler, no AdaIN) around a Wasserstein pre-process with noise and
    a transposed-conv decoder stand-in: weight [C, nc, ratio], stride ratio, one extra output sample to crop."""
    out = []
    for name, nc, tc, C, n_noise, ratio, T, seed in (("mono_to_2", 1, 2, 3, 2, 4, 5, 41),
                                                     ("mono_to_3", 1, 3, 2, 1, 2, 6, 42),
                                                     ("stereo_to_4", 2, 4, 3, 2, 4, 4, 43),
                                                     ("stereo_to_1", 2, 1, 3, 2, 2, 5, 44)):
        g = torch.Generator().manual_seed(seed)
        w = torch.randn(C + n_noise, nc, ratio + 1, generator=g, dtype=torch.float64)
        z = torch.randn(1, C, T, generator=g, dtype=torch.float64)

        class Dec(nn.Module):
            def forward(self, x):
                return F.conv_transpose1d(x, w, stride=ratio)

        o = _obj(E.WasserteinScriptedRAVE, encoder=types.SimpleNamespace(noise_augmentation=n_noise), decoder=Dec(),
                 pqmf=None, resampler=None, is_using_adain=False, stereo_mode=False, n_channels=nc,
                 target_channels=tc, decode_params=[1, ratio])
        torch.manual_seed(seed)
        with _Record() as r:
            y = o.decode(z)
        noise = r.draws[0]
        assert y.shape == (1, tc, T * ratio), (name, y.shape)
        out.append(dict(name=name, n_channels=nc, target_channels=tc, weight=w, ratio=ratio, z=z, noise=noise, y=y))
        print(f"channels {name:12s} nc={nc} tc={tc} -> {tuple(y.shape)}")
    return out


def main():
    ns, E = load_export()
    torch.set_grad_enabled(False)
    fixture = {
        "variational": variational_cases(ns, E),
        "discrete": discrete_cases(ns, E),
        "wasserstein": wasserstein_cases(E),
        "spherical": spherical_cases(E),
        "latent_size": fidelity_cases(E),
        "channels": channels_cases(E),
    }
    path = os.path.join(GOLDEN, "export_latent.pt")
    torch.save(fixture, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

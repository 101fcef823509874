"""Writes tests/golden/reference_pins.pt: outputs of the unmodified reference for the modules whose oracle restatements
tests/test_oracle_golden.py and tests/test_quantization_cpu.py pin (PQMF, Descript MPD / MRD / preprocess,
NoiseGeneratorV2, ResidualVectorQuantization).

Parameter sets and feature maps are not stored whole: every parameter is replaced by seeded_state_dict(),
which the test regenerates from the stored key / shape list, and of each Descript feature map only a fixed sample of
elements is kept (sample()).  Run once where the reference sources are available:

    python -m oracle.make_reference_pins
"""
import os

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "reference_pins.pt")


def seeded_state_dict(shapes, seed, scale=0.05):
    """{key: tensor} with N(0, scale^2) values drawn in key order from one CPU generator."""
    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn(tuple(s), generator=g) * scale for k, s in shapes}


def sample(t, n=1024, seed=0):
    """(shape, flat indices, values) of a fixed, seeded sample of at most n elements of t."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.randperm(t.numel(), generator=g)[:n].sort().values
    return tuple(t.shape), idx, t.reshape(-1)[idx].clone()


def _reseed(module, seed):
    shapes = [(k, tuple(v.shape)) for k, v in module.named_parameters()]
    module.load_state_dict(seeded_state_dict(shapes, seed), strict=False)
    return shapes


def _buffers(module):
    return {k: v.clone() for k, v in module.named_buffers()}


def rvq_run(mod, x):
    """Three training-mode passes of mod.ResidualVectorQuantization (k-means init, EMA updates, dead-code revival):
    every output, then the final state."""
    if x is None:
        return None
    torch.manual_seed(123)
    rvq = mod.ResidualVectorQuantization(num_quantizers=4, dim=8, codebook_size=16)
    rvq.train()
    res = []
    for step in range(3):
        q, loss, idx = rvq(x * (1 + step))
        res += [q.detach().clone(), loss.detach().clone(), idx.clone()]
    return res + [v.clone() for v in rvq.state_dict().values()]


@torch.no_grad()
def main():
    from oracle.ref_loader import load_reference
    R = load_reference()
    pins = {}

    torch.manual_seed(0)
    p = R.pqmf.CachedPQMF(attenuation=100, n_band=16)
    x = torch.randn(1, 1, 4096)
    y = p(x)
    pins["pqmf"] = dict(hk=p.hk.clone(), x=x, y=y, x_rec=p.inverse(y))

    mpd = R.descript_discriminator.MPD(3)
    shapes = _reseed(mpd, 1)
    x = torch.randn(2, 1, 999)
    yp = torch.randn(2, 1, 500)
    pins["descript_mpd"] = dict(shapes=shapes, seed=1, buffers=_buffers(mpd), x=x, out=[sample(t) for t in mpd(x)], y=yp,
                                preprocessed=R.descript_discriminator.DescriptDiscriminator().preprocess(yp))

    mrd = R.descript_discriminator.MRD(512)
    shapes = _reseed(mrd, 2)
    x = torch.randn(2, 1, 4000)
    pins["descript_mrd"] = dict(shapes=shapes, seed=2, buffers=_buffers(mrd), x=x, out=[sample(t) for t in mrd(x)])

    torch.manual_seed(0)
    ng = R.blocks.NoiseGeneratorV2(in_size=48, hidden_size=64, data_size=16, ratios=[2, 2, 2], noise_bands=32)
    shapes = _reseed(ng, 3)
    x = torch.randn(2, 48, 256)
    torch.manual_seed(77)
    pins["noise_generator_v2"] = dict(shapes=shapes, seed=3, buffers=_buffers(ng), x=x, y=ng(x))

    with torch.enable_grad():
        pins["rvq"] = dict(x=torch.randn(3, 8, 40))
        pins["rvq"]["out"] = rvq_run(R.quantization, pins["rvq"]["x"])

    torch.save(pins, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()

"""TEST INFRASTRUCTURE -- generates the fixture of the export's resampler by EXECUTING THE UNMODIFIED REFERENCE:
rave/resampler.py's `Resampler` and `ScriptedRAVE.encode` / `decode` (scripts/export.py:247-300) around it, loaded under
the stubs of oracle/ref_loader.py and oracle/make_golden_export.py.  Objects are made with `__new__` and given only the
attributes the methods read; the encoder and decoder are fixed strided-conv stand-ins.  `set_padding_mode("causal")`
plays configs/causal.gin.  Writes a new file only:

    python -m oracle.make_golden_resampler

  tests/golden/resampler.pt   per ratio (2, 3) and padding mode: the float32 taps of `downsample` / `upsample`, seeded
                              mono and stereo inputs (lengths that are and are not multiples of the ratio) and both
                              directions run in float32 and float64; the construction failure of ratios 4-8; the
                              encode / decode order, crop and encode ratio of ScriptedRAVE at ratios 2 and 3.
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import resampler_oracle as RO
from oracle.make_golden import GOLDEN
from oracle.make_golden_export import _obj, load_export
from oracle.ref_loader import REFERENCE_ROOT, set_padding_mode

SR = 44100
ENC_STRIDE = 64           # stand-in encoder: one latent frame per 64 model-rate samples
LATENT = 3


def load_resampler():
    ns, E = load_export()
    path = os.path.join(REFERENCE_ROOT, "rave", "resampler.py")
    spec = importlib.util.spec_from_file_location("rave.resampler", path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules["rave.resampler"] = mod
    spec.loader.exec_module(mod)
    sys.modules["rave"].resampler = mod
    return ns, E, mod


def _signals(ratio, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for shape in ((1, 1, 60 * ratio), (2, 1, 97 * ratio + 1), (2, 2, 71 * ratio), (1, 2, 53 * ratio + ratio - 1)):
        out.append(torch.randn(*shape, generator=g, dtype=torch.float64) * .5)
    return out


def direction_cases(R):
    out = []
    for mode in ("centered", "causal"):
        set_padding_mode(mode)
        for ratio in (2, 3):
            rs = R.Resampler(ratio * SR, SR)
            down_w = rs.downsample.weight.detach().clone()
            up_w = rs.upsample.weight.detach().clone()
            assert down_w.dtype == up_w.dtype == torch.float32
            bank = RO.phase_bank(down_w.reshape(-1).double().numpy(), ratio)
            assert np.array_equal(bank, up_w[:, 0].double().numpy()), (mode, ratio)
            assert rs.downsample._pad == RO.get_padding(down_w.shape[-1], mode)
            assert rs.upsample._pad == RO.get_padding(up_w.shape[-1], mode)
            case = dict(mode=mode, ratio=ratio, down_weight=down_w, up_weight=up_w, down_pad=rs.downsample._pad,
                        up_pad=rs.upsample._pad, x=[], down32=[], down64=[], up32=[], up64=[])
            rs64 = R.Resampler(ratio * SR, SR).double()
            for x in _signals(ratio, 100 * ratio + (mode == "causal")):
                d32 = rs.to_model_sampling_rate(x.float())
                u32 = rs.from_model_sampling_rate(x.float())
                d64 = rs64.to_model_sampling_rate(x)
                u64 = rs64.from_model_sampling_rate(x)
                assert d64.shape[-1] == -(-x.shape[-1] // ratio) and u64.shape[-1] == x.shape[-1] * ratio
                assert np.allclose(RO.down(x.numpy(), down_w.reshape(-1).double().numpy(), ratio, mode), d64.numpy(),
                                   rtol=0, atol=1e-12)
                assert np.allclose(RO.up(x.numpy(), bank, mode), u64.numpy(), rtol=0, atol=1e-12)
                for k, v in (("x", x), ("down32", d32), ("down64", d64), ("up32", u32), ("up64", u64)):
                    case[k].append(v.clone())
            print(f"{mode:8s} ratio {ratio}: down {tuple(down_w.shape)} pad {rs.downsample._pad}, "
                  f"up {tuple(up_w.shape)} pad {rs.upsample._pad}, rows sum {up_w.sum((1, 2)).tolist()}")
            out.append(case)
    set_padding_mode("centered")
    return out


def failure_cases(R):
    out = []
    for ratio in range(4, 9):
        try:
            R.Resampler(ratio * SR, SR)
        except RuntimeError as e:           # reshape(-1, ratio) of a length that ratio does not divide
            out.append(dict(ratio=ratio, error=type(e).__name__, message=str(e)))
            print(f"ratio {ratio}: {type(e).__name__}: {e}")
            continue
        raise AssertionError(f"ratio {ratio} was built")
    return out


def scripted_cases(R, E):
    """ScriptedRAVE.encode / decode with the resampler (a Wasserstein model without noise: its latent processing is the
    identity), a stand-in encoder conv(stride ENC_STRIDE) on the input padded up to a multiple of ENC_STRIDE and a
    stand-in decoder conv_transpose(stride ENC_STRIDE, one extra sample), and the encode ratio taken by
    ScriptedRAVE.__init__'s probe: 2^14 // encode(zeros(1, n_channels, 2^14)).shape[-1]."""
    out = []
    for ratio in (2, 3):
        for nc in (1, 2):
            g = torch.Generator().manual_seed(10 * ratio + nc)
            we = torch.randn(LATENT, nc, ENC_STRIDE, generator=g, dtype=torch.float64) / ENC_STRIDE
            wd = torch.randn(LATENT, nc, ENC_STRIDE + 1, generator=g, dtype=torch.float64)

            class Enc(nn.Module):
                def forward(self, x):
                    return F.conv1d(F.pad(x, (0, (-x.shape[-1]) % ENC_STRIDE)), we, stride=ENC_STRIDE)

            class Dec(nn.Module):
                def forward(self, z):
                    return F.conv_transpose1d(z, wd, stride=ENC_STRIDE)

            rs = R.Resampler(ratio * SR, SR).double()
            o = _obj(E.WasserteinScriptedRAVE, encoder=Enc(), decoder=Dec(), pqmf=None, spectrogram=None,
                     resampler=rs, input_mode="raw", is_using_adain=False, stereo_mode=False, n_channels=nc,
                     target_channels=nc)
            o.encoder.noise_augmentation = 0
            x_len = 2 ** 14
            z = o.encode(torch.zeros(1, nc, x_len, dtype=torch.float64))
            ratio_encode = x_len // z.shape[-1]
            o.decode_params = [1, ratio_encode]
            x = torch.randn(2, nc, 9 * ENC_STRIDE * ratio + 5, generator=g, dtype=torch.float64) * .5
            z = o.encode(x)
            y = o.decode(z)
            assert y.shape[-1] == z.shape[-1] * ratio_encode
            out.append(dict(ratio=ratio, n_channels=nc, enc_weight=we, dec_weight=wd, enc_stride=ENC_STRIDE,
                            encode_ratio=ratio_encode, x=x, z=z, y=y))
            print(f"ScriptedRAVE ratio {ratio} n_channels {nc}: encode ratio {ratio_encode} "
                  f"({ratio} x {ENC_STRIDE} = {ratio * ENC_STRIDE}), x {tuple(x.shape)} -> z {tuple(z.shape)} -> "
                  f"y {tuple(y.shape)}")
    return out


def main():
    ns, E, R = load_resampler()
    torch.set_grad_enabled(False)
    fixture = {
        "sr": SR,
        "directions": direction_cases(R),
        "failures": failure_cases(R),
        "scripted": scripted_cases(R, E),
    }
    path = os.path.join(GOLDEN, "resampler.pt")
    torch.save(fixture, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

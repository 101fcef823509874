"""TEST INFRASTRUCTURE -- generates the fixture of the training-batch transforms by EXECUTING THE UNMODIFIED REFERENCE:
`get_dataset`'s transform list (rave/dataset.py:207-262, with `normalize_signal`, `random_phase_mangle` and the
derivator) and `AudioDataset.__getitem__`'s int16 decode, plus `RandomMute` / `RandomGain` (rave/transforms.py), under
the stubs of oracle/ref_loader.py and a few more for the modules rave/dataset.py imports (udls, tqdm's use is none).
Writes a new file only:

    python -m oracle.make_golden_transforms

  tests/golden/transforms.pt   per case: the seeds of the input and of the reference's RNGs, the options, the recorded
                               draws (crop offset, allpass applied, omega, keep) and the reference's float32 output.
                               The dequantisation noise is the first np.random draw after np.random.seed(seed), so it
                               is regenerated from the seed (the generator checks that it was).

The reference's `random` / `np.random` calls are wrapped to record what they returned; the values pass through.
"""
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np
import torch

from oracle import transforms_oracle as TO
from oracle.make_golden import GOLDEN
from oracle.ref_loader import REFERENCE_ROOT, load_reference

SR = 44100


def _stub_udls():
    udls = types.ModuleType("udls")
    gen = types.ModuleType("udls.generated")
    tr = types.ModuleType("udls.transforms")

    class _Precision:
        INT16 = 1

    class _Buffer:
        def __init__(self, data):
            self.data, self.precision = data, _Precision.INT16

    class AudioExample:
        Precision = _Precision

        def __init__(self, buffers=None):
            self.buffers = buffers or {}

        @staticmethod
        def FromString(s):
            return AudioExample({"waveform": _Buffer(s)})

    gen.AudioExample = AudioExample
    udls.AudioExample = AudioExample
    udls.generated = gen
    udls.transforms = tr
    return {"udls": udls, "udls.generated": gen, "udls.transforms": tr}


def load_dataset_modules():
    ns = load_reference()
    sys.modules.update(_stub_udls())
    lmdb = sys.modules["lmdb"]                    # ref_loader's empty module; dataset.py annotates with this name
    if not hasattr(lmdb, "Environment"):
        lmdb.Environment = object
    pkg = sys.modules["rave"]
    mods = {}
    for name in ("transforms", "dataset"):
        spec = importlib.util.spec_from_file_location("rave." + name, os.path.join(REFERENCE_ROOT, "rave", name + ".py"))
        mod = importlib.util.module_from_spec(spec)
        sys.modules["rave." + name] = mod
        spec.loader.exec_module(mod)
        setattr(pkg, name, mod)
        mods[name] = mod
    return ns, mods["dataset"], mods["transforms"]


def make_input(seed, C, L, kind):
    """Seeded database chunk [C, L]: a few partials + noise at one of three levels (int16), or float32."""
    rng = np.random.default_rng(seed)
    if kind == "silent":
        return np.zeros((C, L), np.int16)
    t = np.arange(L)[None, :]
    f = rng.uniform(50, 3000, (C, 3, 1))
    amp = {"loud": 0.45, "quiet": 0.01, "float": 0.3}[kind]
    x = amp * (np.sin(2 * np.pi * f[:, 0] * t / SR) + 0.5 * np.sin(2 * np.pi * f[:, 1] * t / SR)) / 1.5
    x = x + 0.1 * amp * rng.standard_normal((C, L))
    if kind == "float":
        return x.astype(np.float32)
    return np.clip(np.round(x * 32767), -32768, 32767).astype(np.int16)


# (name, channels, n_signal, L, input kind, normalize, derivative, augmentations, seed)
CASES = [
    ("mono", 1, 4096, 8192, "loud", False, False, (), 11),
    ("mono_skip", 1, 4096, 8192, "loud", False, False, (), 7),
    ("stereo", 2, 5000, 10000, "loud", False, False, (), 12),
    ("stereo_norm", 2, 5000, 10000, "quiet", True, False, (), 13),
    ("mono_norm", 1, 4096, 8192, "loud", True, False, (), 14),
    ("mono_norm_skip", 1, 4096, 8192, "quiet", True, False, (), 23),
    ("norm_derivative_skip", 1, 4096, 8192, "loud", True, True, (), 24),
    ("silent_norm", 1, 3000, 6000, "silent", True, False, (), 15),
    ("derivative", 1, 4096, 8192, "loud", False, True, (), 16),
    ("norm_derivative_stereo", 2, 3000, 6000, "quiet", True, True, (), 17),
    ("mute_gain", 1, 4096, 8192, "loud", False, False, ("gain", "mute"), 18),
    ("mute_gain_b", 1, 4096, 8192, "loud", False, False, ("gain", "mute"), 31),
    ("float32_input", 1, 4096, 4096, "float", False, True, (), 19),
]


def main():
    ns, D, T = load_dataset_modules()
    import random as pyrandom
    rec = {}

    def recording(mod, name, key):
        orig = getattr(mod, name)

        def f(*a, **k):
            v = orig(*a, **k)
            rec.setdefault(key, []).append(v)
            return v
        setattr(mod, name, f)

    recording(T, "randint", "randint")       # RandomCrop
    recording(T, "random", "apply_u")        # RandomApply
    recording(D, "random", "angle_u")        # random_angle

    captured = {}

    class _Capture:
        def __init__(self, db_path, n_signal, sr, transforms, n_channels):
            captured["t"] = transforms

    D.LazyAudioDataset = _Capture
    cases = []
    with tempfile.TemporaryDirectory() as db:
        with open(os.path.join(db, "metadata.yaml"), "w") as f:
            f.write(f"sr: {SR}\nlazy: true\n")
        for name, C, N, L, kind, normalize, derivative, augs, seed in CASES:
            objs = [T.RandomGain() if a == "gain" else T.RandomMute(0.5) for a in augs]
            D.get_dataset(db, SR, N, derivative=derivative, normalize=normalize, augmentations=objs, n_channels=C)
            transform = captured["t"]
            raw = make_input(seed, C, L, kind)
            rec.clear()
            pyrandom.seed(seed)
            np.random.seed(seed)
            torch.manual_seed(seed)
            mute = []
            orig_binomial = np.random.binomial

            def binomial(*a, **k):
                v = orig_binomial(*a, **k)
                mute.append(int(v[0]))
                return v
            np.random.binomial = binomial
            try:
                if raw.dtype == np.int16:
                    ds = D.AudioDataset.__new__(D.AudioDataset)
                    ds._env, ds._keys, ds._audio_key = None, [b"0"], "waveform"
                    ds._transforms, ds._n_channels = transform, C

                    class _Txn:
                        def __enter__(self):
                            return self

                        def __exit__(self, *a):
                            return False

                        def get(self, k):
                            return raw.tobytes()

                    ds._env = types.SimpleNamespace(begin=lambda: _Txn())
                    out = ds[0]
                else:
                    out = transform(raw.copy())
            finally:
                np.random.binomial = orig_binomial
            applied = rec["apply_u"][0] < .8
            omega = TO.random_angle(rec["angle_u"][0], 20, 2000, SR) if applied else 0.0
            draws = (float(rec["randint"][0]), float(applied), float(omega), float(mute[0]) if mute else 1.0)
            np.random.seed(seed)
            noise = np.random.rand(C, N)
            mine = TO.transform_example(raw, N, draws, noise, normalize, derivative)
            assert out.dtype == np.float32 and out.shape == (C, N)
            assert np.array_equal(mine.view(np.int32), out.view(np.int32)), name
            print(f"{name:24s} C={C} N={N} L={L} draws={draws} peak={np.abs(out).max():.3e}")
            cases.append({"name": name, "C": C, "N": N, "L": L, "kind": kind, "normalize": normalize,
                          "derivative": derivative, "augmentations": list(augs), "seed": seed,
                          "draws": torch.tensor(draws, dtype=torch.float64), "out": torch.from_numpy(out.copy())})
    path = os.path.join(GOLDEN, "transforms.pt")
    torch.save({"sr": SR, "numpy": np.__version__, "cases": cases}, path)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()

"""rave_b200 -- H100-native (sm_90a) waveform hot path of acids-ircam/RAVE.

The package mirrors the reference's module surface for the path BASELINE.json names
(`pqmf`, `blocks`, `discriminator`, `descript_discriminator`, `core` losses, `model.RAVE`)
and executes it on hand-written CUDA kernels behind the C ABI of include/rave_b200.h.
There is no CPU / PyTorch fallback: see _lib.py.
"""
from . import cc, ops, pqmf, blocks, discriminator, core, model, configs, engine, prior  # noqa: F401
from .ema import EMA  # noqa: F401
from .model import RAVE, BetaWarmupCallback, WarmupCallback  # noqa: F401
from .configs import build_prior, build_rave  # noqa: F401
from .engine import set_precision, precision  # noqa: F401

__version__ = "0.1.0"

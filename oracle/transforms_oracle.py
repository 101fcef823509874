"""Restatement of the reference's training-batch transforms (get_dataset's transform list, rave/dataset.py:207-262,
rave/transforms.py) in numpy / scipy with explicit draws, following the reference's dtype flow under numpy 2.3: pinned
exactly against tests/golden/transforms.pt (tests/test_transforms_cpu.py) and used as the float64 yardstick of the
device kernel (tests/test_gpu_transforms.py).

One example: raw [C, L] int16 or float32, draws (offset, applied, omega, keep), noise [C, n_signal] float64 in [0, 1).
"""
import numpy as np
from scipy.signal import lfilter


def decode(raw: np.ndarray) -> np.ndarray:
    """AudioDataset.__getitem__ (rave/dataset.py:76-77): float32 division by 32767; float32 passes through."""
    if raw.dtype == np.int16:
        return raw.astype(np.float32) / (2**15 - 1)
    return raw.astype(np.float32)


def pole_to_z_filter(omega, amplitude=.99):
    """rave/dataset.py:281-285"""
    z0 = amplitude * np.exp(1j * omega)
    a = [1, -2 * np.real(z0), abs(z0)**2]
    b = [abs(z0)**2, -2 * np.real(z0), 1]
    return b, a


def random_angle(u, min_f=20, max_f=2000, sr=44100):
    """random_angle (rave/dataset.py:273-278) of the uniform u its random() returned."""
    min_f = np.log(min_f)
    max_f = np.log(max_f)
    rand = np.exp(u * (max_f - min_f) + min_f)
    return 2 * np.pi * rand / sr


def _log10_f32_rounded(p):
    return np.float32(np.log10(np.float64(p)))


def normalize_signal(x, max_gain_db=30, device_log10=False):
    """rave/dataset.py:196-204.  device_log10: the float32 log10 and power correctly rounded (through float64), as the
    device computes them, instead of numpy's float32 loops (whose SIMD log10 is host-dependent, DESIGN §5.9)."""
    peak = np.max(abs(x))
    if peak == 0:
        return x
    if device_log10 and x.dtype == np.float32:
        log_peak = 20 * _log10_f32_rounded(peak)
    else:
        log_peak = 20 * np.log10(peak)
    log_gain = min(max_gain_db, -log_peak)
    if device_log10 and x.dtype == np.float32 and isinstance(log_gain, np.float32):
        gain = np.float32(10.0 ** np.float64(log_gain / 20))
    else:
        gain = 10**(log_gain / 20)
    return x * gain


def transform_example(raw, n_signal, draws, noise, normalize=False, derivative=False, device_log10=False):
    offset, applied, omega, keep = draws
    x = decode(raw)
    offset = int(offset)
    x = x[..., offset:offset + n_signal].copy()
    if applied:
        b, a = pole_to_z_filter(omega, .99)
        x = lfilter(b, a, x)
    x += noise / 2**16                       # in place: float32 stays float32
    if normalize:
        x = normalize_signal(x, device_log10=device_log10)
    if derivative:
        x = lfilter([.5, -.5], [1], x)
    x = x * np.array([int(keep)])            # RandomMute's int64 mask (keep = 1 without one)
    return x.astype(np.float32)


def transform_batch(raw, n_signal, draws, noise, normalize=False, derivative=False, device_log10=False):
    """raw [B, C, L], draws [B, 4], noise [B, C, n_signal] -> [B, C, n_signal] float32"""
    return np.stack([transform_example(raw[i], n_signal, draws[i], noise[i], normalize, derivative, device_log10)
                     for i in range(raw.shape[0])])

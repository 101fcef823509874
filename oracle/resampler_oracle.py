"""Float64 restatement of the export's resampler (rave/resampler.py) in its phase-bank form, pinned to the reference by
tests/test_resampler_cpu.py against tests/golden/resampler.pt:

    y[r, i P + p] = sum_{k < K} W[p, k] x[r, i S + k - pad_l],   x = 0 outside the row,

down (`to_model_sampling_rate`): W = filt[None], P = 1, S = ratio; up (`from_model_sampling_rate`): W = the polyphase
bank, P = ratio, S = 1.  `pad` is cached_conv's get_padding of the conv's kernel size (stride ignored)."""
import numpy as np


def get_padding(kernel_size: int, mode: str = "centered"):
    if kernel_size == 1:
        return (0, 0)
    p = kernel_size
    return ((p - 1) // 2, p // 2) if mode == "centered" else (p - 1, 0)


def phase_bank(filt: np.ndarray, ratio: int) -> np.ndarray:
    """filt [K] -> [ratio, K']: phase p holds taps p, p + ratio, ... of the filter left-padded by K % ratio, and the rows
    are left-padded by one zero when their length is even."""
    f = np.concatenate([np.zeros(len(filt) % ratio), filt])
    if len(f) % ratio:
        raise ValueError(f"a {len(filt)}-tap filter does not split into {ratio} phases")
    bank = f.reshape(-1, ratio).T
    if bank.shape[1] % 2 == 0:
        bank = np.concatenate([np.zeros((ratio, 1)), bank], 1)
    return bank


def fir(x, W, stride: int, pad):
    """x [..., L], W [P, K] -> y [..., n P] in float64 (n = (L + pad_l + pad_r - K) // stride + 1); also returns
    sum_k |W[p, k] x_k| per output, the scale of the precision bound."""
    x = np.asarray(x, dtype=np.float64)
    W = np.asarray(W, dtype=np.float64)
    P, K = W.shape
    L = x.shape[-1]
    xp = np.concatenate([np.zeros(x.shape[:-1] + (pad[0],)), x, np.zeros(x.shape[:-1] + (pad[1],))], -1)
    n = (L + pad[0] + pad[1] - K) // stride + 1
    idx = np.arange(n)[:, None] * stride + np.arange(K)[None, :]          # [n, K]
    win = xp[..., idx]                                                    # [..., n, K]
    y = np.einsum("...nk,pk->...np", win, W)
    a = np.einsum("...nk,pk->...np", np.abs(win), np.abs(W))
    return y.reshape(x.shape[:-1] + (n * P,)), a.reshape(x.shape[:-1] + (n * P,))


def down(x, filt, ratio: int, mode: str = "centered"):
    return fir(x, np.asarray(filt)[None], ratio, get_padding(len(filt), mode))[0]


def up(x, bank, mode: str = "centered"):
    return fir(x, bank, 1, get_padding(np.asarray(bank).shape[1], mode))[0]


def bound(y32, scale, K: int):
    """The kernel's precision contract per output: one float32 ulp of the result plus K 2^-24 sum_k |W x|."""
    y32 = np.asarray(y32, dtype=np.float32)
    ulp = np.spacing(np.abs(y32)).astype(np.float64)
    return ulp + K * 2.0 ** -24 * np.asarray(scale)

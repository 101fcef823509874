"""PQMF analysis / synthesis -- module surface of rave/pqmf.py (`PQMF`, `CachedPQMF`) on the
sm_90a kernels of csrc/pqmf.cu.

Filter design (host side, once at init; rave/pqmf.py:32-89) is numpy/scipy exactly as the
reference does it, written against the current scipy API (`firwin(fs=2*pi)` is scipy-1.10's
`nyq=pi`; `scipy.signal.kaiser` moved to `scipy.signal.windows`).  The per-step arithmetic
(rave/pqmf.py:279-294) is one kernel per direction.
"""
import math

import numpy as np
import torch
import torch.nn as nn

from . import cc, ops
from ._lib import RaveB200Error


def reverse_half(x):
    """rave/pqmf.py:13-17 (kept for API parity; the kernels apply the sign internally)."""
    mask = torch.ones_like(x)
    mask[..., 1::2, ::2] = -1
    return x * mask


def center_pad_next_pow_2(x):
    next_2 = 2 ** math.ceil(math.log2(x.shape[-1]))
    pad = next_2 - x.shape[-1]
    return nn.functional.pad(x, (pad // 2, pad // 2 + int(pad % 2)))


def make_odd(x):
    if not x.shape[-1] % 2:
        x = nn.functional.pad(x, (0, 1))
    return x


def get_qmf_bank(h, n_band):
    """Cosine modulation of the prototype (rave/pqmf.py:32-52)."""
    k = torch.arange(n_band).reshape(-1, 1)
    N = h.shape[-1]
    t = torch.arange(-(N // 2), N // 2 + 1)
    p = (-1) ** k * math.pi / 4
    mod = torch.cos((2 * k + 1) * math.pi / (2 * n_band) * t + p)
    return 2 * h * mod


def kaiser_filter(wc, atten, N=None):
    """Kaiser low-pass (rave/pqmf.py:55-70)."""
    from scipy.signal import firwin, kaiserord
    N_, beta = kaiserord(atten, wc / np.pi)
    N_ = 2 * (N_ // 2) + 1
    N = N if N is not None else N_
    return firwin(N, wc, window=("kaiser", beta), scale=False, fs=2 * np.pi)


def loss_wc(wc, atten, M, N):
    h = kaiser_filter(wc, atten, N)
    g = np.convolve(h, h[::-1], "full")
    g = abs(g[g.shape[-1] // 2::2 * M][1:])
    return np.max(g)


def get_prototype(atten, M, N=None):
    from scipy.optimize import fmin
    wc = fmin(lambda w: loss_wc(w, atten, M, N), 1 / M, disp=0)[0]
    return kaiser_filter(wc, atten, N)


class PQMF(nn.Module):
    """Pseudo-QMF bank.  Buffers `hk` [n_band, 2^k] and `h` as in rave/pqmf.py:192-210.

    The polyphase / classic formulations of the reference (pqmf.py:92-176) are alternative
    evaluations of the same operator; on the device there is a single evaluation (the polyphase
    shared-memory kernel), so `polyphase` is accepted and recorded only.  Outputs follow the
    reference's PQMF conventions: `inverse` has no 16-sample delay (CachedPQMF has one)."""

    def __init__(self, attenuation, n_band, polyphase=True, n_channels=1):
        super().__init__()
        h = get_prototype(attenuation, n_band)
        if polyphase:
            power = math.log2(n_band)
            assert power == math.floor(power), \
                "when using the polyphase algorithm, n_band must be a power of 2"
        h = torch.from_numpy(h).float()
        hk = center_pad_next_pow_2(get_qmf_bank(h, n_band))
        self.register_buffer("hk", hk)
        self.register_buffer("h", h)
        self.n_band = n_band
        self.polyphase = polyphase
        self.n_channels = n_channels
        self._cache_key = None
        self._cache = None

    # -- kernel-ready filter tables -----------------------------------------------------------
    def _analysis_taps(self):
        """taps[k][j] for y[k][n] = sum_j taps[k][j] x[16 n + j - pad_l]: PQMF.forward =
        classic_forward = conv(stride M, padding K/2)[..., :-1]."""
        return self.hk, (self.hk.shape[-1] // 2, self.hk.shape[-1] // 2 - 1)

    def _synthesis_weight(self):
        M, K = self.hk.shape
        hki = self.hk.flip(-1).reshape(M, K // M, M).permute(2, 0, 1).contiguous()  # [m, c, t]
        # polyphase_inverse: conv(padding K/M/2 + 1)[..., :-1], then drop 2 * M samples
        return hki, (K // M) // 2 + 1 - 2

    def _tables(self):
        taps, (pl, pr) = self._analysis_taps()
        w, wpad = self._synthesis_weight()
        key = (taps.data_ptr(), taps._version, w.data_ptr(), w._version, str(taps.device))
        if self._cache_key != key:
            self._cache = _build_tables(taps.detach(), pl, pr, w.detach(), wpad)
            self._cache_key = key
        return self._cache

    def forward(self, x):
        if x.ndim == 2:
            return torch.stack([self.forward(x[i]) for i in range(x.shape[0])])
        if self.n_band == 1:
            return x
        _require_16(self.n_band)
        t = self._tables()
        return ops.PqmfAnalysisFn.apply(x, t["taps"], t["taps_bwd"], t["pad_l"], t["pad_r"], t["taps_bwd_pad"])

    def inverse(self, x):
        if x.ndim == 2:
            if self.n_channels == 1:
                return self.inverse(x[0]).unsqueeze(0)
            x = x.split(self.n_channels, -2)
            return torch.stack([self.inverse(x[i]) for i in range(len(x))])
        if self.n_band == 1:
            return x
        _require_16(self.n_band)
        t = self._tables()
        return ops.PqmfSynthesisFn.apply(x, t["w"], t["w_bwd"], t["w_pad"], t["w_bwd_pad"])


import os as _os
USE_FAST = _os.environ.get("RAVE_PQMF_DENSE", "0") != "1"      # factorised kernels when the bank is cosine-modulated (always, for rave/pqmf.py designs)


def _require_16(n_band):
    if n_band != 16:
        raise RaveB200Error(f"only the 16-band PQMF (every shipped config) has a device kernel, got {n_band}")


def _factorise(H, tol=5e-6):
    """H [16 bands][n] (n <= 544): rank-one-per-residue factorisation H[k][32 i + r] = C[k][r] Q[r][i] of a
    cosine-modulated bank (the modulating cosine of rave/pqmf.py:43-52 flips sign every 2M = 32 taps).  Computed in
    float64 on the host from the table itself -- whatever was loaded from a checkpoint is what gets factorised --
    and verified: returns None (-> dense kernels) if the table is not rank one to `tol` (relative Frobenius).
    Returns (C [16][32], Qt [17][32]) as float32 CPU tensors."""
    M, n = H.shape
    if M != 16 or n > 32 * 17:
        return None
    Hp = torch.zeros(16, 32 * 17, dtype=torch.float64)
    Hp[:, :n] = H.detach().to("cpu", torch.float64)
    A = Hp.view(16, 17, 32).permute(2, 0, 1)                    # [r][k][i]
    U, S, Vh = torch.linalg.svd(A, full_matrices=False)
    root = S[:, 0].clamp_min(0).sqrt()
    C = (U[:, :, 0] * root[:, None]).t().contiguous()            # [k][r]
    Q = (Vh[:, 0, :] * root[:, None])                            # [r][i]
    resid = (A - torch.einsum("kr,ri->rki", C, Q)).norm() / A.norm().clamp_min(1e-300)
    if not bool(resid <= tol):
        return None
    return C.float().contiguous(), Q.t().float().contiguous()


def _build_tables(taps, pad_l, pad_r, w, w_pad):
    """Kernel-ready filter tables for analysis / synthesis and their adjoints (see ops.py).

    analysis  : y[k][n]        = s(k,n) sum_j taps[k][j] x[16 n + j - pad_l]
    synthesis : out[16t+15-m]  = 16 sum_c sum_j w[m][c][j] s(c,tau) x[c][tau], tau = t + j - w_pad
    adjoint of analysis  = a synthesis with   w'[m][c][j'] = taps[c][15 - m + D - 16 j'], pad P
    adjoint of synthesis = an analysis with   T'[c][i] = 16 w[15 - i%16][c][K-1 - i//16], pad 16 (K-1-w_pad)
    """
    M, ntaps = taps.shape
    dev = taps.device
    if pad_l > 512 or ntaps > 528:
        raise RaveB200Error("pqmf: filter longer than the kernel supports")
    # adjoint of analysis
    P = (512 - pad_l) // 16
    D = pad_l + 16 * P
    m = torch.arange(16, device=dev).view(16, 1, 1)
    jp = torch.arange(33, device=dev).view(1, 1, 33)
    idx = (15 - m) + D - 16 * jp                                  # [16 m, 1, 33]
    valid = (idx >= 0) & (idx < ntaps)
    idx = idx.clamp(0, ntaps - 1).expand(16, 16, 33)
    tk = taps.view(1, 16, ntaps).expand(16, 16, ntaps)
    taps_bwd = torch.gather(tk, 2, idx) * valid
    # adjoint of synthesis
    K = w.shape[2]
    i = torch.arange(16 * K, device=dev)
    mm = 15 - (i % 16)
    jj = K - 1 - (i // 16)
    w_bwd = 16.0 * w[mm, :, jj].transpose(0, 1).contiguous()       # [c][i]
    out = dict(taps=taps.contiguous(), pad_l=pad_l, pad_r=pad_r, taps_bwd=taps_bwd.contiguous(),
               taps_bwd_pad=P, w=w.contiguous(), w_pad=w_pad, w_bwd=w_bwd,
               w_bwd_pad=16 * (K - 1 - w_pad), dense=dict(taps=taps.contiguous(), taps_bwd=taps_bwd.contiguous(),
                                                          w=w.contiguous(), w_bwd=w_bwd))
    if USE_FAST and K <= 33:
        # factorised tables for the fast kernels (csrc/pqmf.cu): analysis-form tables are [16][n], synthesis-form
        # weights w[m][c][j] are the band filters H[c][16 j + m]
        def syn_as_bank(wt):
            return wt.permute(1, 2, 0).reshape(16, -1)
        fa, fs = _factorise(taps), _factorise(syn_as_bank(w))
        fab, fsb = _factorise(syn_as_bank(taps_bwd)), _factorise(w_bwd)
        if all(f is not None for f in (fa, fs, fab, fsb)):
            out["taps"] = (fa[0].t().contiguous().to(dev), fa[1].to(dev), ntaps)          # Ct [32][16], Qt
            out["w"] = (fs[0].to(dev), fs[1].to(dev))                                        # Cc [16][32], Qt
            out["taps_bwd"] = (fab[0].to(dev), fab[1].to(dev))
            out["w_bwd"] = (fsb[0].t().contiguous().to(dev), fsb[1].to(dev), w_bwd.shape[1])
    return out


class CachedPQMF(PQMF):
    """`pqmf.CachedPQMF` (rave/pqmf.py:245-294): the variant every shipped config uses
    (configs/v1.gin:37-39,96).  Keeps `forward_conv` / `inverse_conv` (and their `weight`
    state_dict entries) as the source of the filter taps."""

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        hkf = make_odd(self.hk).unsqueeze(1)
        M = self.hk.shape[0]
        hki = self.hk.flip(-1)
        hki = hki.reshape(M, hki.shape[-1] // M, M).permute(2, 0, 1)  # "c (t m) -> m c t"
        hki = make_odd(hki)
        self.forward_conv = cc.Conv1d(hkf.shape[1], hkf.shape[0], hkf.shape[2],
                                      padding=cc.get_padding(hkf.shape[-1]), stride=hkf.shape[0],
                                      bias=False)
        self.forward_conv.weight.data.copy_(hkf)
        self.inverse_conv = cc.Conv1d(hki.shape[1], hki.shape[0], hki.shape[-1],
                                      padding=cc.get_padding(hki.shape[-1]), bias=False)
        self.inverse_conv.weight.data.copy_(hki)

    def script_cache(self):
        self.forward_conv.script_cache()
        self.inverse_conv.script_cache()

    def _analysis_taps(self):
        return self.forward_conv.weight[:, 0, :], self.forward_conv._pad

    def _synthesis_weight(self):
        return self.inverse_conv.weight, self.inverse_conv._pad[0]

    # -- streaming (cc.use_cached_conv(True) at construction, SURVEY 8f.4): the two convs carry ring buffers; the bank is
    #    evaluated chunk by chunk through them exactly as rave/pqmf.py:279-294 does (the offline kernels above fuse the
    #    sign flips / x16 / interleave, the streaming path keeps them as separate small passes: chunks are short).
    @property
    def streaming(self) -> bool:
        return bool(getattr(self.forward_conv, "_cached", False))

    def forward(self, x):
        if not self.streaming or self.n_band == 1:
            return super().forward(x)
        return reverse_half(self.forward_conv(x))

    def inverse(self, x):
        if not self.streaming or self.n_band == 1:
            return super().inverse(x)
        m = self.hk.shape[0]
        y = self.inverse_conv(reverse_half(x)) * m                  # [B, m, t]
        y = y.flip(1).permute(0, 2, 1)                              # [B, t, m]
        y = y.reshape(y.shape[0], y.shape[1], -1, m).permute(0, 2, 1, 3)
        return y.reshape(y.shape[0], y.shape[1], -1)


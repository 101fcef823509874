"""TEST INFRASTRUCTURE -- float64 restatement of the exported model's `prior(temp)` (ExportedRAVE.prior,
csrc/prior_sample.cu prior_stream; scripts/export.py TraceModel at a `--streaming` export), built on
oracle/prior_oracle.py's dense forward and tests/prior_sample_ref.py's inverse CDF.  Device-agnostic."""
import math

import torch
import torch.nn.functional as F

from oracle import prior_oracle as P
from tests import prior_sample_ref as S


def temperature(temp_in):
    """temp [B, 1, T] -> the call's row temperatures [B]: softplus(mean) / ln 2."""
    return F.softplus(temp_in.double().mean(-1)[:, 0]) / math.log(2)


class StreamRef:
    """The generation state of B rows: every class frame so far (frame 0 = class R // 2 in every dim) and the diagonal
    cache of the D - 1 newest decoded frames (initially 0.0).  `argmax` replaces the inverse CDF by the first argmax."""

    def __init__(self, sd, cfg, D, B, argmax=False):
        self.sd, self.cfg, self.D, self.R, self.argmax = sd, cfg, D, cfg["resolution"], argmax
        self.cls = torch.full((B, D, 1), self.R // 2, dtype=torch.long)
        self.cache = torch.zeros(B, D - 1, D, dtype=torch.float64)

    def __call__(self, temp_in, uniform, dither):
        """temp_in [B, 1, T], uniform / dither [B, T, D] -> (output [B, D, T] float64, classes [B, T, D])."""
        B, D, R = self.cls.shape[0], self.D, self.R
        temp = temperature(temp_in)
        outs, classes = [], []
        for i in range(temp_in.shape[-1]):
            x = P.stack_one_hot(self.cls, R).double()
            lg = P.forward(x, self.sd, self.cfg, D)[..., -1].reshape(B, D, R) / temp[:, None, None]
            k = lg.argmax(-1) if self.argmax else S.inverse_cdf(lg, uniform[:, i].double())
            self.cls = torch.cat([self.cls, k[:, :, None]], -1)
            y = (k.double() / R + dither[:, i].double() / R)
            y = torch.clamp(torch.erfinv(2 * y - 1) * math.sqrt(2), -4, 4)
            seq = torch.cat([self.cache, y[:, None]], 1)                      # [B, D frames (newest last), D dims]
            outs.append(torch.diagonal(seq, dim1=1, dim2=2))                  # dim d: frame D - 1 - d before the newest
            self.cache = seq[:, 1:]
            classes.append(k)
        return torch.stack(outs, -1), torch.stack(classes, 1)

"""`Resampler`: the export's sample-rate converter (rave/resampler.py), so that a model trained at `model_sr` runs in a
host at `target_sr = ratio * model_sr`.

`to_model_sampling_rate` low-passes every (batch, channel) row with a Kaiser filter (cut-off pi / ratio, 140 dB) and
keeps every ratio-th sample; `from_model_sampling_rate` runs the same filter as a bank of `ratio` phases and interleaves
them.  Both are one launch of csrc/resample.cu.  The taps are the reference's float32 tensors, in `downsample.weight`
[1, 1, K] and `upsample.weight` [ratio, 1, K'], so `state_dict`s match.  The padding follows `cc.get_padding` at
construction: centred, or causal inside `cc.configure(padding_mode="causal")`.

Two quirks of the reference are kept (DESIGN §5.12): the up path's gain is 1 / ratio (the bank is not scaled by
`ratio`, so a down / up round trip divides the signal by `ratio`), and only ratios 2 and 3 can be built: for every ratio
from 4 to 9 the left-padded filter length is not a multiple of the ratio, and the reference fails at construction.  The
next ratios it can build (10, 14, ...) need more taps (185, 259, ...) than the kernel takes, and raise here too.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import cc, ops
from .pqmf import kaiser_filter

MAX_TAPS = 64   # csrc/resample.cu: RS_MAX_K


def resampler_taps(ratio: int):
    """(down [K] float32, up [ratio, K'] float32): the reference's filter and its polyphase bank."""
    filt = torch.from_numpy(kaiser_filter(np.pi / ratio, 140)).float()
    n = len(filt)
    if (n + n % ratio) % ratio:
        raise ValueError(f"resampling ratio {ratio} cannot be built: its {n}-tap filter, left-padded by {n % ratio}, "
                         f"does not split into {ratio} phases, and the reference fails at construction")
    if n > MAX_TAPS:
        raise ValueError(f"resampling ratio {ratio} needs a {n}-tap filter; the resampling kernel takes at most "
                         f"{MAX_TAPS} taps (ratios 2 and 3)")
    bank = F.pad(filt, (n % ratio, 0)).reshape(-1, ratio).t()
    bank = F.pad(bank, ((bank.shape[-1] + 1) % 2, 0))
    return filt, bank.contiguous()


class Resampler(nn.Module):
    """Resampler(target_sr, model_sr): target_sr must be a multiple (2 or 3) of model_sr.  CUDA tensors only."""

    def __init__(self, target_sr: int, model_sr: int):
        super().__init__()
        if target_sr == model_sr:
            raise ValueError("identical source and target rates")
        if target_sr % model_sr or target_sr < model_sr:
            raise ValueError(f"target rate {target_sr} is not a multiple of the model's rate {model_sr}")
        self.model_sr = model_sr
        self.target_sr = target_sr
        self.ratio = ratio = target_sr // model_sr
        down, up = resampler_taps(ratio)
        self.downsample = cc.Conv1d(1, 1, len(down), stride=ratio, padding=cc.get_padding(len(down), ratio),
                                    bias=False)
        self.downsample.weight.data.copy_(down.reshape(1, 1, -1))
        self.upsample = cc.Conv1d(1, ratio, up.shape[-1], stride=1, padding=cc.get_padding(up.shape[-1]), bias=False)
        self.upsample.weight.data.copy_(up.unsqueeze(1))

    def to_model_sampling_rate(self, x):
        """x [B, C, N] at target_sr -> [B, C, ceil(N / ratio)] at model_sr."""
        conv = self.downsample
        return ops.resample(x, conv.weight.detach().reshape(1, -1), self.ratio, conv._pad)

    def from_model_sampling_rate(self, x):
        """x [B, C, T] at model_sr -> [B, C, T ratio] at target_sr."""
        conv = self.upsample
        return ops.resample(x, conv.weight.detach().reshape(self.ratio, -1), 1, conv._pad)

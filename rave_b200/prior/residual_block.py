"""rave/prior/residual_block.py: dilated causal conv -> gated unit -> residual (rconv) and skip (sconv) 1x1 convs.
All three convs carry biases (scripts/train_prior.py:90 clears the RAVE's gin bindings, so `cc.Conv1d.bias = False`
does not reach the prior).  rconv / sconv are `nn.Conv1d` in the reference; here they are the library's `cc.Conv1d`
with the same parameters and `state_dict` keys, so that the residual / skip sums fuse into the conv."""
import torch.nn as nn

from .. import cc, ops


class ResidualBlock(nn.Module):

    def __init__(self, res_size, skp_size, kernel_size, dilation):
        super().__init__()
        fks = (kernel_size - 1) * dilation + 1
        self.dconv = cc.Conv1d(res_size, 2 * res_size, kernel_size, padding=(fks - 1, 0), dilation=dilation, bias=True)
        self.rconv = cc.Conv1d(res_size, res_size, 1, bias=True)
        self.sconv = cc.Conv1d(res_size, skp_size, 1, bias=True)

    def forward(self, x, skp):
        g = ops.gate(self.dconv(x))
        res = self.rconv(g, res=x)
        skp = self.sconv(g, res=skp) if skp.dim() == 3 else self.sconv(g) + skp
        return res, skp

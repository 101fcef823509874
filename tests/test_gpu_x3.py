"""GPU: the split-operand ("bf16x3") mode of the wgmma conv engine -- the accurate fast mode.  Operands are carried
as x = hi + lo (two bf16 halves, 16-bit significand) and every product is hi*hi + lo*hi + hi*lo accumulated in fp32 on
the tensor cores.  Stated tolerance: 2e-5 rel-L2 per conv against the fp32 CPU oracle on UN-rounded operands, 1e-4
rel-L2 end to end for PQMF + encoder + generator (the north-star tolerance; single-pass bf16 sits at ~1e-2)."""
import pytest
import torch
import torch.nn as nn

from oracle import rave_oracle as O
from tests.conftest import rel_l2

pytestmark = pytest.mark.gpu

X3_CASES = [
    # B, Cin, Cout, L, K, stride, dil, pad, bias, res
    (2, 64, 64, 256, 3, 1, 1, (1, 1), False, False),
    (2, 96, 96, 512, 3, 1, 3, (3, 3), False, True),
    (3, 96, 96, 384, 1, 1, 1, (0, 0), False, True),
    (2, 16, 96, 512, 7, 1, 1, (3, 3), False, False),        # stem: 16-channel K blocks
    (2, 96, 192, 512, 8, 4, 1, (3, 4), False, False),       # strided down conv
    (4, 768, 1536, 64, 4, 2, 1, (1, 2), False, False),
    (5, 1536, 256, 32, 3, 1, 1, (1, 1), True, False),
    (2, 192, 192, 1000, 3, 1, 9, (9, 9), True, True),       # ragged length
    (2, 96, 32, 300, 7, 1, 1, (6, 0), True, False),          # small N: single-CTA kernel, causal padding
    (2, 384, 384, 256, 3, 1, 1, (1, 1), False, False),
]


def split(t):
    hi = t.bfloat16()
    return hi, (t - hi.float()).bfloat16()


@pytest.mark.parametrize("case", X3_CASES)
def test_conv1d_tc_x3_vs_fp32_oracle(case):
    from rave_b200 import ops
    B, Cin, Cout, L, K, stride, dil, pad, use_bias, use_res = case
    g = torch.Generator().manual_seed(hash(case) % (2 ** 31))
    x = torch.randn(B, Cin, L, generator=g)
    w = torch.randn(Cout, Cin, K, generator=g) / (Cin * K) ** 0.5
    bias = torch.randn(Cout, generator=g) if use_bias else None
    y_ref = O.conv1d(x, w, bias, stride, dil, pad)
    res = torch.randn(y_ref.shape, generator=g) if use_res else None
    if use_res:
        y_ref = y_ref + res
    xa = ops.ncl_to_cl_x3(x.cuda())
    hi, lo = split(x.permute(0, 2, 1))
    assert torch.equal(xa.cpu(), torch.cat([hi, lo], -1))
    (norm, wt, _), = ops.weight_prep_tc_multi([(w.cuda(), None, list(range(K)), [], Cout, Cin)], x3=True)
    whi, wlo = split(w.permute(2, 0, 1))
    assert torch.equal(wt.cpu(), torch.cat([whi, wlo], 0))
    res_cl = res.permute(0, 2, 1).contiguous().cuda() if use_res else None
    out_f32, out_act = ops.conv1d_tc(xa, wt, bias.cuda() if use_bias else None, res_cl, stride, dil, pad, ops.ACT_LEAKY,
                                     0.2, want_f32=True, want_act=True, x3=True)
    torch.cuda.synchronize()
    y = ops.cl_to_ncl(out_f32)
    assert y.shape == y_ref.shape
    r = rel_l2(y, y_ref)
    assert r < 2e-5, r
    a = out_act[..., :Cout].float() + out_act[..., Cout:].float()
    assert rel_l2(a, O.leaky_relu(y_ref, 0.2).permute(0, 2, 1)) < 2e-5
    # the recovered-residual epilogue: + inverse LeakyReLU of another split operand
    if Cout == Cin and stride == 1:
        o2, _ = ops.conv1d_tc(xa, wt, None, None, stride, dil, pad, ops.ACT_NONE, 0.2, want_f32=True, want_act=False,
                              x3=True, res_act=ops.ncl_to_cl_x3(O.leaky_relu(x, 0.2).cuda()), res_slope=0.2)
        y2 = O.conv1d(x, w, None, stride, dil, pad) + x
        assert rel_l2(ops.cl_to_ncl(o2), y2) < 2e-5


@pytest.mark.parametrize("name,B,T", [("v2_small", 2, 65536), ("v2", 1, 65536)])
def test_forward_x3_within_north_star_tolerance(name, B, T):
    """BASELINE config 2 (v2_small; and v2 at full capacity): PQMF + encoder + generator forward in the accurate fast
    mode against the fp32 CPU oracle: z and y within 1e-4 rel-L2 (SURVEY 8d)."""
    import rave_b200
    from rave_b200 import configs
    from rave_b200.model import _pqmf_decode, _pqmf_encode
    torch.manual_seed(0)
    pq, enc, dec = configs.make_autoencoder(name)
    holder = nn.Module()
    holder.pqmf, holder.encoder, holder.decoder = pq, enc, dec
    sd = {k: v.detach().clone() for k, v in holder.state_dict().items()}
    gen = torch.Generator().manual_seed(1234)
    x = (0.5 * torch.randn(B, 1, T, generator=gen)).clamp(-1, 1)
    cfg = O.v2_small_config() if name == "v2_small" else O.ArchConfig()
    import numpy as np
    eps = torch.randn(B, 128, T // (16 * int(np.prod(cfg.ratios))), generator=torch.Generator().manual_seed(4321))
    taps = {}
    y_o = O.rave_forward(x, sd, cfg, eps, taps)
    holder.cuda().eval()
    holder.train()            # training-mode modules (AdaIN identity etc.), no autograd
    rave_b200.set_precision("bf16x3")
    try:
        with torch.no_grad():
            from rave_b200 import _lib
            n0 = _lib.launch_count()
            z = enc(_pqmf_encode(pq, x.cuda()))
            zs, _ = enc.reparametrize(z, eps.cuda())
            y = _pqmf_decode(pq, dec(zs), batch_size=x.shape[:-2], n_channels=1)
            torch.cuda.synchronize()
            assert _lib.launch_count() > n0
    finally:
        rave_b200.set_precision("fp32")
    rz, ry = rel_l2(z, taps["z"]), rel_l2(y, y_o)
    print(f"bf16x3 {name}: z rel-L2 {rz:.3e}, y rel-L2 {ry:.3e}")
    assert rz < 1e-4 and ry < 1e-4

"""GPU: the pipelining of the wgmma conv / weight-gradient main loops and the conv epilogue across the shapes they have to
handle: one k-block per tile, fewer k-blocks than pipeline stages, k-block counts that are not a multiple of the stages,
several tiles per persistent CTA, ragged last tiles, every BLOCK_N / BLOCK_K instance, every epilogue operand and the
split-operand (x3) mode.  Each launch is compared against the emulator (tests/tc_emulator.py) on the same bf16 operands
(fp32 accumulation order is the only difference: 2e-5 rel-L2) and run twice to check that it is bitwise repeatable."""
import pytest
import torch

from tests import tc_emulator as E
from tests.conftest import rel_l2

pytestmark = pytest.mark.gpu


def _plan(B, Cin, Cout, Lout, K):
    from rave_b200 import _lib
    v = _lib.load().rave_conv1d_tc_plan(B, Cin, Cout, Lout, K)
    return v & 0xFFF, (v >> 12) & 0xFFF


def _run_conv(B, Cin, Cout, L, K, stride=1, dil=1, pad=(0, 0), *, bias=False, res=False, res_bf16=False, dact=False,
              res_act=False, fm=0, want_f32=True, want_act=True, act=1, phases=None, seed=0):
    """fm: 0 = no feature-matching term, 1 = [real; fake] batch (fm_bh > 0), -1 = fake half with partner rows before it.
    phases: (out_row_stride, out_row_offset) of a transposed-conv phase (rows of the other phases stay zero)."""
    from rave_b200 import ops
    g = torch.Generator().manual_seed(seed)
    Lout = (L + pad[0] + pad[1] - dil * (K - 1) - 1) // stride + 1
    ors, oro = phases if phases else (0, 0)
    rows = Lout * ors + 3 if phases else Lout
    x = torch.randn(B, L, Cin, generator=g).bfloat16()
    wt = (torch.randn(K, Cout, Cin, generator=g) / (Cin * K) ** 0.5).bfloat16()
    t = dict(bias=torch.randn(Cout, generator=g) if bias else None,
             res=torch.randn(B, rows, Cout, generator=g) if res else None,
             res_bf16=torch.randn(B, rows, Cout, generator=g).bfloat16() if res_bf16 else None,
             res_act=torch.nn.functional.leaky_relu(torch.randn(B, rows, Cout, generator=g), 0.2).bfloat16()
             if res_act else None)
    full = None
    if dact or fm:
        full = torch.nn.functional.leaky_relu(torch.randn(2 * B if fm < 0 else B, rows, Cout, generator=g), 0.2).bfloat16()
    fm_d = torch.tensor([0.37, -0.21]) if fm else None
    kw = dict(stride=stride, dil=dil, pad=pad, act=act, slope=0.2, want_f32=False, want_act=False, Lout=Lout, Lin=L,
              out_rows=rows if phases else 0, out_row_stride=ors, out_row_offset=oro)

    def outs(dev):
        o32 = torch.zeros(B, rows, Cout, device=dev) if want_f32 else None
        oa = torch.zeros(B, rows, Cout, dtype=torch.bfloat16, device=dev) if want_act else None
        return o32, oa

    def args(dev):
        mv = lambda v: v.to(dev) if v is not None else None
        f = mv(full)
        return dict(bias=mv(t["bias"]), res_cl=mv(t["res"]), res_bf16=mv(t["res_bf16"]), res_act=mv(t["res_act"]),
                    dact_src=(f[B:] if fm < 0 else f) if f is not None else None,
                    fm_partner=f[:B] if fm < 0 else None, fm_d=mv(fm_d))

    r32, ra = outs("cpu")
    E.conv1d_tc(x, wt, out_f32=r32, out_act=ra, **args("cpu"), **kw)
    got = []
    for _ in range(2):
        o32, oa = outs("cuda")
        ops.conv1d_tc(x.cuda(), wt.cuda(), out_f32=o32, out_act=oa, **args("cuda"), **kw)
        got.append((o32, oa))
    torch.cuda.synchronize()
    for a, b in zip(got[0], got[1]):
        if a is not None:
            assert torch.equal(a, b), "run-to-run difference"
    o32, oa = got[0]
    if want_f32:
        assert rel_l2(o32, r32) < 2e-5
    if want_act:
        assert rel_l2(oa.float(), ra.float()) < 5e-3          # bf16 rounding of the stored operand
    if phases:
        idx = torch.arange(Lout) * ors + oro
        mask = torch.ones(rows, dtype=torch.bool)
        mask[idx] = False
        for o in (o32, oa):
            if o is not None:
                assert float(o[:, mask].float().abs().max()) == 0.0   # rows of other phases untouched


BK_CIN = {16: 48, 32: 96, 64: 192}        # Cin = 3 k-blocks per tap of each BLOCK_K
BN_SHAPE = {16: (16, 3, 1000), 32: (32, 3, 1000), 48: (48, 3, 1000),       # Cout, B, L
            64: (64, 3, 6000), 96: (96, 3, 6000), 128: (128, 3, 6000)}   # >= 132 M tiles: the widest N is taken


@pytest.mark.parametrize("bk", [16, 32, 64])
@pytest.mark.parametrize("bn", [16, 32, 48, 64, 96, 128])
def test_every_instance(bn, bk):
    """3 taps x 3 k-blocks = 9 k-blocks per tile (not a multiple of the stages); L = 1000 / 6000 leave a ragged last
    tile; the 6000-row shapes have 141 M tiles, more than the SMs, so CTAs run several tiles."""
    Cout, B, L = BN_SHAPE[bn]
    Cin = BK_CIN[bk]
    assert _plan(B, Cin, Cout, L, 3) == (bn, bk)
    _run_conv(B, Cin, Cout, L, 3, pad=(1, 1), bias=True, res=True, seed=bn * 100 + bk)


@pytest.mark.parametrize("many", [False, True])
@pytest.mark.parametrize("cin", [16, 32, 64])
def test_single_kblock_per_tile(cin, many):
    """K = 1, Cin <= BLOCK_K: every tile is one k-block, so each tile both starts and ends the in-flight group.  With
    many=True there are 256 M tiles (two per CTA), which carries the stage / phase bookkeeping across tiles."""
    B, L = (4, 8192) if many else (2, 300)
    _run_conv(B, cin, 64, L, 1, bias=True, res=True, seed=cin + many)


@pytest.mark.parametrize("case", [
    (1, 128, 2, 6000),      # 2 k-blocks: fewer than the stages
    (5, 64, 5, 6000),       # 5 k-blocks
    (3, 96, 9, 700),        # 9 k-blocks of BLOCK_K = 32, few tiles
    (15, 32, 15, 2048),     # 15 k-blocks
])
def test_kblock_counts(case):
    K, Cin, _kblocks, L = case
    _run_conv(3, Cin, 96, L, K, stride=1, pad=(K // 2, K // 2), bias=True, seed=K * 1000 + Cin)


EPI_CASES = {
    "f32_only": dict(want_act=False),
    "act_only": dict(want_f32=False),
    "f32_act_bias": dict(bias=True),
    "res": dict(res=True, act=0),
    "res_bf16": dict(res_bf16=True, want_f32=False, act=0),
    "dact": dict(dact=True, want_f32=False, act=0),
    "res_act": dict(res_act=True, bias=True),
    "fm_pos": dict(fm=1, want_f32=False, act=0),
    "fm_neg": dict(fm=-1, want_f32=False, act=0),
    "phases": dict(bias=True, phases=(4, 3)),
    "phases_fm": dict(fm=1, want_f32=False, act=0, phases=(2, 1)),
}


@pytest.mark.parametrize("cout", [48, 96, 128])
@pytest.mark.parametrize("name", list(EPI_CASES))
def test_epilogue_operands(name, cout):
    """Each epilogue operand alone at the conv level; Cout = 48 is a 32 + 16 column tile, 128 the widest."""
    kw = EPI_CASES[name]
    _run_conv(4, 64, cout, 515, 3, pad=(2, 0), seed=list(EPI_CASES).index(name) * 1000 + cout, **kw)


@pytest.mark.parametrize("case", [
    # B, Cin, Cout, L, act_cs, res_act
    (3, 64, 128, 6000, 0, True),     # <128, 64> x3: two pipeline stages, several tiles per CTA
    (2, 32, 96, 1000, 48, False),    # 48 channels per position: [hi | lo] rows in 16-column chunks
    (2, 64, 48, 777, 0, True),
])
def test_x3(case):
    from rave_b200 import ops
    B, Cin, Cout, L, act_cs, use_ra = case
    g = torch.Generator().manual_seed(B * Cin + Cout)
    K = 3
    x = torch.randn(B, L, Cin, generator=g)
    hi = x.bfloat16()
    xa = torch.cat([hi, (x - hi.float()).bfloat16()], -1)
    w = torch.randn(K, Cout, Cin, generator=g) / (Cin * K) ** 0.5
    wh = w.bfloat16()
    wt = torch.cat([wh, (w - wh.float()).bfloat16()], 0)
    bias = torch.randn(Cout, generator=g)
    ra = None
    if use_ra:
        r = torch.nn.functional.leaky_relu(torch.randn(B, L, Cout, generator=g), 0.2)
        rh = r.bfloat16()
        ra = torch.cat([rh, (r - rh.float()).bfloat16()], -1)
    kw = dict(stride=1, dil=1, pad=(1, 1), act=1, slope=0.2, want_f32=False, want_act=False, x3=True, act_cs=act_cs,
              res_slope=0.2)
    r32 = torch.zeros(B, L, Cout)
    r_a = torch.zeros(B, L, 2 * Cout, dtype=torch.bfloat16)
    E.conv1d_tc(xa, wt, bias, None, out_f32=r32, out_act=r_a, res_act=ra, **kw)
    got = []
    for _ in range(2):
        o32 = torch.zeros(B, L, Cout, device="cuda")
        oa = torch.zeros(B, L, 2 * Cout, dtype=torch.bfloat16, device="cuda")
        ops.conv1d_tc(xa.cuda(), wt.cuda(), bias.cuda(), None, out_f32=o32, out_act=oa,
                      res_act=ra.cuda() if ra is not None else None, **kw)
        got.append((o32, oa))
    torch.cuda.synchronize()
    assert torch.equal(got[0][0], got[1][0]) and torch.equal(got[0][1], got[1][1])
    o32, oa = got[0]
    assert rel_l2(o32, r32) < 2e-5
    cs = act_cs or Cout

    def value(a):       # hi + lo of every position
        a = a.float().cpu().reshape(B, L, Cout // cs, 2, cs)
        return (a[:, :, :, 0] + a[:, :, :, 1]).reshape(B, L, Cout)
    assert rel_l2(value(oa), value(r_a)) < 2e-5


@pytest.mark.parametrize("case", [
    # B, Cm, Cn, L, K: 64-row chunks per split
    (1, 96, 64, 40, 3),       # 2 chunks of 32 rows: fewer than the stages
    (1, 192, 192, 200, 3),    # 4 chunks, two N tiles
    (2, 96, 64, 1000, 5),     # 32 chunks split into slices of 8
    (3, 128, 128, 700, 7),    # 33 chunks: slices not a multiple of the stages
])
def test_wgrad_chunk_counts(case):
    from rave_b200 import _lib, ops
    B, Cm, Cn, L, K = case
    g = torch.Generator().manual_seed(L + K)
    pad_l = K // 2
    x = torch.randn(B, Cn, L, generator=g).bfloat16().float()
    Lout = L + 2 * pad_l - K + 1
    dy = torch.randn(B, Cm, Lout, generator=g).bfloat16().float()
    w = torch.zeros(Cm, Cn, K, requires_grad=True)
    y = torch.nn.functional.conv1d(torch.nn.functional.pad(x, (pad_l, pad_l)), w)
    (dw_ref,) = torch.autograd.grad(y, w, dy)
    P = dy.permute(0, 2, 1).contiguous().bfloat16().cuda()
    Q = x.permute(0, 2, 1).contiguous().bfloat16().cuda()
    assert _lib.load().rave_conv1d_tc_wgrad_splits(B, Cm, Lout, Cn, K) >= 1
    outs = []
    for _ in range(2):
        db = torch.zeros(Cm, device="cuda")
        dw = ops.tapmajor_to_weight(ops.conv1d_tc_wgrad(P, Q, K, 1, 1, pad_l, dbias=db))
        outs.append((dw, db))
    torch.cuda.synchronize()
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert rel_l2(outs[0][0], dw_ref) < 2e-5
    assert rel_l2(outs[0][1], dy.sum((0, 2))) < 1e-5

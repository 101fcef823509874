"""GPU: forward launches on the ping-pong kernel (conv_tc_pp_fwd_kernel: two MMA warpgroups on alternate tiles, bias
and LeakyReLU applied straight from the accumulator registers, the bf16 tile stored by TMA from a shared-memory slot).

It runs the conv launches whose only output is bf16 and whose epilogue is bias and / or LeakyReLU (no residual, no
mask).  Each launch is checked on the same bf16 operands: its fp32 stream (the same launch with out_f32 also requested,
which runs conv_tc_kernel) against the emulator (tests/tc_emulator.py) at 2e-5; its bf16 output bit for bit against
that launch's, against a second launch of itself, and against the fp32 stream rounded on the host.  Output rows the
launch does not own -- other phases, the pitch slack past Lout -- must keep the value they were pre-filled with.
Every case asserts the BLOCK_N / BLOCK_K instance it runs (rave_conv1d_tc_plan) and whether the ping-pong kernel takes it
(rave_conv1d_tc_pp_fwd_stages); one test reads the kernel names off the profiler.  BLOCK_N 16 ... 128, BLOCK_K 16 / 32
/ 64, tiles of one k-block, K = 5 and 15 at stride 4, bias or none, LeakyReLU or none, a ragged last time tile, short
rows with several batches per tile and a part-empty last batch group, and the phase rows of a transposed conv."""
import json
import os
import subprocess
import sys

import pytest
import torch

from tests import tc_emulator as E
from tests.conftest import rel_l2

pytestmark = pytest.mark.gpu

FILL = 7.0
SLOPE = 0.2


def _instance(B, Cin, Cout, Lout, K):
    """(BLOCK_N, BLOCK_K, ping-pong ring stages; 0 = the launch runs conv_tc_kernel)"""
    from rave_b200 import _lib
    lib = _lib.load()
    plan = lib.rave_conv1d_tc_plan(B, Cin, Cout, Lout, K)
    return plan & 0xFFF, (plan >> 12) & 0xFFF, lib.rave_conv1d_tc_pp_fwd_stages(B, Cin, Cout, Lout, K)


def _run(B, Cin, Cout, L, K=1, stride=1, pad=(0, 0), *, bias=True, leaky=True, phases=None, slack=0, seed=0,
         bn=None, bk=None, pp=True):
    from rave_b200 import ops
    g = torch.Generator().manual_seed(seed)
    Lout = (L + pad[0] + pad[1] - (K - 1) - 1) // stride + 1
    BN, BK, stages = _instance(B, Cin, Cout, Lout, K)
    assert (bn is None or BN == bn) and (bk is None or BK == bk), (BN, BK)
    assert (stages >= 2) if pp else (stages == 0), (BN, BK, stages)
    ors, oro = phases if phases else (1, 0)
    rows = Lout * ors + slack
    x = torch.randn(B, L, Cin, generator=g).bfloat16()
    wt = (torch.randn(K, Cout, Cin, generator=g) / (Cin * K) ** 0.5).bfloat16()
    b = torch.randn(Cout, generator=g) if bias else None
    kw = dict(stride=stride, dil=1, pad=pad, act=1 if leaky else 0, slope=SLOPE, want_f32=False, want_act=False,
              Lout=Lout, Lin=L, out_rows=rows, out_row_stride=ors, out_row_offset=oro)

    ref32 = torch.full((B, rows, Cout), FILL)
    ref = torch.full((B, rows, Cout), FILL, dtype=torch.bfloat16)
    E.conv1d_tc(x, wt, b, out_f32=ref32, out_act=ref, **kw)

    xc, wc, bc = x.cuda(), wt.cuda(), b.cuda() if bias else None

    def launch(with_f32=False):
        oa = torch.full((B, rows, Cout), FILL, dtype=torch.bfloat16, device="cuda")
        o32 = torch.full((B, rows, Cout), FILL, device="cuda") if with_f32 else None
        ops.conv1d_tc(xc, wc, bc, out_f32=o32, out_act=oa, **kw)
        return oa, o32

    (out, _), (again, _), (single, single32) = launch(), launch(), launch(with_f32=True)
    torch.cuda.synchronize()
    out, again, single, single32 = out.cpu(), again.cpu(), single.cpu(), single32.cpu()
    idx = torch.arange(Lout) * ors + oro
    other = torch.ones(rows, dtype=torch.bool)
    other[idx] = False
    assert rel_l2(single32[:, idx], ref32[:, idx]) < 2e-5
    assert rel_l2(out[:, idx].float(), ref[:, idx].float()) < 5e-3
    assert bool((out[:, other].float() == FILL).all()), "rows outside the launch's output rows were written"
    assert torch.equal(out.view(torch.int16), again.view(torch.int16)), "two launches of the same inputs differ"
    assert torch.equal(out[:, idx].view(torch.int16), single[:, idx].view(torch.int16)), \
        "differs from the single-warpgroup kernel"
    v = single32[:, idx]
    host = (torch.maximum(v, v * SLOPE) if leaky else v).bfloat16()
    assert torch.equal(out[:, idx].view(torch.int16), host.view(torch.int16)), "differs from the rounded fp32 stream"


EPI = {
    "bias_leaky": dict(bias=True, leaky=True),
    "bias": dict(bias=True, leaky=False),
    "leaky": dict(bias=False, leaky=True),
    "plain": dict(bias=False, leaky=False),
}


@pytest.mark.parametrize("cin", [16, 32, 64, 96, 192])
@pytest.mark.parametrize("epi", list(EPI))
@pytest.mark.parametrize("cout", [16, 32, 48, 64, 96, 128, 384])
def test_ragged_time_tile(cout, epi, cin):
    """Lout = 4500 is not a multiple of BL = 128 (4 x 36 = 144 M tiles), and the pitch has slack rows past Lout.  K = 1:
    16 / 32 / 64 input channels are one k-block of BLOCK_K 16 / 32 / 64, 96 and 192 three of BLOCK_K 32 / 64; every
    output width up to 128 is its own BLOCK_N."""
    _run(4, cin, cout, 4500, slack=5, seed=cout + cin, bn=min(cout, 128), bk={96: 32, 192: 64}.get(cin, cin), **EPI[epi])


@pytest.mark.parametrize("epi", list(EPI))
@pytest.mark.parametrize("cin,cout,K", [(96, 192, 5), (96, 192, 15), (192, 384, 15), (384, 768, 5)])
def test_strided_long_k(cin, cout, K, epi):
    """The discriminators' strided convs: K = 5 / 15 at stride 4 (15 to 45 k-blocks per tile), BLOCK_N 96 and 128.
    The ping-pong kernel takes every one but the 45 k-blocks per tile at BLOCK_N = 96, which stays on conv_tc_kernel."""
    _run(16, cin, cout, 4400, K=K, stride=4, pad=(K // 2, K // 2), seed=cin + K, bn=96 if cout == 192 else 128,
         pp=not (cout == 192 and K == 15), **EPI[epi])


@pytest.mark.parametrize("epi", list(EPI))
@pytest.mark.parametrize("cout", [96, 384])
def test_short_rows_ragged_batch(cout, epi):
    """L = 20 -> BL = 32, four batches per tile; B = 530 leaves the last of 133 batch groups half empty."""
    _run(530, 64, cout, 21, K=2, seed=cout + 1, bn=96 if cout == 96 else 128, **EPI[epi])


@pytest.mark.parametrize("oro", [1, 3])
@pytest.mark.parametrize("epi", ["bias_leaky", "plain"])
@pytest.mark.parametrize("cout", [192, 384])
def test_phase_rows(cout, epi, oro):
    """Phase oro of a stride-4 transposed conv: output row = l * 4 + oro; the other phases keep their contents."""
    _run(24, 96, cout, 300, K=3, pad=(1, 1), phases=(4, oro), slack=2, seed=cout + oro, **EPI[epi])


def test_many_tiles_per_cta():
    """The first-layer shape (64 im2col channels -> 384, K = 1): 1536 tiles of 128 x 128 over at most 132 CTAs, so the
    ring, the output slots and the ordering barriers go through several phases."""
    _run(16, 64, 384, 4096, seed=11, bn=128, bk=64)


# Run in a fresh process: later in a long test process that has already opened a profiler window (the input-gradient
# test does), torch.profiler came back without the library's kernels.
_PROFILE_CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import torch
from torch.profiler import ProfilerActivity, profile
from rave_b200 import ops

def launch(f32):
    B, Cin, Cout, L = 4, 64, 384, 4500
    x = torch.randn(B, L, Cin, device="cuda").bfloat16()
    wt = torch.randn(1, Cout, Cin, device="cuda").bfloat16()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ops.conv1d_tc(x, wt, torch.randn(Cout, device="cuda"), act=1, slope=0.2, want_f32=False, want_act=True,
                      Lout=L, out_f32=torch.empty(B, L, Cout, device="cuda") if f32 else None)
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "conv_tc" in e.name]

print(json.dumps([launch(False), launch(True)]))
"""


def test_kernel_names():
    """The profiler sees conv_tc_pp_fwd_kernel run the forward launch, and conv_tc_kernel run the same launch with the
    fp32 stream requested."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", _PROFILE_CHILD, root], cwd=root, capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    pp, single = json.loads(out.stdout.strip().splitlines()[-1])
    assert any("conv_tc_pp_fwd_kernel<128, 64, true, true>" in n for n in pp) and \
        not any("conv_tc_kernel" in n for n in pp), pp
    assert any("conv_tc_kernel<128, 64" in n for n in single) and not any("pp_" in n for n in single), single

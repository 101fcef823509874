"""GPU: forward launches on the wide kernel (conv_tc_wide_kernel: 128 x 192 tiles, two MMA warpgroups on the rows 0-63
and 64-127 of every tile, bias and LeakyReLU applied from the accumulator registers, the bf16 tile stored by TMA).

The shapes are the v2 discriminator's long-k forward convs at the training step's [real; fake] batch: the MSD layers
2-4 (K = 15, stride 4) at the three scales and the MPD layers 2-4 (K = 5, stride 4) at the five periods, whose Lout
leaves ragged last time tiles.  Each case asserts that the launch runs the wide kernel (rave_conv1d_tc_wide_stages > 0)
and that its bf16 output equals, byte for byte, the output of the same launch with the fp32 stream also requested,
which runs conv_tc_kernel on 96- or 128-column tiles.  Rows the launch does not own (other phases, pitch slack past
Lout) must keep the value they were pre-filled with.  Also: the four epilogue operand sets, a batch group past B, the
phase rows of a transposed conv, and a profiler check of the kernel name."""
import json
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

FILL = 7.0
SLOPE = 0.2


def _lout(L, K, stride, pad):
    return (L + 2 * pad - K) // stride + 1


def _run(B, Cin, Cout, L, K, stride=4, *, bias=True, leaky=True, phases=None, slack=0, seed=0):
    from rave_b200 import _lib, ops
    pad = K // 2
    Lout = _lout(L, K, stride, pad)
    stages = _lib.load().rave_conv1d_tc_wide_stages(B, Cin, Cout, Lout, K)
    assert stages == (4 if Cin % 64 == 0 else 8), stages
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.zeros(B, -(-L // stride) * stride, Cin, device="cuda", dtype=torch.bfloat16)   # pitch: whole strides
    x[:, :L] = torch.randn(B, L, Cin, device="cuda", generator=g).bfloat16()
    wt = (torch.randn(K, Cout, Cin, device="cuda", generator=g) / (Cin * K) ** 0.5).bfloat16()
    b = torch.randn(Cout, device="cuda", generator=g) if bias else None
    ors, oro = phases if phases else (1, 0)
    rows = Lout * ors + slack
    kw = dict(stride=stride, dil=1, pad=(pad, pad), act=1 if leaky else 0, slope=SLOPE, want_f32=False,
              want_act=False, Lout=Lout, Lin=L, out_rows=rows, out_row_stride=ors, out_row_offset=oro)

    def launch(with_f32):
        oa = torch.full((B, rows, Cout), FILL, dtype=torch.bfloat16, device="cuda")
        o32 = torch.full((B, rows, Cout), FILL, device="cuda") if with_f32 else None
        ops.conv1d_tc(x, wt, b, out_f32=o32, out_act=oa, **kw)
        return oa

    wide, single = launch(False), launch(True)
    torch.cuda.synchronize()
    idx = torch.arange(Lout, device="cuda") * ors + oro
    other = torch.ones(rows, dtype=torch.bool, device="cuda")
    other[idx] = False
    assert bool((wide[:, other].float() == FILL).all()), "rows outside the launch's output rows were written"
    assert bool(torch.isfinite(wide[:, idx].float()).all())
    assert torch.equal(wide.view(torch.int16), single.view(torch.int16)), "differs from conv_tc_kernel"


# (B, Cin, Cout, Lin, K) of the v2 step's discriminator forward launches ([real; fake] batch of 2 x 32)
MSD = [(64, 96, 192, 16384 >> s, 15) for s in range(3)] + \
      [(64, 192, 384, 4096 >> s, 15) for s in range(3)] + \
      [(64, 384, 768, 1024 >> s, 15) for s in range(3)]
MPD_L2_LIN = {2: 2048, 3: 1366, 5: 820, 7: 586, 11: 373}
MPD = []
for _p, _l in MPD_L2_LIN.items():
    _l3 = _lout(_l, 5, 4, 2)
    MPD += [(64 * _p, 96, 192, _l, 5), (64 * _p, 192, 384, _l3, 5), (64 * _p, 384, 768, _lout(_l3, 5, 4, 2), 5)]


@pytest.mark.parametrize("shape", MSD + MPD, ids=[f"B{s[0]}-{s[1]}to{s[2]}-L{s[3]}-K{s[4]}" for s in MSD + MPD])
def test_v2_discriminator_shapes(shape):
    B, Cin, Cout, L, K = shape
    _run(B, Cin, Cout, L, K, slack=3, seed=sum(shape))


EPI = {
    "bias": dict(bias=True, leaky=False),
    "leaky": dict(bias=False, leaky=True),
    "plain": dict(bias=False, leaky=False),
}


@pytest.mark.parametrize("epi", list(EPI))
@pytest.mark.parametrize("cin,cout,K", [(96, 192, 15), (192, 384, 5), (384, 768, 15)])
def test_epilogue_operand_sets(cin, cout, K, epi):
    _run(16, cin, cout, 1500, K, slack=2, seed=cin + K, **EPI[epi])


def test_ragged_batch_group():
    """Lout = 21 -> BL = 32, four batches per tile; B = 530 leaves the last batch group half empty."""
    _run(530, 192, 384, 84, 15, seed=5)


@pytest.mark.parametrize("oro", [1, 3])
def test_phase_rows(oro):
    """Phase oro of a stride-4 transposed conv: output row = l * 4 + oro; the other phases keep their contents."""
    _run(8, 192, 768, 900, 15, stride=1, phases=(4, oro), slack=2, seed=oro)


# a fresh process, as in test_gpu_conv_pingpong_fwd.py: a long test process that already opened a profiler window
# may get a trace without the library's kernels
_PROFILE_CHILD = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import torch
from torch.profiler import ProfilerActivity, profile
from rave_b200 import ops

B, Cin, Cout, L, K = 16, 192, 384, 4096, 15
x = torch.randn(B, L, Cin, device="cuda").bfloat16()
wt = torch.randn(K, Cout, Cin, device="cuda").bfloat16()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    ops.conv1d_tc(x, wt, torch.randn(Cout, device="cuda"), stride=4, pad=(7, 7), act=1, slope=0.2, want_f32=False,
                  want_act=True)
    torch.cuda.synchronize()
print(json.dumps([e.name for e in prof.events() if "conv_tc" in e.name]))
"""


def test_kernel_name():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", _PROFILE_CHILD, root], cwd=root, capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    names = json.loads(out.stdout.strip().splitlines()[-1])
    assert any("conv_tc_wide_kernel<64, true, true>" in n for n in names), names
    assert not any("conv_tc_kernel" in n or "pp_fwd" in n for n in names), names

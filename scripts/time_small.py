"""Graph-timed small kernels of the v2 step at BASELINE config 3 sizes (B = 64 rows of 65536 samples = [real; fake]):
im2col_c1 of the MSD / MPD first layers, gather_c1, the multi-tensor weight-norm backward of an MSD net."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch
from rave_b200 import ops
from _timing import graph_time_us

torch.manual_seed(0)
dev = "cuda"
Bs, T = 64, 65536
src = [torch.randn(Bs, T, device=dev) for _ in range(3)]
for name, K, stride, pad, period, pool in [("msd0", 15, 4, 7, 1, 1), ("msd2", 15, 4, 7, 1, 4), ("mpd2", 5, 4, 2, 2, 1),
                                           ("mpd11", 5, 4, 2, 11, 1), ("dmpd7", 5, 3, 2, 7, 1)]:
    Lin = (T + period - 1) // period if period > 1 else T // pool
    Lout = (Lin + 2 * pad - K) // stride + 1
    pitch = (Lout + 3) // 4 * 4
    us = graph_time_us(lambda i: ops.im2col_c1(src[i % 3], Lin, Lout, pitch, K, stride, pad, period, pool), n=9)
    mb = (Bs * T * 4 + Bs * period * pitch * 32) / 1e6
    print(f"im2col_c1 {name:6s} {us:7.1f} us  {mb / us * 1e3:7.0f} GB/s", flush=True)      # MB / us = TB/s
    P = [torch.randn(Bs * period, pitch, 16, device=dev) for _ in range(3)]
    us = graph_time_us(lambda i: ops.gather_c1(P[i % 3], (Bs, T), Lin, Lout, K, stride, pad, period, pool), n=9)
    print(f"gather_c1 {name:6s} {us:7.1f} us", flush=True)

# weight-norm backward of one MSD net (96-192-384-768 channels, k15): dwt partial tiles -> (dv, dg)
jobs = []
for C0, C1, K, S in [(96, 16, 15, 1), (192, 96, 15, 2), (384, 192, 15, 1), (768, 384, 15, 1), (768, 768, 5, 1)]:
    v = torch.randn(C0, C1, K, device=dev)
    g = torch.rand(C0, 1, 1, device=dev) + 0.5
    norm = v.flatten(1).norm(dim=1)
    C0p, C1p = (C0 + 15) // 16 * 16, (C1 + 15) // 16 * 16
    dwt = torch.randn(S, K, C0p, C1p, device=dev)
    jobs.append((dwt, v, g, norm))
n_par = sum(j[1].numel() for j in jobs)
us = graph_time_us(lambda i: ops.weight_norm_bwd_multi(jobs), n=6)
print(f"weight_norm_bwd_multi ({n_par / 1e6:.1f} M weights) {us:7.1f} us", flush=True)

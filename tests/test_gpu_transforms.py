"""Training-batch transforms on the GPU (csrc/augment.cu through rave_b200/transforms.py): the reference's own outputs
(tests/golden/transforms.pt) and the numpy restatement (oracle/transforms_oracle.py) element by element, a naive serial
recurrence, the device draws' statistics, determinism, batch invariance, CUDA-graph capture, the GraphedTrainer path
and the launch count."""
import math
import os

import numpy as np
import pytest
import torch
from scipy.signal import lfilter

from oracle import transforms_oracle as TO
from oracle.make_golden_transforms import make_input
from rave_b200 import _lib
from rave_b200 import transforms as T

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "transforms.pt")
SR = 44100


def assert_ulp(got, ref, what="", atol=1e-12):
    """every element within one float32 ulp of ref, + atol (a scalar or one value per example)"""
    got = np.asarray(got, np.float64)
    ref32 = np.asarray(ref, np.float32)
    atol = np.asarray(atol, np.float64).reshape((-1,) + (1,) * (ref32.ndim - 1)) if np.ndim(atol) else atol
    tol = np.spacing(np.abs(ref32)).astype(np.float64) + atol
    err = np.abs(got - ref32.astype(np.float64))
    bad = err > tol
    assert not bad.any(), (what, int(bad.sum()), float((err / tol).max()))


def scan_atol(raw, n_signal, draws, normalize):
    """Per example: 1e-12 + the float64 rounding the allpass recurrence amplifies.  An error made at one step reaches
    the output through the all-pole part's impulse response h, so lfilter and the scan each carry up to about
    eps64 * sum |h| * max |w| (sum |h| ~ 1 / (1 - .99)^2 = 1e4 for a pole at 20 Hz): ~1e-12 absolute, which only
    matters where the output is close to zero."""
    out = []
    for i in range(raw.shape[0]):
        if not draws[i][1]:
            out.append(1e-12)
            continue
        b, a = TO.pole_to_z_filter(draws[i][2], .99)
        g = np.abs(lfilter([1.0], a, np.r_[1.0, np.zeros(20000)])).sum()
        x = np.abs(TO.decode(raw[i])).max() + 2**-16
        out.append(1e-12 + 8 * np.finfo(np.float64).eps * g * 4 * x * (10**1.5 if normalize else 1.0))
    return np.array(out)


def run(raw_np, n_signal, draws, noise, normalize=False, derivative=False, augmentations=()):
    B, C, L = raw_np.shape
    t = T.get_transforms(SR, n_signal, derivative=derivative, normalize=normalize, augmentations=augmentations,
                         n_channels=C)
    out = t(torch.from_numpy(raw_np).cuda(), draws=torch.as_tensor(draws, dtype=torch.float64).cuda(),
            noise=torch.from_numpy(noise).cuda())
    torch.cuda.synchronize()
    return out.cpu().numpy()


def test_reference_fixture_cases():
    fx = torch.load(GOLDEN, weights_only=False)
    for case in fx["cases"]:
        C, N, L, seed = case["C"], case["N"], case["L"], case["seed"]
        raw = make_input(seed, C, L, case["kind"])
        np.random.seed(seed)
        noise = np.random.rand(C, N)
        got = run(raw[None], N, case["draws"][None].numpy(), noise[None], case["normalize"], case["derivative"])
        assert_ulp(got[0], case["out"].numpy(), case["name"])


def _random_batch(seed, B, C, L, int16=True):
    rng = np.random.default_rng(seed)
    kinds = ["loud", "quiet", "loud", "float"]
    raw = np.stack([make_input(seed * 100 + i, C, L, "float" if not int16 else kinds[i % 3]) for i in range(B)])
    return raw, rng


def _draws(rng, B, L, N, omegas=None):
    d = np.zeros((B, 4))
    d[:, 0] = rng.integers(0, L - N + 1, B)
    d[:, 1] = rng.random(B) < 0.8
    d[:, 2] = omegas if omegas is not None else 2 * np.pi * np.exp(rng.uniform(np.log(20), np.log(2000), B)) / SR
    d[:, 3] = rng.random(B) < 0.9
    d[0, 1] = 1
    if B > 1:
        d[1, 1] = 0
    return d


# (B, C, N, L, int16, normalize, derivative)
LONG = [
    (32, 1, 131072, 2 * 131072, True, False, False),
    (32, 1, 131072, 2 * 131072, True, True, True),
    (4, 2, 65536, 65536, False, True, False),          # L = n_signal: offset 0
    (3, 1, 1000, 3000, True, True, True),              # n_signal smaller than one scan chunk
    (4, 2, 5003, 9000, True, False, True),             # not a multiple of the chunk
]


@pytest.mark.parametrize("B,C,N,L,int16,normalize,derivative", LONG)
def test_long_rows_vs_restatement(B, C, N, L, int16, normalize, derivative):
    raw, rng = _random_batch(B + N % 97, B, C, L, int16)
    d = _draws(rng, B, L, N)
    noise = rng.random((B, C, N))
    got = run(raw, N, d, noise, normalize, derivative)
    ref = TO.transform_batch(raw, N, d, noise, normalize, derivative, device_log10=True)
    assert_ulp(got, ref, (B, C, N, L), scan_atol(raw, N, d, normalize))


@pytest.mark.parametrize("derivative", [False, True])
def test_poles_at_both_ends_of_the_range(derivative):
    B, C, N, L = 4, 1, 20000, 30000
    raw, rng = _random_batch(7, B, C, L)
    omegas = 2 * np.pi * np.array([20.0, 20.0 * (1 + 1e-9), 2000.0, 2000.0 * (1 - 1e-9)]) / SR
    d = _draws(rng, B, L, N, omegas)
    d[:, 1] = 1
    noise = rng.random((B, C, N))
    got = run(raw, N, d, noise, True, derivative)
    assert_ulp(got, TO.transform_batch(raw, N, d, noise, True, derivative, device_log10=True), "poles",
               scan_atol(raw, N, d, True))


def test_serial_recurrence_one_row():
    N, L = 6000, 7000
    raw = make_input(5, 1, L, "loud")
    off, omega = 123, 2 * np.pi * 300 / SR
    rng = np.random.default_rng(5)
    noise = rng.random((1, N))
    got = run(raw[None], N, np.array([[off, 1, omega, 1]]), noise[None])[0, 0]
    x = (raw.astype(np.float32) / np.float32(32767))[0, off:off + N].astype(np.float64)
    re, im = .99 * math.cos(omega), .99 * math.sin(omega)
    a2, a1 = math.hypot(re, im) ** 2, -2 * re
    y = np.zeros(N)
    for n in range(N):
        acc = a2 * x[n]
        if n >= 1:
            acc += a1 * x[n - 1] - a1 * y[n - 1]
        if n >= 2:
            acc += x[n - 2] - a2 * y[n - 2]
        y[n] = acc
    assert_ulp(got, y + noise[0] / 2**16, "serial", scan_atol(raw[None], N, [[off, 1, omega, 1]], False))


def test_device_draw_statistics():
    torch.cuda.manual_seed(123)
    n, L, N = 1 << 18, 40 + 1000, 1000
    d = T.sample_draws(n, L, N, SR, keep_prob=0.9, device="cuda").cpu()
    off = d[:, 0].long()
    assert off.min() == 0 and off.max() == L - N
    from scipy.stats import chisquare
    assert chisquare(torch.bincount(off, minlength=L - N + 1).numpy()).pvalue > 1e-4
    f = d[:, 2] * SR / (2 * math.pi)
    lf = ((f.log() - math.log(20)) / (math.log(2000) - math.log(20))).numpy()
    assert lf.min() >= -1e-12 and lf.max() <= 1 + 1e-12
    assert chisquare(np.histogram(lf, bins=64, range=(0, 1))[0]).pvalue > 1e-4
    assert abs(d[:, 1].mean().item() - 0.8) < 5 * math.sqrt(0.16 / n)
    assert abs(d[:, 3].mean().item() - 0.9) < 5 * math.sqrt(0.09 / n)


def test_device_dequantisation_noise():
    B, C, N = 8, 2, 1 << 17
    t = T.get_transforms(SR, N, n_channels=C)
    raw = torch.zeros(B, C, N, dtype=torch.float32, device="cuda")
    draws = torch.tensor([[0, 0, 0.1, 1]] * B, dtype=torch.float64, device="cuda")
    # float32(0 + u / 2^16) * 2^16: u in [0, 1) rounded to float32, which can round up to 1 as the reference's does
    q = t(raw, draws=draws).double().cpu() * 2**16
    assert q.min() >= 0 and q.max() <= 1
    m = q.numel()
    assert abs(q.mean().item() - 0.5) < 5 * math.sqrt(1 / 12 / m)
    assert abs(q.var().item() - 1 / 12) < 5 * math.sqrt(1 / 180 / m)
    # rows differ from each other
    assert not torch.equal(q[0, 0], q[0, 1]) and not torch.equal(q[0, 0], q[1, 0])


def test_determinism_from_generator_state():
    raw = torch.randint(-30000, 30000, (16, 2, 50000), dtype=torch.int16, device="cuda")
    t = T.get_transforms(SR, 30000, normalize=True, derivative=True, augmentations=[T.RandomMute(0.3)], n_channels=2)
    torch.cuda.manual_seed(9)
    a = t(raw)
    torch.cuda.manual_seed(9)
    b = t(raw)
    c = t(raw)
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert not torch.equal(a, c)


def test_batch_invariance():
    B, C, N, L = 32, 1, 40000, 60000
    raw, rng = _random_batch(3, B, C, L)
    d = _draws(rng, B, L, N)
    noise = rng.random((B, C, N))
    full = run(raw, N, d, noise, True, True)
    for i in (0, 5, 31):
        one = run(raw[i:i + 1], N, d[i:i + 1], noise[i:i + 1], True, True)
        assert np.array_equal(one.view(np.int32), full[i:i + 1].view(np.int32)), i
    # the Philox noise is keyed by (b, c, n): row 0 alone and inside the batch see the same uniforms
    t = T.get_transforms(SR, N, n_channels=C)
    rawg, dg = torch.from_numpy(raw).cuda(), torch.from_numpy(d).cuda()
    torch.cuda.manual_seed(4)
    a = t(rawg, draws=dg)
    torch.cuda.manual_seed(4)
    b = t(rawg[:1], draws=dg[:1])
    assert torch.equal(a[:1].view(torch.int32), b.view(torch.int32))


def test_cuda_graph_replay_equals_eager():
    raw = torch.randint(-30000, 30000, (8, 1, 70000), dtype=torch.int16, device="cuda")
    t = T.get_transforms(SR, 65536, normalize=True, augmentations=[T.RandomMute(0.2)])
    out = torch.empty(8, 1, 65536, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        t(raw, out=out)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        t(raw, out=out)
    for seed in (1, 2):
        torch.cuda.manual_seed(seed)
        eager = t(raw)
        torch.cuda.manual_seed(seed)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out.view(torch.int32), eager.view(torch.int32)), seed


def test_out_into_graphed_trainer_static_batch():
    from rave_b200 import configs
    from rave_b200.graphs import GraphedTrainer
    torch.manual_seed(0)
    m = configs.build_rave("v2", capacity=16, latent_size=16, disc_capacity=16).cuda().train()
    raw = torch.randint(-20000, 20000, (2, 1, 2 * 65536), dtype=torch.int16, device="cuda")
    t = T.get_transforms(SR, 65536, normalize=True)
    tr = GraphedTrainer(m, t(raw), warmup_steps=1)
    x = tr.x_static
    ptr = x.data_ptr()
    y = t(raw, out=x)
    assert y.data_ptr() == ptr and torch.isfinite(x).all() and x.abs().max() > 0
    logs = tr.step(x, 0)
    torch.cuda.synchronize()
    assert all(torch.isfinite(torch.as_tensor(v)).all() for v in logs.values() if isinstance(v, torch.Tensor))


def test_launch_count():
    raw = torch.zeros(4, 1, 5000, dtype=torch.int16, device="cuda")
    for normalize, launches in ((False, 1), (True, 2)):
        t = T.get_transforms(SR, 4096, normalize=normalize, derivative=True)
        n0 = _lib.launch_count()
        t(raw)
        assert _lib.launch_count() - n0 == launches

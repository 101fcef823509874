"""GPU: the export's resampler (csrc/resample.cu, rave_b200.resampler) against the float64 oracle
(oracle/resampler_oracle.py, pinned to the reference by tests/test_resampler_cpu.py) element by element within the
kernel's precision contract, against the reference's fixture, on long and odd rows, for determinism and batch
invariance, and inside ExportedRAVE(target_sr=...) on tiny models."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import resampler_oracle as RO
from rave_b200 import _lib, cc, configs
from rave_b200.export import ExportedRAVE
from rave_b200.resampler import Resampler
from tests.conftest import rel_l2

pytestmark = pytest.mark.gpu

SR = 48000


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _resampler(ratio, mode):
    with cc.configure(padding_mode=mode):
        return Resampler(ratio * SR, SR).cuda()


def _banks(rs):
    """(W, stride, pad) of each direction."""
    return {"down": (rs.downsample.weight.detach().reshape(1, -1), rs.ratio, rs.downsample._pad),
            "up": (rs.upsample.weight.detach().reshape(rs.ratio, -1), 1, rs.upsample._pad)}


def _run(rs, direction, x):
    return rs.to_model_sampling_rate(x) if direction == "down" else rs.from_model_sampling_rate(x)


def _fir64(x, W, stride, pad):
    """RO.fir on the device in float64, for rows too long for numpy: (y, sum_k |W x|)."""
    P, K = W.shape
    xp = F.pad(x.double().reshape(-1, 1, x.shape[-1]), pad)
    Wd = W.double()[:, None]
    y = F.conv1d(xp, Wd, stride=stride).permute(0, 2, 1).reshape(*x.shape[:-1], -1)
    a = F.conv1d(xp.abs(), Wd.abs(), stride=stride).permute(0, 2, 1).reshape(*x.shape[:-1], -1)
    return y, a


def _within(got, want, scale, K, factor=1.0):
    ulp = torch.from_numpy(np.spacing(np.abs(got.float().cpu().numpy()))).double()
    bound = ulp + K * 2.0 ** -24 * scale.double().cpu()
    err = (got.double().cpu() - want.double().cpu()).abs()
    return bool((err <= factor * bound).all()), (err / bound.clamp_min(1e-300)).max().item()


@pytest.mark.parametrize("mode", ["centered", "causal"])
@pytest.mark.parametrize("ratio", [2, 3])
@pytest.mark.parametrize("shape", [(1, 1, 4096), (2, 2, 3001), (3, 1, 5), (1, 2, 2 ** 13 + 1)])
def test_directions_against_float64_oracle(ratio, mode, shape):
    rs = _resampler(ratio, mode)
    x = (torch.randn(*shape, generator=_g(ratio + shape[-1])) * .5).cuda()
    x[..., :3] = torch.tensor([1e4, -3e-3, 0.0])[:min(3, shape[-1])]        # a wide dynamic range
    for direction, (W, S, pad) in _banks(rs).items():
        got = _run(rs, direction, x)
        want, scale = RO.fir(x.double().cpu().numpy(), W.double().cpu().numpy(), S, pad)
        n = (shape[-1] - 1) // S + 1
        assert got.shape == (*shape[:-1], n * W.shape[0])
        ok, worst = _within(got, torch.from_numpy(want), torch.from_numpy(scale), W.shape[1])
        assert ok, (direction, worst)


@pytest.mark.parametrize("case", range(4))
def test_against_the_reference_fixture(case):
    fx = torch.load("tests/golden/resampler.pt")
    c = fx["directions"][case]
    rs = _resampler(c["ratio"], c["mode"])
    assert torch.equal(rs.downsample.weight.cpu(), c["down_weight"]) and torch.equal(rs.upsample.weight.cpu(),
                                                                                      c["up_weight"])
    banks = _banks(rs)
    for i, x in enumerate(c["x"]):
        x32 = x.float().cuda()
        for direction, ref64, ref32 in (("down", c["down64"][i], c["down32"][i]), ("up", c["up64"][i], c["up32"][i])):
            W, S, pad = banks[direction]
            got = _run(rs, direction, x32)
            _, scale = RO.fir(x.numpy(), W.double().cpu().numpy(), S, pad)
            scale = torch.from_numpy(scale)
            # the fixture's float64 runs on the float64 input: the float32 input adds at most 2^-24 sum |W x|
            ok, worst = _within(got, ref64, scale * (1 + 1 / W.shape[1]), W.shape[1])
            assert ok, (direction, worst)
            # the reference's float32 output lies within the same bound of float64: the two meet within twice it
            ok, worst = _within(got, ref32, scale * (1 + 1 / W.shape[1]), W.shape[1], factor=2.0)
            assert ok, (direction, worst)


@pytest.mark.parametrize("ratio", [2, 3])
def test_long_rows_and_odd_lengths(ratio):
    rs = _resampler(ratio, "centered")
    for L in (2 ** 21, 2 ** 21 - 7):
        x = (torch.randn(16, 1, L, generator=_g(L + ratio)) * .3).cuda()
        for direction, (W, S, pad) in _banks(rs).items():
            got = _run(rs, direction, x)
            want, scale = _fir64(x, W, S, pad)
            assert got.shape == want.shape
            ok, worst = _within(got, want, scale, W.shape[1])
            assert ok, (L, direction, worst)
            del got, want, scale


@pytest.mark.parametrize("ratio", [2, 3])
def test_bitwise_determinism_batch_invariance_and_one_launch(ratio):
    rs = _resampler(ratio, "causal")
    x = (torch.randn(4, 4, 70001, generator=_g(77)) * .5).cuda()
    for direction in ("down", "up"):
        n0 = _lib.launch_count()
        a = _run(rs, direction, x)
        assert _lib.launch_count() - n0 == 1
        assert torch.equal(a, _run(rs, direction, x))
        assert torch.equal(a[2:3, 1:2], _run(rs, direction, x[2:3, 1:2].contiguous()))
        assert torch.equal(a[1:3], _run(rs, direction, x[1:3].contiguous()))


# ------------------------------------------------------------------ ExportedRAVE(target_sr=...)
def _tiny(n_channels=1, seed=0):
    torch.manual_seed(seed)
    m = configs.build_rave("v2", sampling_rate=SR, capacity=16, latent_size=8, n_channels=n_channels).cuda()
    g = _g(seed + 1)
    with torch.no_grad():
        m.latent_pca.copy_(torch.linalg.qr(torch.randn(8, 8, generator=g, dtype=torch.float64))[0].float())
        m.latent_mean.copy_(torch.randn(8, generator=g) * .1)
        m.fidelity.copy_(torch.tensor([.5, .7, .9, .96, .97, .98, .99, 1.]))
    return m


def _oracle_path(plain, ratio, x, eps, noise, encode_ratio, reps=1):
    """The same calls without the resampler, the resampling done by the float64 oracle: down before encode; up after
    the model's decode, then the crop to T * encode_ratio."""
    filt = Resampler(ratio * SR, SR).downsample.weight.detach().reshape(-1).double().numpy()
    bank = RO.phase_bank(filt, ratio)
    xd = torch.from_numpy(RO.down(x.double().cpu().numpy(), filt, ratio)).float().cuda()
    z = plain.encode(xd, eps=eps)
    zr = z.repeat_interleave(reps, 0) if reps > 1 else z
    with torch.no_grad():
        y = plain.model.decode(plain.pre_process_latent(zr, noise))
    y = torch.from_numpy(RO.up(y.double().cpu().numpy(), bank))[..., :z.shape[-1] * encode_ratio]
    return z, y


@pytest.mark.parametrize("ratio", [2, 3])
@pytest.mark.parametrize("n_channels,channels", [(1, None), (2, None), (1, 2)])
def test_exported_target_sr_against_oracle_path(ratio, n_channels, channels):
    m = _tiny(n_channels)
    ex = ExportedRAVE(m, channels=channels, target_sr=ratio * SR)
    plain = ExportedRAVE(m, channels=channels)
    assert ex.sr == ratio * SR and plain.sr == SR and plain.resampler is None
    if ratio == 2:
        assert ex.encode_ratio == 2 * plain.encode_ratio
    x = (0.3 * torch.randn(2, n_channels, 3 * 2 ** 14 + 11, generator=_g(5))).clamp(-1, 1).cuda()
    T = ex.encode(x).shape[-1]
    reps = 2 if channels == 2 else 1
    g = _g(6)
    eps = torch.randn(2, 8, T, generator=g).cuda()
    noise = torch.randn(2 * reps, 8 - ex.latent_size, T, generator=g).cuda()
    z = ex.encode(x, eps=eps)
    z_want, y_want = _oracle_path(plain, ratio, x, eps, noise, ex.encode_ratio, reps)
    assert z.shape == z_want.shape == (2, ex.latent_size, T)
    assert rel_l2(z, z_want) < 1e-5
    y = ex.decode(z_want, noise=noise)
    if reps > 1:
        y_want = y_want.reshape(2, reps * n_channels, -1)
    assert y.shape == (2, channels or n_channels, T * ex.encode_ratio) == y_want.shape
    assert rel_l2(y, y_want) < 1e-5


@pytest.mark.parametrize("ratio", [2, 3])
def test_exported_target_sr_graph_replay(ratio):
    ex = ExportedRAVE(_tiny(), target_sr=ratio * SR)
    x = (0.3 * torch.randn(2, 1, 2 ** 15, generator=_g(14))).clamp(-1, 1).cuda()
    T = ex.encode(x).shape[-1]
    g = _g(15)
    eps = torch.randn(2, 8, T, generator=g).cuda()
    noise = torch.randn(2, 8 - ex.latent_size, T, generator=g).cuda()

    def run():
        return ex.decode(ex.encode(x, eps=eps), noise=noise)

    eager = run()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = run()
    graph.replay()
    torch.cuda.synchronize()
    assert out.shape == (2, 1, T * ex.encode_ratio)
    assert torch.equal(out, eager)

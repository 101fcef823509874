"""GPU: the exported model's latent kernels (csrc/export.cu) against the float64 oracle (oracle/export_oracle.py, pinned
to the reference by tests/test_export_cpu.py), and rave_b200.ExportedRAVE on tiny models of every latent kind, in fp32 and
on the bf16 engine: encode / decode against the oracle applied to model.encode / model.decode, `channels`, determinism and
CUDA-graph capture."""
import pytest
import torch

import rave_b200
from oracle import export_oracle as EO
from rave_b200 import configs, ops
from rave_b200.export import ExportedRAVE
from tests.conftest import rel_l2

pytestmark = pytest.mark.gpu

# fp32 kernels against float64 on O(1) inputs: fixed-order fp32 sums of <= 128 terms
TOL = 1e-5


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _orth(L, g):
    return torch.linalg.qr(torch.randn(L, L, generator=g, dtype=torch.float64))[0]


# ------------------------------------------------------------------ kernels
@pytest.mark.parametrize("B,L,T,l", [(3, 16, 37, 5), (1, 128, 64, 32), (2, 8, 5, 8)])
def test_latent_project_and_unproject(B, L, T, l):
    g = _g(B * 100 + L)
    z = torch.randn(B, 2 * L, T, generator=g, dtype=torch.float64) * 2
    eps = torch.randn(B, L, T, generator=g, dtype=torch.float64)
    mean = torch.randn(L, generator=g, dtype=torch.float64) * .3
    pca = _orth(L, g)
    f = lambda t: t.float().cuda()  # noqa: E731
    got = ops.latent_project(f(z), f(eps), f(mean), f(pca), l)
    want = EO.variational_post(f(z).double(), f(eps).double(), f(mean).double(), f(pca).double(), l)
    assert got.shape == (B, l, T) and rel_l2(got, want) < TOL
    assert torch.equal(got, ops.latent_project(f(z), f(eps), f(mean), f(pca), l))           # deterministic
    noise = torch.randn(B, L - l, T, generator=g, dtype=torch.float64)
    back = ops.latent_unproject(got, f(noise) if l < L else None, f(mean), f(pca))
    want = EO.variational_pre(got.double(), f(noise).double(), f(mean).double(), f(pca).double())
    assert back.shape == (B, L, T) and rel_l2(back, want) < TOL


def _rvq_case(B, D, T, Q, K, seed, scale=1.0):
    g = _g(seed)
    cbs = torch.randn(Q, K, D, generator=g) * (0.5 ** torch.arange(Q, dtype=torch.float32))[:, None, None]
    x = torch.randn(B, D, T, generator=g) * scale
    return x.cuda(), cbs.cuda()


# An fp32 distance |r|^2 - 2 r.c + |c|^2 (D fixed-order terms, then two additions) is off by at most ~(2 D + 8) 2^-24 of
# |r|^2 + max|c|^2.  The float64 argmin runs on the residuals rounded to fp32 as the kernel's are (the subtraction is
# the same there), and a stage's code is compared with it when that stage and every earlier one of the frame have a
# best-to-second gap above this bound (EO.rvq_encode's relative gaps): a near tie changes every later residual.
def _argmin64(x, codebooks):
    return EO.rvq_encode(x.double(), codebooks.double(), return_gaps=True, residual_dtype=torch.float32)


def _clear(gaps, D):
    return (gaps > (2 * D + 8) * 2.0 ** -24).int().cumprod(1).bool()


@pytest.mark.parametrize("B,D,T,Q,K", [(2, 128, 300, 16, 1024), (3, 20, 41, 3, 100), (1, 256, 33, 2, 70)])
def test_rvq_encode_matches_float64_argmin(B, D, T, Q, K):
    x, cbs = _rvq_case(B, D, T, Q, K, seed=D + K)
    got = ops.rvq_encode(x, cbs)
    want, gaps = _argmin64(x, cbs)
    clear = _clear(gaps, D)
    assert clear.float().mean() > .5
    assert got.dtype == torch.int32 and got.shape == (B, Q, T)
    assert torch.equal(got.long()[clear], want[clear])
    assert torch.equal(got, ops.rvq_encode(x, cbs))                # two runs, same bits


def test_rvq_encode_recovers_codes_of_codebook_sums():
    # stage scales 0.2^q: what the later stages add stays well inside half the distance between two codes of a stage
    B, D, T, Q, K = 2, 128, 257, 4, 1024
    g = _g(7)
    cbs = torch.randn(Q, K, D, generator=g) * (0.2 ** torch.arange(Q, dtype=torch.float32))[:, None, None]
    k = torch.randint(0, K, (B, Q, T), generator=g)
    x = sum(cbs[q][k[:, q]] for q in range(Q)).permute(0, 2, 1)
    x = x + 1e-6 * torch.randn(x.shape, generator=g)
    got = ops.rvq_encode(x.contiguous().cuda(), cbs.cuda())
    assert torch.equal(got.long().cpu(), k)
    assert torch.equal(got.long().cpu(), EO.rvq_encode(x.double(), cbs.double()))


def test_rvq_encode_ties_go_to_the_lowest_code():
    D, K = 8, 64
    cbs = torch.zeros(1, K, D)
    cbs[0, 10] = 1.0
    cbs[0, 40] = 1.0                                               # duplicate of code 10
    x = torch.zeros(1, D, 3)
    x[0, :, 0] = 1.0                                               # codes 10 and 40 tie
    got = ops.rvq_encode(x.cuda(), cbs.cuda()).cpu()
    assert got[0, 0].tolist() == [10, 0, 0]


def test_rvq_decode_clamps_truncates_and_appends_noise():
    B, D, T, Q, K, Nn = 2, 12, 19, 4, 37, 5
    _, cbs = _rvq_case(B, D, T, Q, K, seed=3)
    g = _g(4)
    codes = torch.randint(0, K, (B, Q, T), generator=g).float()
    codes[0, 0, :4] = torch.tensor([-3.7, K + 5.5, 2.9, -0.4])
    noise = torch.randn(B, Nn, T, generator=g)
    got = ops.rvq_decode(codes.cuda(), cbs, noise.cuda())
    want = EO.rvq_decode(codes.double(), cbs.double().cpu(), noise.double())
    assert got.shape == (B, D + Nn, T) and rel_l2(got, want) < TOL
    assert torch.equal(got[:, D:].cpu(), noise)
    assert rel_l2(ops.rvq_decode(codes.cuda(), cbs), want[:, :D]) < TOL


def test_sphere_to_angles_against_float64():
    B, L, T = 3, 16, 200
    x = torch.randn(B, L, T, generator=_g(9)).cuda()
    got = ops.sphere_to_angles(x)
    want = EO.sphere_to_angles(x.double())
    # arccos is ill-conditioned near +-1: the tight check where the float64 argument is away from it
    sq = x.double().flip(1).pow(2)
    sq[:, 1] += sq[:, 0]
    arg = x.double()[:, :-1] / sq[:, 1:].cumsum(1).flip(1).sqrt()
    calm = arg.abs() < .9999
    assert (got - want).abs()[calm].max() < TOL
    assert (got - want).abs().max() < 1e-3


def test_sphere_zero_frame_and_reflection():
    x = torch.randn(2, 5, 4, generator=_g(10))
    x[0, :, 0] = 0                                                 # NaN angles, as the reference gives
    x[0, -1, 1], x[0, -1, 2] = -abs(x[0, -1, 1]), abs(x[0, -1, 2])
    got = ops.sphere_to_angles(x.cuda()).cpu()
    assert torch.isnan(got[0, :, 0]).all() and not torch.isnan(got[:, :, 1:]).any()
    assert got[0, -1, 1] > 0 and got[0, -1, 2] <= 0                # reflected last angle lies in (0, 1)
    want = EO.sphere_to_angles(x.double())
    assert torch.allclose(got[:, :, 1:].double(), want[:, :, 1:], atol=1e-5)


def test_angles_sphere_round_trip():
    B, L, T = 2, 12, 300
    g = _g(11)
    a = torch.rand(B, L - 1, T, generator=g) * 1.8 - .9            # away from the poles (+-1)
    a[:, -1] = torch.rand(B, T, generator=g) * 1.98 - .99          # the last angle spans the circle
    s = ops.angles_to_sphere(a.cuda())
    assert rel_l2(s, EO.angles_to_sphere(a.double())) < TOL
    assert torch.allclose(s.norm(dim=1), torch.ones(B, T, device="cuda"), atol=1e-5)
    back = ops.sphere_to_angles(s).cpu()
    d = (back - a + 1) % 2 - 1                                     # wrapped difference
    assert d.abs().max() < 1e-5
    wide = torch.rand(B, L - 1, T, generator=g) * 8 - 4            # outside [-1, 1): floor modulo
    assert rel_l2(ops.angles_to_sphere(wide.cuda()), EO.angles_to_sphere(wide.double())) < TOL


# ------------------------------------------------------------------ ExportedRAVE on tiny models
KINDS = ["v2", "discrete", "v2_wasserstein", "v2_spherical", "v3"]


def _tiny(name, seed=0):
    torch.manual_seed(seed)
    m = configs.build_rave(name, capacity=16, latent_size=8).cuda()
    g = _g(seed + 1)
    with torch.no_grad():
        m.latent_pca.copy_(_orth(8, g).float())
        m.latent_mean.copy_(torch.randn(8, generator=g) * .1)
        m.fidelity.copy_(torch.tensor([.5, .7, .9, .96, .97, .98, .99, 1.]))   # latent_size 4 at fidelity .95
        if name == "discrete":
            for q, vq in enumerate(m.encoder.rvq.layers):
                vq._codebook.embed.copy_(torch.randn(vq.codebook_size, 8, generator=g) * .5 ** q)
    return m


def _oracle_post(ex, z, eps):
    z = z.double()
    if ex.kind == "variational":
        return EO.variational_post(z, eps.double(), ex.model.latent_mean.double(), ex.model.latent_pca.double(),
                                   ex.latent_size)
    if ex.kind == "discrete":
        return _argmin64(z, ex._codebooks())
    if ex.kind == "wasserstein":
        return z
    return EO.sphere_to_angles(z)


def _oracle_pre(ex, z, noise):
    z = z.double()
    if ex.kind == "variational":
        return EO.variational_pre(z, noise.double(), ex.model.latent_mean.double(), ex.model.latent_pca.double())
    if ex.kind == "discrete":
        return EO.rvq_decode(z, ex._codebooks().double(), noise.double())
    if ex.kind == "wasserstein":
        return EO.wasserstein_pre(z, noise.double())
    return EO.angles_to_sphere(z)


def _draws(ex, B, T, reps=1, seed=0):
    g = _g(seed)
    eps = torch.randn(B, ex.full_latent_size, T, generator=g).cuda() if ex.kind == "variational" else None
    n = ex.full_latent_size - ex.latent_size if ex.kind == "variational" else ex.n_noise
    noise = torch.randn(B * reps, n, T, generator=g).cuda() if n else None
    return eps, noise


@pytest.fixture(params=["fp32", "bf16"])
def precision(request):
    rave_b200.set_precision(request.param)
    yield request.param
    rave_b200.set_precision("fp32")


@pytest.mark.parametrize("name", KINDS)
def test_exported_encode_decode_against_oracle(name, precision):
    m = _tiny(name)
    ex = ExportedRAVE(m)
    assert ex.latent_size == {"v2": 4, "v3": 4, "discrete": 16, "v2_wasserstein": 8, "v2_spherical": 7}[name]
    x = (0.3 * torch.randn(2, 1, 2 ** 15, generator=_g(5))).clamp(-1, 1).cuda()
    T = x.shape[-1] // ex.encode_ratio
    eps, noise = _draws(ex, 2, T, seed=6)
    z = ex.encode(x, eps=eps)
    assert z.shape == (2, ex.latent_size, T) and z.dtype == torch.float32
    with torch.no_grad():
        raw = m.encode(x)
    want = _oracle_post(ex, raw, eps)
    if ex.kind == "discrete":
        codes, gaps = want
        clear = _clear(gaps, raw.shape[1])
        assert clear.float().mean() > .5
        assert torch.equal(z.long()[clear], codes[clear])
        z = codes.float().cuda()                     # decode the float64 codes: decode is then exactly comparable
    elif ex.kind == "spherical":
        assert (z - want).abs().max() < 1e-3 and rel_l2(z, want) < 1e-4       # arccos near +-1
    else:
        assert rel_l2(z, want) < TOL
    y = ex.decode(z, noise=noise)
    assert y.shape == (2, 1, T * ex.encode_ratio)
    with torch.no_grad():
        y_want = m.decode(_oracle_pre(ex, z, noise).float())[..., :T * ex.encode_ratio]
    # same decoder on latents that differ by fp32 rounding; the bf16 engine rounds its operands to 8 bits
    assert rel_l2(y, y_want) < (1e-5 if precision == "fp32" else 2e-2)


def test_channels_decode_each_example_with_its_own_noise():
    m = _tiny("v2")
    one, two = ExportedRAVE(m), ExportedRAVE(m, channels=2)
    x = (0.3 * torch.randn(2, 1, 2 ** 14, generator=_g(12))).clamp(-1, 1).cuda()
    T = x.shape[-1] // two.encode_ratio
    eps, noise = _draws(two, 2, T, reps=2, seed=13)
    z = two.encode(x, eps=eps)
    y = two.decode(z, noise=noise)
    assert y.shape == (2, 2, x.shape[-1])
    assert rel_l2(y[:, 0], y[:, 1]) > 1e-2                          # two different channels
    for b in range(2):
        for i in range(2):
            single = one.decode(z[b:b + 1], noise=noise[2 * b + i:2 * b + i + 1])
            assert rel_l2(y[b, i], single[0, 0]) < 1e-5


@pytest.mark.parametrize("name", ["v2", "discrete", "v2_spherical"])
def test_encode_decode_graph_replay(name):
    m = _tiny(name)
    ex = ExportedRAVE(m)
    x = (0.3 * torch.randn(2, 1, 2 ** 14, generator=_g(14))).clamp(-1, 1).cuda()
    T = x.shape[-1] // ex.encode_ratio
    eps, noise = _draws(ex, 2, T, seed=15)

    def injected():
        return ex.decode(ex.encode(x, eps=eps), noise=noise)

    def drawn():
        return ex.decode(ex.encode(x))

    eager = injected()
    drawn()
    torch.cuda.synchronize()
    g1, g2 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.graph(g1):
        out1 = injected()
    with torch.cuda.graph(g2):
        out2 = drawn()
    g1.replay()
    torch.cuda.synchronize()
    assert torch.equal(out1, eager)
    torch.cuda.manual_seed(123)
    g2.replay()
    first = out2.clone()
    g2.replay()
    assert not torch.equal(out2, first) or ex.kind == "spherical"   # fresh draws per replay (spherical draws none)
    torch.cuda.manual_seed(123)
    g2.replay()
    torch.cuda.synchronize()
    assert torch.equal(out2, first)

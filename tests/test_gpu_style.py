"""GPU: the v3 style transfer on the wgmma engine -- rave_adain_cl_stats / rave_adain_snake_cl_fwd against float64, the
reference's learn / transfer / reset sequence (tests/golden/style_v3_tiny.pt) in fp32 and on the bf16 engine, the eval
chains staying on the engine, the identity state costing nothing in accuracy, CUDA-graph replays across style changes,
and a full-size transfer against the fp32 path."""
import os

import pytest
import torch
import torch.nn as nn

import rave_b200
from oracle import style_oracle as S
from rave_b200 import _lib, blocks, cc, configs, engine, ops
from rave_b200.model import _pqmf_decode, _pqmf_encode
from tests.conftest import GOLDEN, rel_l2

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture
def bf16():
    rave_b200.set_precision("bf16")
    yield
    rave_b200.set_precision("fp32")


# ---------------------------------------------------------------------------------------------------------------------
# 1. the kernels against float64
# ---------------------------------------------------------------------------------------------------------------------

def _stream(B, L, C, seed, slack=5):
    """Channel-last bf16 stream [B][pitch][C] with zero slack rows; per (b, c) offsets of either sign and scales, so that
    |mean| is of the order of the std (the relative check of the mean is meaningful)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    pitch = L + slack
    off = (0.5 + torch.rand(B, 1, C, generator=g, device=DEV)) * torch.where(
        torch.rand(B, 1, C, generator=g, device=DEV) < 0.5, -1.0, 1.0)
    sc = 0.2 + torch.rand(B, 1, C, generator=g, device=DEV)
    h = torch.zeros(B, pitch, C, device=DEV, dtype=torch.bfloat16)
    h[:, :L] = ((torch.randn(B, L, C, generator=g, device=DEV) + off) * sc).to(torch.bfloat16)
    return h


def _buffers(C, seed, n_x=0.0, n_y=0.0, learn_x=0.0, learn_y=0.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    N = cc.MAX_BATCH_SIZE
    return dict(mean_x=torch.randn(N, C, 1, generator=g, device=DEV), std_x=0.5 + torch.rand(N, C, 1, generator=g, device=DEV),
                mean_y=torch.randn(N, C, 1, generator=g, device=DEV), std_y=0.5 + torch.rand(N, C, 1, generator=g, device=DEV),
                learn_x=torch.full((1,), learn_x, device=DEV), learn_y=torch.full((1,), learn_y, device=DEV),
                num_update_x=torch.full((1,), n_x, device=DEV), num_update_y=torch.full((1,), n_y, device=DEV))


def _stats(h, bufs, L):
    return ops.adain_cl_stats(h, L, *(bufs[k] for k in ("mean_x", "std_x", "mean_y", "std_y", "learn_x", "learn_y",
                                                       "num_update_x", "num_update_y")))


def _f64_stats(h, L):
    x = h[:, :L].double()
    return x.mean(1), x.std(1)        # [B, C]; NaN std for L = 1, as torch.std


CASES = [(1, 16, 2), (3, 96, 31), (64, 768, 31), (1, 768, 30000), (3, 96, 4096), (64, 16, 4096), (3, 16, 30000),
         (64, 96, 2), (1, 96, 30000), (3, 768, 2), (64, 96, 4096), (1, 16, 31)]


@pytest.mark.parametrize("B,C,L", CASES)
def test_stats_kernel_against_float64(B, C, L):
    h = _stream(B, L, C, seed=B * 7919 + C * 31 + L)
    h0 = h.clone()
    m64, s64 = _f64_stats(h, L)
    # the statistics themselves: learn_y from zero buffers with zero counters stores them exactly ((v - 0) / 1 + 0)
    b = _buffers(C, 1, learn_y=1.0)
    b["mean_y"].zero_(), b["std_y"].zero_()
    scale, shift = _stats(h, b, L)
    m, s = b["mean_y"][:B, :, 0].double(), b["std_y"][:B, :, 0].double()
    assert ((m - m64).abs() <= 1e-5 * m64.abs() + 1e-6 * s64).all(), (m - m64).abs().max().item()
    assert ((s - s64).abs() <= 1e-5 * s64).all(), ((s - s64).abs() / s64).max().item()
    assert torch.equal(scale, torch.ones_like(scale)) and torch.equal(shift, torch.zeros_like(shift))
    assert b["num_update_y"].item() == 1 and b["num_update_x"].item() == 0
    assert torch.equal(h, h0)
    # two runs are bit-identical
    b2 = _buffers(C, 1, learn_y=1.0)
    b2["mean_y"].zero_(), b2["std_y"].zero_()
    _stats(h, b2, L)
    assert torch.equal(b2["mean_y"], b["mean_y"]) and torch.equal(b2["std_y"], b["std_y"])


def _update64(old, stat, n):
    return old.double() + (stat - old.double()) / (n + 1)


@pytest.mark.parametrize("B,C,L", CASES[:6])
def test_stats_kernel_update_branches(B, C, L):
    h = _stream(B, L, C, seed=B + C + L)
    m64, s64 = _f64_stats(h, L)
    tol = dict(rtol=2e-5, atol=2e-6)
    # learn_y (learn_x ignored): the y buffers move, the x buffers do not, no transfer
    b = _buffers(C, 2, n_x=2.0, n_y=3.0, learn_x=1.0, learn_y=1.0)
    old = {k: v.clone() for k, v in b.items()}
    scale, shift = _stats(h, b, L)
    torch.testing.assert_close(b["mean_y"][:B, :, 0].double(), _update64(old["mean_y"][:B, :, 0], m64, 3.0), **tol)
    torch.testing.assert_close(b["std_y"][:B, :, 0].double(), _update64(old["std_y"][:B, :, 0], s64, 3.0), **tol)
    for k in ("mean_x", "std_x"):
        assert torch.equal(b[k], old[k])
    assert torch.equal(b["mean_y"][B:], old["mean_y"][B:])
    assert (b["num_update_y"].item(), b["num_update_x"].item()) == (4.0, 2.0)
    assert torch.equal(scale, torch.ones_like(scale)) and torch.equal(shift, torch.zeros_like(shift))
    # learn_x: the x buffers move, the transfer applies with the updated buffers
    b = _buffers(C, 3, n_x=0.0, n_y=2.0, learn_x=1.0)
    old = {k: v.clone() for k, v in b.items()}
    scale, shift = _stats(h, b, L)
    mx, sx = _update64(old["mean_x"][:B, :, 0], m64, 0.0), _update64(old["std_x"][:B, :, 0], s64, 0.0)
    torch.testing.assert_close(b["mean_x"][:B, :, 0].double(), mx, **tol)
    torch.testing.assert_close(b["std_x"][:B, :, 0].double(), sx, **tol)
    for k in ("mean_y", "std_y"):
        assert torch.equal(b[k], old[k])
    assert (b["num_update_y"].item(), b["num_update_x"].item()) == (2.0, 1.0)
    sc64 = old["std_y"][:B, :, 0].double() / (sx + 1e-5)
    torch.testing.assert_close(scale.double(), sc64, **tol)
    torch.testing.assert_close(shift.double(), old["mean_y"][:B, :, 0].double() - mx * sc64, rtol=2e-5, atol=2e-5)
    # nothing learned: buffers and counters untouched; the affine of the frozen statistics, or the identity when a
    # counter is zero
    for n_x, applies in ((5.0, True), (0.0, False)):
        b = _buffers(C, 4, n_x=n_x, n_y=1.0)
        old = {k: v.clone() for k, v in b.items()}
        scale, shift = _stats(h, b, L)
        for k in b:
            assert torch.equal(b[k], old[k]), k
        if applies:
            sc = b["std_y"][:B, :, 0] / (b["std_x"][:B, :, 0] + 1e-5)
            torch.testing.assert_close(scale, sc, rtol=1e-6, atol=0)
            torch.testing.assert_close(shift, b["mean_y"][:B, :, 0] - b["mean_x"][:B, :, 0] * sc, rtol=1e-6, atol=1e-6)
        else:
            assert torch.equal(scale, torch.ones_like(scale)) and torch.equal(shift, torch.zeros_like(shift))


def test_stats_kernel_nan_for_one_row_and_batch_limit():
    h = _stream(2, 1, 16, seed=5)
    b = _buffers(16, 5, learn_y=1.0)
    _stats(h, b, 1)
    assert torch.isnan(b["std_y"][:2]).all() and torch.isfinite(b["mean_y"][:2]).all()
    with pytest.raises(_lib.RaveB200Error, match="batch 65"):
        _stats(_stream(65, 31, 16, seed=6), _buffers(16, 6, learn_y=1.0), 31)
    with pytest.raises(_lib.RaveB200Error):
        _stats(_stream(2, 31, 12, seed=6), _buffers(12, 6, learn_y=1.0), 31)


def _snake64(x, alpha):
    a = alpha.double().view(1, 1, -1)
    return x + torch.sin(a * x) ** 2 / (a + 1e-9)


@pytest.mark.parametrize("B,C,L", CASES)
def test_adain_snake_kernel(B, C, L):
    h = _stream(B, L, C, seed=B * 3 + C + 7 * L)
    alpha = (0.5 + torch.rand(C, device=DEV)).reshape(C, 1)
    # identity: the operand is bit for bit the plain Snake kernel's, h is not rewritten
    one, zero = torch.ones(B, C, device=DEV), torch.zeros(B, C, device=DEV)
    h0 = h.clone()
    a = ops.adain_snake_cl_fwd(h, alpha, one, zero, L)
    assert torch.equal(a, ops.snake_cl_fwd(h0, alpha)) and torch.equal(h, h0)
    # an affine: h' = bf16(h scale + shift) in place, a = bf16(Snake(h')), slack rows zero in both
    g = torch.Generator(device=DEV).manual_seed(L)
    scale = 0.5 + torch.rand(B, C, generator=g, device=DEV)
    shift = torch.randn(B, C, generator=g, device=DEV)
    a = ops.adain_snake_cl_fwd(h, alpha, scale, shift, L)
    want = (h0[:, :L].double() * scale[:, None].double() + shift[:, None].double())
    ulp = want.abs() * 2.0 ** -8
    assert ((h[:, :L].double() - want).abs() <= ulp + 1e-30).all()
    a64 = _snake64(h[:, :L].double(), alpha)
    assert ((a[:, :L].double() - a64).abs() <= a64.abs() * 2.0 ** -8 + 1e-6).all()
    assert not h[:, L:].any() and not a[:, L:].any()
    a2 = ops.adain_snake_cl_fwd(h0.clone(), alpha, scale, shift, L)
    assert torch.equal(a2, a)


# ---------------------------------------------------------------------------------------------------------------------
# 2 - 5. the tiny v3 of the fixture
# ---------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def fixture():
    return S.load_fixture(os.path.join(GOLDEN, "style_v3_tiny.pt"))


def _tiny(g):
    torch.manual_seed(0)
    _, enc, dec = configs.make_autoencoder("v3", capacity=g["capacity"], latent_size=g["latent_size"],
                                           ratios=g["ratios"])
    holder = nn.Module()
    holder.encoder, holder.decoder = enc, dec
    shapes = [(k, tuple(v.shape)) for k, v in holder.named_parameters()]
    holder.load_state_dict(S.style_params(shapes, g["param_seed"]), strict=False)
    return holder.to(DEV).eval()


def _buffers_of(holder, B):
    return S.snapshot({k: v for k, v in holder.state_dict().items()}, B)


def _run_fixture_sequence(holder, g):
    out = []
    with torch.no_grad():
        for step in g["steps"]:
            assert blocks.update_adain(holder, **step["update_adain"]) == 22
            e = holder.encoder.encoder(g["inputs"][step["input"]].to(DEV))
            y = holder.decoder(g["latents"][step["input"]].to(DEV))
            out.append((e, y, _buffers_of(holder, g["B"])))
    return out


def test_reference_sequence_fp32(fixture):
    g = fixture
    got = _run_fixture_sequence(_tiny(g), g)
    for i, ((e, y, bufs), step) in enumerate(zip(got, g["steps"])):
        assert rel_l2(e, step["encoder"]) < 1e-4, i
        assert rel_l2(y, step["decoder"]) < 1e-4, i
        for k, v in step["buffers"].items():
            assert rel_l2(bufs[k], v) < 1e-4 if v.numel() > 1 else bufs[k].item() == v.item(), (i, k)


def test_reference_sequence_bf16_engine(fixture, bf16):
    """Outputs within 3e-2 rel-L2 of the reference.  Buffers against the float64 restatement fed the same inputs: each
    statistic is a mean (or root-mean-square deviation) of a stream the bf16 chain computes to ~1e-2 rel-L2, so its
    error is bounded by that stream error times the stream's rms; per layer and buffer, the rel-L2 of the (b, c) vector
    must stay below 3e-2 -- the chain's own end-to-end bound -- and the counters and flags are exact."""
    g = fixture
    got = _run_fixture_sequence(_tiny(g), g)
    holder = _tiny(g)
    sd = {k: v.detach().cpu().clone() for k, v in holder.state_dict().items()}
    ref64 = S.run_sequence(sd, g["inputs"], g["latents"], S.style_cfg(g["capacity"], g["latent_size"]),
                           dtype=torch.float64)
    worst = {}
    for i, ((e, y, bufs), step, (_, _, b64)) in enumerate(zip(got, g["steps"], ref64)):
        assert rel_l2(e, step["encoder"]) < 3e-2, (i, rel_l2(e, step["encoder"]))
        assert rel_l2(y, step["decoder"]) < 3e-2, (i, rel_l2(y, step["decoder"]))
        for k, v in b64.items():
            if v.numel() == 1:
                assert bufs[k].item() == v.item() == step["buffers"][k].item(), (i, k)
                continue
            r = rel_l2(bufs[k], v)
            worst[k.rsplit(".", 1)[-1]] = max(worst.get(k.rsplit(".", 1)[-1], 0.0), r)
            assert r < 3e-2, (i, k, r)
    print("worst buffer rel-L2 vs float64:", {k: f"{v:.2e}" for k, v in worst.items()})


def test_eval_chains_issue_no_fp32_conv(fixture, bf16, monkeypatch):
    g = fixture
    holder = _tiny(g)
    blocks.update_adain(holder, learn_target=True)
    n0 = _lib.launch_count()

    def refuse(*a, **k):
        raise AssertionError("fp32 parity conv launched by a v3 eval chain in bf16")
    monkeypatch.setattr(ops, "conv1d", refuse)
    monkeypatch.setattr(ops, "conv_transpose1d", refuse)
    with torch.no_grad():
        z = holder.encoder.encoder(g["inputs"]["target0"].to(DEV))
        y = holder.decoder(g["latents"]["target0"].to(DEV))
        blocks.update_adain(holder, learn_source=True)
        holder.encoder.encoder(g["inputs"]["source"].to(DEV))
        blocks.update_adain(holder)
        holder.decoder(g["latents"]["source"].to(DEV))
    assert torch.isfinite(z).all() and torch.isfinite(y).all() and _lib.launch_count() > n0
    # under autograd and for streaming modules the module path is kept
    with pytest.raises(AssertionError, match="fp32 parity conv"):
        holder.encoder.encoder(g["inputs"]["source"].to(DEV))


def test_cached_v3_keeps_the_module_path(bf16, monkeypatch):
    cc.use_cached_conv(True)
    try:
        _, enc, _ = configs.make_autoencoder("v3", capacity=16, latent_size=16)
    finally:
        cc.use_cached_conv(False)
    enc = enc.to(DEV).eval()

    def refuse(*a, **k):
        raise AssertionError("engine chain")
    monkeypatch.setattr(engine, "run_chain", refuse)
    with torch.no_grad():
        z = enc.encoder(torch.randn(1, 16, 512, device=DEV))
    assert torch.isfinite(z).all()


def test_identity_state_is_free(fixture, bf16):
    """No style state: the eval chains equal the train-mode no_grad chains bit for bit; so does a learn-target call."""
    g = fixture
    holder = _tiny(g)
    x, z = g["inputs"]["source"].to(DEV), g["latents"]["source"].to(DEV)
    with torch.no_grad():
        holder.train()
        e_tr, y_tr = holder.encoder.encoder(x), holder.decoder(z)
        holder.eval()
        blocks.update_adain(holder, reset_target=True, reset_source=True)
        e_ev, y_ev = holder.encoder.encoder(x), holder.decoder(z)
        assert torch.equal(e_ev, e_tr) and torch.equal(y_ev, y_tr)
        blocks.update_adain(holder, learn_target=True)
        e_l, y_l = holder.encoder.encoder(x), holder.decoder(z)
        assert torch.equal(e_l, e_tr) and torch.equal(y_l, y_tr)
        # ... and the learned statistics are those of the stream: one AdaIN learned once
        ad = next(m for m in holder.modules() if isinstance(m, blocks.AdaptiveInstanceNormalization))
        assert ad.num_update_y.item() == 1 and torch.isfinite(ad.std_y).all()


def test_graph_replays_follow_style_changes(fixture, bf16):
    g = fixture
    holder = _tiny(g)
    init = {k: v.clone() for k, v in holder.state_dict().items()}
    B, lat = g["B"], g["latent_size"]
    seq = [(dict(learn_target=True, reset_target=True, reset_source=True), "target0"), (dict(learn_target=True), "target1"),
           (dict(learn_source=True), "source"), (dict(), "source"), (dict(reset_target=True), "source")]

    def restore():
        with torch.no_grad():
            for k, v in holder.state_dict().items():
                v.copy_(init[k])

    def body(x):
        z = holder.encoder.encoder(x)
        return holder.decoder(z[:, :lat].contiguous())          # the posterior mean: no random draw in the graph

    eager = []
    with torch.no_grad():
        for kw, which in seq:
            blocks.update_adain(holder, **kw)
            eager.append((body(g["inputs"][which].to(DEV)).clone(), _buffers_of(holder, B)))
    restore()
    static_x = g["inputs"]["target0"].to(DEV).clone()
    with torch.no_grad():
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            body(static_x)                                   # warm-up in the identity state
        torch.cuda.current_stream().wait_stream(s)
        restore()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            static_y = body(static_x)
    restore()

    def replayed():
        out = []
        for kw, which in seq:
            blocks.update_adain(holder, **kw)
            static_x.copy_(g["inputs"][which].to(DEV))
            graph.replay()
            out.append((static_y.clone(), _buffers_of(holder, B)))
        return out
    run1 = replayed()
    restore()
    run2 = replayed()
    for i, ((ye, be), (y1, b1), (y2, b2)) in enumerate(zip(eager, run1, run2)):
        assert torch.equal(y1, ye), i
        assert torch.equal(y2, y1), i
        for k in be:
            assert torch.equal(b1[k], be[k]) and torch.equal(b2[k], b1[k]), (i, k)
    assert rel_l2(eager[3][0], eager[4][0]) > 1e-2          # the transfer changed the output


# ---------------------------------------------------------------------------------------------------------------------
# 6. full size
# ---------------------------------------------------------------------------------------------------------------------

def test_full_size_transfer_against_fp32():
    torch.manual_seed(11)
    pq, enc, dec = configs.make_autoencoder("v3")
    holder = nn.Module()
    holder.pqmf, holder.encoder, holder.decoder = pq, enc, dec
    holder = holder.to(DEV).eval()
    init = {k: v.clone() for k, v in holder.state_dict().items()}
    gen = torch.Generator(device=DEV).manual_seed(12)
    B, T = 4, 65536
    tgt = (0.5 * torch.randn(B, 1, T, generator=gen, device=DEV)).clamp(-1, 1)
    src = (0.1 * torch.randn(B, 1, T, generator=gen, device=DEV)).clamp(-1, 1)

    def run():
        with torch.no_grad():
            for k, v in holder.state_dict().items():
                v.copy_(init[k])
            for kw, x in ((dict(learn_target=True), tgt), (dict(learn_source=True), src), (dict(), src)):
                blocks.update_adain(holder, **kw)
                z = enc.encoder(_pqmf_encode(pq, x))
                y = _pqmf_decode(pq, dec(z[:, :128].contiguous()), batch_size=x.shape[:-2], n_channels=1)
        return y
    y32 = run()
    rave_b200.set_precision("bf16")
    try:
        y16 = run()
    finally:
        rave_b200.set_precision("fp32")
    r = rel_l2(y16, y32)
    print(f"full-size v3 transfer, B={B} T={T}: bf16 engine vs fp32 rel-L2 {r:.3e}")
    assert torch.isfinite(y16).all() and r < 3e-2, r

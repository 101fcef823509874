"""GPU: every launch of the bf16 engine's real training steps checked against float64, element by element.

tests/launch_checker.py wraps each rave_b200.ops entry point the engine calls; each call is run on the real kernel and
compared with the float64 evaluation of tests/tc_emulator.py on the same operands, under an error bound derived from
those operands (see the checker's docstring).  Workloads: three bf16 steps (phase-1 generator, phase-2 discriminator,
phase-2 generator) per configuration, eager, one discriminator stream; a bf16x3 encode -> decode; one bf16
VariationalPrior step.  Each checked conv / weight-gradient call is attributed to the kernel instance the dispatch runs for
it, predicted from the library's host-side plan queries (rave_conv1d_tc_plan, _pp_stages, _pp_fwd_stages), and each
workload prints its instances with the worst bound ratio of their launches.  The workloads also run under torch.profiler
as a cross-check of that prediction: the traced conv_tc* / wgrad_tc* kernels must appear, in order, among the predicted
ones (the trace may miss records; it may not contradict the prediction).  A synthetic sweep runs every instance the conv
dispatch can select and the weight-gradient geometries (one split, the 32-split cap, ragged channel counts) through the
same checker and fails if any selectable instance is left unchecked."""
import math
import re

import pytest
import torch

from tests import launch_checker as lc
from tests import test_launch_checker_cpu as selftest

pytestmark = pytest.mark.gpu

T = 65536
KERNEL_RE = re.compile(r"((?:conv_tc_pp_fwd_kernel|conv_tc_pp_kernel|conv_tc_kernel|wgrad_tc_kernel)<[^>]*>)")


@pytest.fixture
def bf16_engine(monkeypatch):
    import rave_b200
    from rave_b200 import discriminator
    monkeypatch.setattr(discriminator, "DISC_STREAMS", 1)
    rave_b200.set_precision("bf16")
    yield
    rave_b200.set_precision("fp32")


def _profile():
    from torch.profiler import ProfilerActivity, profile
    return profile(activities=[ProfilerActivity.CUDA])


def _instances(prof):
    """The library's tensor-core kernel instances in launch order."""
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    ev.sort(key=lambda e: e.time_range.start)
    out = []
    for e in ev:
        m = KERNEL_RE.search(e.name)
        if m:
            out.append(re.sub(r"\s+", "", m.group(1)))
    return out


def predict_instance(op, a):
    """The kernel instance the library's dispatch (conv1d_tc_fwd_impl, rave_conv1d_tc_wgrad) runs for a call, from its
    host-side plan queries; None for entry points outside the tensor-core conv families."""
    from rave_b200 import _lib, ops
    lib = _lib.load()
    if op == "conv1d_tc_wgrad":
        return f"wgrad_tc_kernel<{64 if a['Q_cl'].shape[2] <= 64 else 128}>"
    if op != "conv1d_tc":
        return None
    x3 = a["x3"]
    B, Cin = a["xa_cl"].shape[0], a["xa_cl"].shape[2] // (2 if x3 else 1)
    Cout = a["wt"].shape[1]
    _, Lout, K = lc._conv_rows(a)
    plan = lib.rave_conv1d_tc_plan(B, Cin, Cout, Lout, K)
    BN, BK = plan & 0xFFF, (plan >> 12) & 0xFFF
    if x3:
        return f"conv_tc_kernel<{BN},{BK},true>"
    out_f32 = a["out_f32"] is not None or a["want_f32"]
    out_act = a["out_act"] is not None or a["want_act"]
    bf16_only = out_act and a["res_cl"] is None and a["res_act"] is None and not out_f32
    fm, rs = a["fm_d"] is not None, a["res_bf16"] is not None
    b = lambda v: str(bool(v)).lower()
    if bf16_only and a["dact_src"] is not None and a["bias"] is None and a["act"] == ops.ACT_NONE and \
            lib.rave_conv1d_tc_pp_stages(B, Cin, Cout, Lout, K, int(fm), int(rs)) > 0:
        return f"conv_tc_pp_kernel<{BN},{BK},{b(fm)},{b(rs)}>"
    if bf16_only and a["dact_src"] is None and not rs and not fm and lib.rave_conv1d_tc_pp_fwd_stages(B, Cin, Cout, Lout,
                                                                                                    K) > 0:
        return f"conv_tc_pp_fwd_kernel<{BN},{BK},{b(a['bias'] is not None)},{b(a['act'] == ops.ACT_LEAKY)}>"
    return f"conv_tc_kernel<{BN},{BK},false>"


def _checker(workload, monkeypatch=None, **kw):
    ck = lc.LaunchChecker(workload, **kw)
    ck.instance_fn = predict_instance
    if monkeypatch is not None:
        ck.install(monkeypatch)
    return ck


def _cross_check(ck, prof):
    """The traced instances are the predicted ones, in launch order; records the trace lacks are allowed."""
    want = [i for i in ck.instances if i is not None]
    traced = _instances(prof)
    it = iter(want)
    bad = [t for t in traced if not any(t == w for w in it)]
    assert traced and not bad, (f"{ck.workload}: {len(traced)} traced tensor-core kernels are not a subsequence of the "
                                f"{len(want)} predicted; first mismatch {bad[:1]}")
    return len(traced), len(want)


def _instance_table(ck):
    rows = {}
    for inst, (_, _, st, _) in zip(ck.instances, ck.records):
        if inst is not None:
            r = rows.setdefault(inst, [0, lc.Stat()])
            r[0] += 1
            r[1].merge(st)
    print(f"  {'instance':44s} {'launches':>8s} {'worst bound':>11s} {'worst tile/limit':>16s}")
    for inst, (n, st) in sorted(rows.items()):
        print(f"  {inst:44s} {n:8d} {st.ratio:11.3g} {st.tile:16.3g}")
    return rows


def _report(ck, workload):
    fams = {}
    for op, fam, st, _ in ck.records:
        f = fams.setdefault(fam, [0, lc.Stat()])
        f[0] += 1
        f[1].merge(st)
    print(f"\n{workload}: {len(ck.records)} launches checked")
    for fam, (n, st) in sorted(fams.items()):
        print(f"  {fam:12s} {n:5d} launches  worst bound ratio {st.ratio:.3g} ({st.where})  worst tile "
              f"rel-L2 {st.tile_rel:.3g} = {st.tile:.3g} of its limit ({st.tile_where}); largest tile limit in force "
              f"{st.tile_limit:.3g}")


def _noise(B, C, seed):
    g = torch.Generator().manual_seed(seed)
    return (0.5 * torch.randn(B, C, T, generator=g)).clamp(-1, 1).cuda()


WORKLOADS = [
    ("v2", 32, {}),
    ("v2_small", 4, {}),
    ("v3", 4, {}),
    ("v2_nopqmf", 4, {}),
    ("v2_spectral", 4, {}),
    ("v2", 4, {"n_channels": 2}),
    ("v2_hybrid", 4, {}),
    ("discrete", 4, {}),
]


@pytest.mark.parametrize("name,B,kw", WORKLOADS, ids=[f"{n}-B{b}" + ("-stereo" if kw else "") for n, b, kw in WORKLOADS])
def test_training_steps_launch_by_launch(name, B, kw, bf16_engine, monkeypatch):
    from rave_b200 import configs
    torch.manual_seed(0)
    m = configs.build_rave(name, **kw).cuda().train()
    x = _noise(B, kw.get("n_channels", 1), 1)
    ck = _checker(f"{name} B={B}" + (" stereo" if kw else ""), monkeypatch)
    with _profile() as prof:
        ck.step = "phase-1 generator step"
        m.training_step(x, 1)
        ck.raise_if_failed()
        m.warmed_up = True
        ck.step = "phase-2 discriminator step"
        m.training_step(x, 0)
        ck.raise_if_failed()
        ck.step = "phase-2 generator step"
        m.training_step(x, 1)
        torch.cuda.synchronize()
    ck.raise_if_failed()
    _report(ck, ck.workload)
    _instance_table(ck)
    print("  traced / predicted tensor-core launches: %d / %d" % _cross_check(ck, prof))


def test_bf16x3_encode_decode_launch_by_launch(monkeypatch):
    import rave_b200
    from rave_b200 import configs
    from rave_b200.model import _pqmf_decode, _pqmf_encode
    torch.manual_seed(0)
    pq, enc, dec = configs.make_autoencoder("v2")
    for mod in (pq, enc, dec):
        mod.cuda().eval()
    x = _noise(4, 1, 2)
    ck = _checker("v2 bf16x3 encode/decode", monkeypatch)
    rave_b200.set_precision("bf16x3")
    try:
        with torch.no_grad(), _profile() as prof:
            ck.step = "encode"
            z = enc(_pqmf_encode(pq, x))
            zs = z[:, :z.shape[1] // 2]
            ck.step = "decode"
            _pqmf_decode(pq, dec(zs), batch_size=x.shape[:-2], n_channels=1)
            torch.cuda.synchronize()
    finally:
        rave_b200.set_precision("fp32")
    ck.raise_if_failed()
    _report(ck, ck.workload)
    assert any(r[1] == "conv_x3" for r in ck.records)
    _instance_table(ck)
    print("  traced / predicted tensor-core launches: %d / %d" % _cross_check(ck, prof))


def test_prior_step_launch_by_launch(monkeypatch):
    import rave_b200
    from rave_b200 import configs
    torch.manual_seed(0)
    m = configs.build_rave("v2")
    prior = configs.build_prior(m, latent_size=16).cuda()
    x = (0.3 * torch.randn(8, 1, prior.min_receptive_field, generator=torch.Generator().manual_seed(3))).clamp(-1, 1)
    ck = _checker("VariationalPrior bf16 step", monkeypatch)
    rave_b200.set_precision("bf16")
    try:
        with _profile() as prof:
            ck.step = "training step"
            loss = prior.training_step(x.cuda())
            loss.backward()
            torch.cuda.synchronize()
    finally:
        rave_b200.set_precision("fp32")
    ck.raise_if_failed()
    _report(ck, ck.workload)
    assert any(r[1] == "wgrad" for r in ck.records)
    _instance_table(ck)
    print("  traced / predicted tensor-core launches: %d / %d" % _cross_check(ck, prof))


# ------------------------------------------------------------------------------------------------ synthetic sweep
BKS, BNS = (64, 32, 16), (128, 96, 64, 48, 32, 16)
SWEEP_B, SWEEP_L = 2, 8448 + 40          # 67 x 2 M tiles (>= 132: BLOCK_N = Cout), a ragged last tile


def _conv_instance_cases():
    """(instance name, kind, BK, BN, flags, K) for every conv instance the dispatch can select; the pp kernels only where
    their ring gets stages (the dispatch falls back to conv_tc_kernel otherwise)."""
    from rave_b200 import _lib
    lib = _lib.load()
    cases = []
    for bk in BKS:
        for bn in BNS:
            for x3 in (False, True):
                cases.append((f"conv_tc_kernel<{bn},{bk},{str(x3).lower()}>", "x3" if x3 else "f32", bk, bn, (), 3))
            for fm in (False, True):
                for rs in (False, True):
                    if lib.rave_conv1d_tc_pp_stages(SWEEP_B, bk, bn, SWEEP_L, 3, int(fm), int(rs)) > 0:
                        cases.append((f"conv_tc_pp_kernel<{bn},{bk},{str(fm).lower()},{str(rs).lower()}>", "dgrad", bk,
                                      bn, (fm, rs), 3))
            Ks = [K for K in (1, 2, 3, 5, 8, 16, 24) if lib.rave_conv1d_tc_pp_fwd_stages(SWEEP_B, bk, bn, SWEEP_L, K) > 0]
            for bias in (False, True):
                for leaky in (False, True):
                    if Ks:
                        cases.append((f"conv_tc_pp_fwd_kernel<{bn},{bk},{str(bias).lower()},{str(leaky).lower()}>",
                                      "fwd", bk, bn, (bias, leaky), Ks[0]))
    return cases


def _conv_case_args(kind, bk, bn, flags, K, g):
    """A launch of the given kind (x3, f32 epilogue, pp forward, pp dgrad) at BLOCK_K = Cin, BLOCK_N = Cout."""
    B, L, Cin, Cout = SWEEP_B, SWEEP_L, bk, bn
    dev = "cuda"

    def bf(*s, scale=1.0):
        return (scale * torch.randn(*s, generator=g)).to(torch.bfloat16).to(dev)
    a = dict(xa_cl=None, wt=None, bias=None, res_cl=None, stride=1, dil=1, pad=((K - 1) // 2, K // 2), act=0, slope=0.2,
             want_f32=False, want_act=False, out_f32=None, out_act=None, out_rows=0, out_row_stride=0, out_row_offset=0,
             Lout=L, res_bf16=None, dact_src=None, Lin=L, res_act=None, res_slope=0.2, fm_d=None, fm_partner=None,
             x3=False, act_cs=0)
    if kind == "x3":
        xf = torch.randn(B, L, Cin, generator=g)
        hi = xf.to(torch.bfloat16)
        lo = (xf - hi.float()).to(torch.bfloat16)
        wf = torch.randn(K, Cout, Cin, generator=g) / math.sqrt(K * Cin)
        whi = wf.to(torch.bfloat16)
        wlo = (wf - whi.float()).to(torch.bfloat16)
        a.update(xa_cl=torch.cat([hi, lo], -1).to(dev), wt=torch.cat([whi, wlo], 0).to(dev), x3=True,
                 bias=torch.randn(Cout, generator=g).to(dev), want_f32=True, want_act=True, act=1)
        return a
    a.update(xa_cl=bf(B, L, Cin), wt=bf(K, Cout, Cin, scale=1 / math.sqrt(K * Cin)))
    if kind == "f32":
        a.update(want_f32=True, want_act=True, bias=torch.randn(Cout, generator=g).to(dev), act=1,
                 res_cl=torch.randn(B, L, Cout, generator=g).to(dev))
    elif kind == "fwd":
        bias, leaky = flags
        a.update(want_act=True, act=1 if leaky else 0, bias=torch.randn(Cout, generator=g).to(dev) if bias else None)
    else:
        fm, rs = flags
        a.update(want_act=True, dact_src=bf(B, L, Cout), res_bf16=bf(B, L, Cout) if rs else None,
                 fm_d=torch.tensor([0.25, -0.125], device=dev) if fm else None)
    return a


WGRAD_CASES = [
    # (B, L, Cm, Cn, K, stride, dil, pad_l): one split; the 32-split cap; ragged channel counts and length; BLOCK_N 64
    (1, 512, 64, 64, 1, 1, 1, 0),
    (4, 8192, 128, 64, 1, 1, 1, 0),
    (3, 1000, 96, 200, 5, 1, 3, 6),
    (5, 777, 136, 48, 3, 2, 1, 1),
    (32, 2048, 192, 96, 3, 1, 9, 9),
]


def _wgrad_case_args(case):
    B, L, Cm, Cn, K, stride, dil, pad_l = case
    g = torch.Generator().manual_seed(sum(case))
    P = torch.randn(B, L, Cm, generator=g).to(torch.bfloat16).cuda()
    Q = torch.randn(B, L * stride, Cn, generator=g).to(torch.bfloat16).cuda()
    return dict(P_cl=P, Q_cl=Q, K=K, stride=stride, dil=dil, pad_l=pad_l, Lp=L, Lq=L * stride,
                dbias=torch.zeros(Cm, device="cuda"))


def test_sweep_checks_every_selectable_instance():
    """Every conv instance the dispatch can select (the pp kernels where their ring gets stages) and both weight-gradient
    instances, each through the checker at a shape whose predicted instance is the intended one."""
    from rave_b200 import _lib, ops
    conv_cases = _conv_instance_cases()
    g = torch.Generator().manual_seed(11)
    ck = _checker("instance sweep", max_failures=1000)
    intended, splits = [], []
    with _profile() as prof:
        for name, kind, bk, bn, flags, K in conv_cases:
            ck.step = name
            ck.checked_call("conv1d_tc", ops.conv1d_tc, _conv_case_args(kind, bk, bn, flags, K, g))
            intended.append(name)
        for case in WGRAD_CASES:
            ck.step = str(case)
            ck.checked_call("conv1d_tc_wgrad", ops.conv1d_tc_wgrad, _wgrad_case_args(case))
            intended.append(f"wgrad_tc_kernel<{64 if case[3] <= 64 else 128}>")
            splits.append(_lib.load().rave_conv1d_tc_wgrad_splits(case[0], case[2], case[1], case[3], case[4]))
    ck.raise_if_failed()
    wrong = [(w, p) for w, p in zip(intended, ck.instances) if w != p]
    assert not wrong, f"cases whose shape does not select the intended instance: {wrong[:8]}"
    assert 1 in splits and 32 in splits, splits
    selectable = {c[0] for c in conv_cases} | {"wgrad_tc_kernel<64>", "wgrad_tc_kernel<128>"}
    missing = selectable - set(ck.instances)
    assert not missing, f"selectable instances never checked: {sorted(missing)}"
    rows = _instance_table(ck)
    print(f"\nsweep: {len(rows)} instances checked; traced / predicted launches: %d / %d" % _cross_check(ck, prof))
    for case, s_, (_, _, st, _) in zip(WGRAD_CASES, splits, ck.records[len(conv_cases):]):
        print(f"wgrad {case}: {s_} split(s), worst bound ratio {st.ratio:.3g}, worst tile {st.tile:.3g} of its limit")


# ------------------------------------------------------------------------------------------------ planted defects
def test_checker_flags_defects_in_real_launch_output():
    """The CPU self-test's defects, planted in the output of real production-shaped launches after they ran."""
    from rave_b200 import ops
    conv = lambda: selftest.conv_args("cuda", B=32, Cin=192, Cout=192, Lin=2100)
    fm = lambda: selftest.fm_args("cuda", Bh=16, Cin=192, Cout=192, L=2100)
    wgrad = lambda: selftest.wgrad_args("cuda", B=32, L=2048, Cm=192, Cn=96)
    for make, op in ((conv, "conv1d_tc"), (fm, "conv1d_tc"), (wgrad, "conv1d_tc_wgrad")):
        clean = selftest.run_case(getattr(ops, op), op, make(), None)
        assert not clean.failures, clean.failures
    for muts, make, op in ((selftest.CONV_MUTATIONS, conv, "conv1d_tc"), (selftest.FM_MUTATIONS, fm, "conv1d_tc"),
                           (selftest.WGRAD_MUTATIONS, wgrad, "conv1d_tc_wgrad")):
        for mutation, (fn, kind) in muts.items():
            print(selftest.flagged_by(selftest.run_case(getattr(ops, op), op, make(), fn), kind, mutation))

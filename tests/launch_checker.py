"""Launch checker: every call the engine makes into rave_b200.ops, checked element by element against the float64
evaluation of its documented semantics (tests/tc_emulator.py under `compute(torch.float64)`).

`LaunchChecker.install(monkeypatch)` wraps the entry points listed in CHECKS.  Each wrapped call:
1. synchronises and snapshots its tensor arguments;
2. fills the region it must write with NaN (caller-provided outputs that alias no input and do not accumulate; buffers
   the entry point allocates itself come NaN-filled from torch's deterministic mode);
3. runs the real kernel;
4. evaluates the float64 reference from the snapshots, in batch chunks for big launches, and checks:
   - an elementwise bound that a correct kernel cannot exceed: with S the same operation on |operands| and n the products
     per output, |got - ref| <= (17 n / 16 + k) 2^-23 S + (k + 1) 2^-23 T, T the sum of the k epilogue terms'
     magnitudes (bias, residuals, feature-matching signs, the slope multiply).  The tensor cores are assumed to add each
     16-product step and the accumulator after aligning them to the largest exponent and truncating (2^-23 per product
     and per step, not round to nearest's 2^-24); that is an assumption, not a documented fact.  A bf16 output may
     differ by that bound plus one bf16 ulp of |ref| + bound;
   - per tile of an fp32 output (128 rows x 16 channels of a conv output, 128 x 16 of one weight-gradient tap): rel-L2
     <= (8 sqrt(n) + m) 2^-24, m the products one accumulator sums (n, or n / splits for a weight gradient): random
     rounding plus the bias of truncating accumulation, which grows with m (measured on the H100: 2.2x the sqrt(n) term
     alone for the v3 discriminator's 6512-row weight gradients, no split).  This catches a dropped k-block or split
     that stays under the worst-case bound and localises an error a whole-tensor rel-L2 averages away.  A tile whose
     reference cancels below |S| / sqrt(n) -- the size of a sum of n products of random sign, the scale of the partial
     sums a correct kernel rounds -- is measured against that.  Stat.tile_limit records the largest limit applied;
   - write coverage: no NaN left in the written region, and every element of each caller-provided output's whole
     allocation outside the written region keeps its bits (slack rows, the other phases' rows of a phase-fused launch,
     the real half of the gradient buffer under an fm_partner launch's fake-half view);
   - inputs: every tensor the call only reads keeps its bits (dact_src, its fm_partner rows, the operands);
   - exact equality where the operation is exact (layout converters, im2col, sign terms).
A failure names the workload, step, call index, arguments and the worst element."""
import inspect
import math

import torch

from tests import tc_emulator as emu

U23 = 2.0 ** -23
U24 = 2.0 ** -24
TILE_M, TILE_N = 128, 16
TILE_K = 8.0                      # per-tile limit: (TILE_K * sqrt(n) + products per accumulator) * 2^-24
CHUNK_ELEMS = 1 << 25             # float64 elements per reference chunk (~256 MB per tensor)


class LaunchError(AssertionError):
    pass


def ulp_bf16(x):
    """One bf16 ulp of |x| (8 significant bits); the smallest normal's ulp at 0."""
    a = x.abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def f64(t):
    return t.detach().to(torch.float64) if torch.is_tensor(t) else t


def unleaky(a, slope):
    return torch.where(a > 0, a, a / slope)


def overlaps(a, b):
    if a is None or b is None:
        return False
    a0, b0 = a.data_ptr(), b.data_ptr()
    return a0 < b0 + b.numel() * b.element_size() and b0 < a0 + a.numel() * a.element_size()


def conv_m_tiles(B, Lout):
    """(BB, BL) of the conv kernels' 128-row M tiles: BB batches x BL positions, BL a power of two <= max(Lout, 8)."""
    BL = 128
    while BL > Lout and BL > 8:
        BL //= 2
    return 128 // BL, BL


class Stat:
    """Worst elementwise bound ratio and worst tile rel-L2 (as a multiple of its limit) of one output."""

    def __init__(self):
        self.ratio, self.where, self.tile, self.tile_rel, self.tile_where = 0.0, None, 0.0, 0.0, None
        self.tile_limit = 0.0         # the largest per-tile rel-L2 limit applied

    def merge(self, other):
        if other.ratio > self.ratio:
            self.ratio, self.where = other.ratio, other.where
        if other.tile > self.tile:
            self.tile, self.tile_rel, self.tile_where = other.tile, other.tile_rel, other.tile_where
        self.tile_limit = max(self.tile_limit, other.tile_limit)


class LaunchChecker:
    def __init__(self, workload="", max_failures=8):
        self.workload, self.step, self.index = workload, "", 0
        self.failures, self.max_failures = [], max_failures
        self.records = []             # (op, family, Stat, args summary), one per checked call
        self.instance_fn = None       # (op, args) -> the kernel instance the call runs, or None
        self.instances = []           # instance_fn's answer for each record

    # ------------------------------------------------------------------ reporting
    def _ctx(self, op, args):
        desc = ", ".join(f"{k}={tuple(v.shape) if torch.is_tensor(v) else v}" for k, v in args.items()
                         if v is not None and not (isinstance(v, (list, tuple)) and len(str(v)) > 80))
        return f"[{self.workload} | {self.step} | call {self.index} {op}({desc})]"

    def fail(self, op, args, kind, msg):
        self.failures.append(f"{kind}: {self._ctx(op, args)} {msg}")
        if len(self.failures) >= self.max_failures:
            self.raise_if_failed()

    def raise_if_failed(self):
        if self.failures:
            msgs, self.failures = self.failures, []
            print("\n".join(msgs), flush=True)
            raise LaunchError(f"{len(msgs)} launch check failure(s):\n" + "\n".join(msgs))

    # ------------------------------------------------------------------ primitive checks
    def elementwise(self, op, args, name, got, ref, bound, bf16_out=False, stat=None, index_of=None):
        """|got - ref| <= bound (+ one bf16 ulp of |ref| + bound for a bf16 output); NaN in got = a missed store."""
        got, ref = f64(got), f64(ref)
        nan = torch.isnan(got)
        if bool(nan.any()):
            i = int(nan.reshape(-1).nonzero()[0])
            self.fail(op, args, "coverage", f"{name}: {int(nan.sum())} element(s) never written, first at "
                      f"{self._unravel(got.shape, i, index_of)}")
            got = torch.where(nan, torch.full_like(got, float("inf")), got)
        allow = bound + (ulp_bf16(ref.abs() + bound) if bf16_out else 0.0)
        err = (got - ref).abs()
        ratio = torch.where(allow > 0, err / allow.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
        worst = int(ratio.reshape(-1).argmax()) if ratio.numel() else 0
        r = float(ratio.reshape(-1)[worst]) if ratio.numel() else 0.0
        if stat is not None and r > stat.ratio:
            stat.ratio, stat.where = r, f"{name}{self._unravel(got.shape, worst, index_of)}"
        if not r <= 1.0:
            at = self._unravel(got.shape, worst, index_of)
            self.fail(op, args, "bound", f"{name}: {int((ratio > 1).sum())} element(s) over the bound; worst at {at}: "
                      f"got {float(got.reshape(-1)[worst]):.9g} ref {float(ref.reshape(-1)[worst]):.9g} allowed "
                      f"{float(allow.reshape(-1)[worst]) if torch.is_tensor(allow) else allow:.3g} ({r:.3g}x)")
        return r

    def exact(self, op, args, name, got, ref):
        g, r = f64(got), f64(ref)
        bad = ~((g == r) | (torch.isnan(g) & torch.isnan(r)))
        if bool(bad.any()):
            i = int(bad.reshape(-1).nonzero()[0])
            self.fail(op, args, "exact", f"{name}: {int(bad.sum())} element(s) differ, first at "
                      f"{self._unravel(g.shape, i)}: got {float(g.reshape(-1)[i])} ref {float(r.reshape(-1)[i])}")

    def tiles(self, op, args, name, got, ref, S, n, rows_of_tile, stat=None, n_acc=None):
        """Per-tile rel-L2 of [T, rows, C] grouped into tiles: rows_of_tile(got) -> [tiles, 128-row group, C]."""
        g, r, s = (rows_of_tile(f64(t)) for t in (got, ref, S))
        nt, m, C = g.shape
        ct = -(-C // TILE_N)
        pad = ct * TILE_N - C
        if pad:
            g, r, s = (torch.nn.functional.pad(t, (0, pad)) for t in (g, r, s))
        shape = (nt, m, ct, TILE_N)
        e2 = (g - r).reshape(shape).square().sum((1, 3))
        r2 = r.reshape(shape).square().sum((1, 3))
        s2 = s.reshape(shape).square().sum((1, 3))
        den = torch.maximum(r2, s2 / max(n, 1)).sqrt()
        rel = torch.where(den > 0, e2.sqrt() / den.clamp_min(1e-300), torch.where(e2 > 0, math.inf, 0.0))
        limit = (TILE_K * math.sqrt(max(n, 1)) + (n if n_acc is None else n_acc)) * U24
        q = rel / limit
        i = int(q.reshape(-1).argmax())
        worst = float(q.reshape(-1)[i])
        where = f"{name} tile (m {i // ct}, n {i % ct})"
        if stat is not None:
            stat.tile_limit = max(stat.tile_limit, limit)
        if stat is not None and worst > stat.tile:
            stat.tile, stat.tile_rel, stat.tile_where = worst, float(rel.reshape(-1)[i]), where
        if not worst <= 1.0:
            self.fail(op, args, "tile", f"{int((q > 1).sum())} tile(s) over rel-L2 {limit:.3g}; worst {where}: "
                      f"rel-L2 {float(rel.reshape(-1)[i]):.3g}")

    def mark_written(self, t, written_mask):
        """Record the elements of the caller's output view t (written_mask, t's shape) that the call may write."""
        entry = self._stores.get(_storage_key(t))
        if entry is not None:
            entry[2].as_strided(t.shape, t.stride(), t.storage_offset())[written_mask] = True
            entry[3].add(id(t))

    def _check_storage(self, op, args, snap):
        """Every element of an output's whole allocation outside the written region keeps its bits: slack rows, the
        other phases' rows, and whatever shares the allocation beyond the view (the real half under fm_partner)."""
        for key, (view, before, mask, marked) in self._stores.items():
            for k in OUTPUTS.get(op, ()):
                t = args.get(k)
                if torch.is_tensor(t) and _storage_key(t) == key and id(t) not in marked:
                    mask.as_strided(t.shape, t.stride(), t.storage_offset()).fill_(True)    # accumulator: the view
            bad = (_bits(view) != _bits(before)) & ~mask
            if bool(bad.any()):
                i = int(bad.nonzero()[0])
                self.fail(op, args, "outside", f"{int(bad.sum())} element(s) of an output's allocation outside the "
                          f"written region changed, first at storage element {i}")

    def _check_inputs(self, op, args, snap):
        """Every input the call only reads keeps its bits (those sharing memory with an output are covered above)."""
        outs = [args[k] for k in OUTPUTS.get(op, ()) if torch.is_tensor(args.get(k))]
        for k, v in args.items():
            if not torch.is_tensor(v) or k in OUTPUTS.get(op, ()) or any(overlaps(v, o) for o in outs):
                continue
            if not torch.equal(_bytes(v), _bytes(snap[k])):
                self.fail(op, args, "input", f"input {k} was modified by the call")

    @staticmethod
    def _unravel(shape, i, index_of=None):
        idx = []
        for d in reversed(shape):
            idx.append(i % d)
            i //= d
        idx = tuple(reversed(idx))
        return index_of(idx) if index_of else idx

    # ------------------------------------------------------------------ installation
    def install(self, monkeypatch):
        from rave_b200 import ops
        for name in CHECKS:
            monkeypatch.setattr(ops, name, self._wrap(name, getattr(ops, name)))

    def _wrap(self, name, orig):
        sig = inspect.signature(orig)

        def wrapped(*a, **kw):
            ba = sig.bind(*a, **kw)
            ba.apply_defaults()
            return self.checked_call(name, orig, dict(ba.arguments))
        return wrapped

    def checked_call(self, name, fn, args, mutate=None):
        """Snapshot, NaN-fill, run fn(**args), then check its result.  mutate(args, out), if given, edits the outputs
        after the call and before the check (how the checker's own tests plant defects)."""
        sync = torch.cuda.synchronize if any(torch.is_tensor(v) and v.is_cuda for v in args.values()) else (lambda: None)
        sync()
        snap = {k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in args.items()}
        self._stores = {}             # whole allocations of the caller's outputs: [view, snapshot, written mask, marked]
        for k in OUTPUTS.get(name, ()):
            t = args.get(k)
            if torch.is_tensor(t) and _storage_key(t) not in self._stores:
                view = _storage_view(t)
                self._stores[_storage_key(t)] = [view, view.clone(), torch.zeros(view.shape, dtype=torch.bool,
                                                                                 device=view.device), set()]
        fill = PREPARE.get(name)
        if fill is not None:
            fill(args)
        with nan_fill():
            out = fn(**args)
        sync()
        if mutate is not None:
            mutate(args, out)
        CHECKS[name](self, name, args, snap, out)
        self.instances.append(self.instance_fn(name, args) if self.instance_fn else None)
        self._check_storage(name, args, snap)
        self._check_inputs(name, args, snap)
        self.index += 1
        return out


def _storage_key(t):
    return (t.device, t.untyped_storage().data_ptr(), t.dtype)


def _storage_view(t):
    """The whole allocation behind t as a flat tensor of t's dtype."""
    st = t.untyped_storage()
    return torch.empty(0, dtype=t.dtype, device=t.device).set_(st, 0, (st.nbytes() // t.element_size(),), (1,))


def _bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _bytes(t):
    return t.detach().reshape(-1).contiguous().view(torch.uint8)


class nan_fill:
    """torch.empty inside the block returns NaN-filled floating tensors (torch's deterministic fill)."""

    def __enter__(self):
        import torch.utils.deterministic as det
        self.saved = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled(),
                      det.fill_uninitialized_memory)
        torch.use_deterministic_algorithms(True, warn_only=True)
        det.fill_uninitialized_memory = True

    def __exit__(self, *exc):
        import torch.utils.deterministic as det
        torch.use_deterministic_algorithms(self.saved[0], warn_only=self.saved[1])
        det.fill_uninitialized_memory = self.saved[2]


def _batch_chunks(B, per_batch, pair_halves=False, align=16):
    """Index tensors of batch chunks with at most CHUNK_ELEMS reference elements each (multiples of `align` batches, the
    conv kernels' largest tile batch group).  pair_halves: batch b and b + B/2 stay in one chunk ([real; fake])."""
    h = B // 2 if pair_halves else B
    step = max(align, (CHUNK_ELEMS // max(per_batch * (2 if pair_halves else 1), 1)) // align * align)
    for i in range(0, h, step):
        j = min(h, i + step)
        idx = torch.arange(i, j)
        yield torch.cat([idx, idx + h]) if pair_halves else idx


# ---------------------------------------------------------------------------------------------- conv1d_tc
def _conv_rows(args):
    xa, Lin = args["xa_cl"], args["Lin"]
    K = args["wt"].shape[0] // (2 if args["x3"] else 1)
    Lin = xa.shape[1] if Lin is None else Lin
    Lout = args["Lout"]
    if Lout is None:
        from rave_b200.ops import conv_out_len
        Lout = conv_out_len(Lin, K, args["stride"], args["dil"], args["pad"][0], args["pad"][1])
    return Lin, Lout, K


def _prep_conv(args):
    """NaN into the rows a conv1d_tc launch writes, in the caller's outputs that alias no input."""
    Lin, Lout, K = _conv_rows(args)
    idx = emu.out_row_index(Lout, args["out_row_stride"], args["out_row_offset"], args["xa_cl"].device)
    ins = [args[k] for k in ("xa_cl", "wt", "bias", "res_cl", "res_bf16", "dact_src", "res_act", "fm_d", "fm_partner")]
    for k in ("out_f32", "out_act"):
        t = args[k]
        if t is not None and not any(overlaps(t, i) for i in ins):
            t[:, idx] = float("nan")


def check_conv1d_tc(ck, op, args, snap, out):
    out_f32, out_act = out
    Lin, Lout, K = _conv_rows(args)
    x3 = args["x3"]
    B, _, Cin = snap["xa_cl"].shape
    Cin //= 2 if x3 else 1
    Cout = snap["wt"].shape[1]
    n = K * Cin * (3 if x3 else 1)
    slope = args["slope"]
    dev = snap["xa_cl"].device
    idx = emu.out_row_index(Lout, args["out_row_stride"], args["out_row_offset"], dev)
    fm_pair = args["fm_d"] is not None and args["fm_partner"] is None
    BB, BL = conv_m_tiles(B, Lout)
    stats = {}
    # the caller's outputs: snapshots (bytes outside the written rows must survive) and the written-row mask
    targets = [("out_f32", out_f32, False), ("out_act", out_act, True)]
    for key, t, _ in targets:
        if t is None or args[key] is None:
            continue
        wm = torch.zeros(t.shape, dtype=torch.bool, device=t.device)
        wm[:, idx] = True
        ck.mark_written(t, wm)
    k_terms = sum(args[k] is not None for k in ("bias", "res_cl", "res_bf16", "res_act")) + \
        (2 if args["fm_d"] is not None else 0) + (1 if args["dact_src"] is not None else 0) + (1 if args["act"] == 1 else 0)
    per_batch = Lout * Cout * (2 if x3 else 1)
    for sel in _batch_chunks(B, per_batch, pair_halves=fm_pair, align=BB):
        sel = sel.to(dev)
        a = dict(snap)
        for k in ("xa_cl", "res_cl", "res_bf16", "dact_src", "res_act", "fm_partner"):
            if snap[k] is not None:
                a[k] = snap[k].index_select(0, sel)
        Bc = len(sel)
        rows = out_f32.shape[1] if out_f32 is not None else out_act.shape[1]
        r32 = torch.zeros(Bc, rows, Cout, dtype=torch.float64, device=dev) if out_f32 is not None else None
        ract = torch.zeros(Bc, rows, out_act.shape[2], dtype=torch.float64, device=dev) if out_act is not None else None
        with emu.compute(torch.float64):
            kw = {k: a[k] for k in ("bias", "res_cl", "stride", "dil", "pad", "act", "slope", "out_rows",
                                    "out_row_stride", "out_row_offset", "Lout", "res_bf16", "dact_src", "Lin", "res_act",
                                    "res_slope", "fm_d", "fm_partner", "x3", "act_cs")}
            kw["bias"] = f64(kw["bias"])
            kw["res_cl"] = f64(kw["res_cl"])
            kw["Lout"] = Lout
            emu.conv1d_tc(a["xa_cl"], a["wt"], want_f32=False, want_act=False, out_f32=r32, out_act=ract, **kw)
            # S: the products on |operands|
            Sv, _ = emu.conv1d_tc(a["xa_cl"].abs(), a["wt"].abs(), None, None, args["stride"], args["dil"], args["pad"],
                                  0, slope, want_f32=True, want_act=False, Lout=Lout, Lin=Lin, x3=x3,
                                  out_rows=Lout) if not x3 else _x3_abs(a, args, Lout, Lin)
        T = torch.zeros_like(Sv)
        if args["bias"] is not None:
            T += f64(args["bias"]).abs()
        for k in ("res_cl", "res_bf16"):
            if args[k] is not None:
                T += f64(a[k][:, idx]).abs()
        if args["res_act"] is not None:
            ra = f64(a["res_act"][:, idx])
            ra = ra[..., :Cout] + ra[..., Cout:] if x3 else ra
            T += unleaky(ra, args["res_slope"]).abs()
        if args["fm_d"] is not None:
            T += f64(args["fm_d"]).abs().sum()
        bound = (n * 17 / 16 + k_terms) * U23 * Sv + (k_terms + 1) * U23 * T
        cbound = bound  # per channel layout of out_f32
        st = stats.setdefault("f32", Stat())

        def tile_rows(t):            # [Bc, Lout, C] -> [tiles, 128, C] in the kernel's M-tile order (ragged tiles padded)
            Bp, Lp = -(-t.shape[0] // BB) * BB, -(-t.shape[1] // BL) * BL
            t = torch.nn.functional.pad(t, (0, 0, 0, Lp - t.shape[1], 0, 0))
            t = torch.cat([t, t.new_zeros(Bp - t.shape[0], *t.shape[1:])]) if Bp > t.shape[0] else t
            C = t.shape[2]
            return t.reshape(Bp // BB, BB, Lp // BL, BL, C).permute(0, 2, 1, 3, 4).reshape(-1, BB * BL, C)

        def index_of(ix, sel=sel):
            return (int(sel[ix[0]]),) + tuple(ix[1:])
        if out_f32 is not None:
            got = out_f32.index_select(0, sel)[:, idx]
            ck.elementwise(op, args, "out_f32", got, r32[:, idx], cbound, stat=st, index_of=index_of)
            ck.tiles(op, args, "out_f32", got, r32[:, idx], Sv, n, tile_rows, stat=st)
        if out_act is not None:
            got = f64(out_act.index_select(0, sel)[:, idx])
            ref = ract[:, idx]
            sa = stats.setdefault("act", Stat())
            if x3:                   # compare hi + lo: the split value carries ~16 significant bits
                cs = args["act_cs"] or Cout
                q = Cout // cs
                g5, r5 = got.reshape(Bc, Lout, q, 2, cs), ref.reshape(Bc, Lout, q, 2, cs)
                gs, rs = (g5.sum(3)).reshape(Bc, Lout, Cout), (r5.sum(3)).reshape(Bc, Lout, Cout)
                b = bound + 2.0 ** -15 * (rs.abs() + bound)
                ck.elementwise(op, args, "out_act(hi+lo)", gs, rs, b, stat=sa, index_of=index_of)
            else:
                ck.elementwise(op, args, "out_act", got, ref, bound, bf16_out=True, stat=sa, index_of=index_of)
    fam = "conv_x3" if x3 else ("conv_dgrad" if args["dact_src"] is not None else "conv_fwd")
    total = Stat()
    for s in stats.values():
        total.merge(s)
    ck.records.append((op, fam, total, (B, Cin, Cout, Lout, K)))


def _x3_abs(a, args, Lout, Lin):
    xa, wt = a["xa_cl"], a["wt"]
    Cin, K = xa.shape[2] // 2, wt.shape[0] // 2
    hi, lo = xa[..., :Cin].abs().contiguous(), xa[..., Cin:].abs().contiguous()
    whi, wlo = wt[:K].abs(), wt[K:].abs()

    def run(x, w):
        return emu.conv1d_tc(x, w, None, None, args["stride"], args["dil"], args["pad"], 0, args["slope"], want_f32=True,
                             want_act=False, Lout=Lout, Lin=Lin)[0]
    return run(hi, whi) + run(lo, whi) + run(hi, wlo), None


# ---------------------------------------------------------------------------------------------- dilated_unit_tc
def _prep_unit(args):
    B, pitch, C = args["xa_cl"].shape
    L = pitch if args["L"] is None else args["L"]
    for k in ("out_f32", "out_act"):
        t = args[k]
        if t is not None and not overlaps(t, args["xa_cl"]):
            t[:, :L] = float("nan")


def check_unit(ck, op, args, snap, out):
    a1, out_f32, out_act = out
    xa = snap["xa_cl"]
    B, pitch, C = xa.shape
    L = pitch if args["L"] is None else args["L"]
    dil, pad_l = args["dil"], args["pad_l"]
    n1, n2 = 3 * C, C
    BB, BL = conv_m_tiles(B, L)
    st = Stat()
    for key in ("out_f32", "out_act"):
        if snap.get(key) is not None:
            wm = torch.zeros(snap[key].shape, dtype=torch.bool, device=xa.device)
            wm[:, :L] = True
            ck.mark_written(args[key], wm)

    def tile_rows(t):
        Bp, Lp = -(-t.shape[0] // BB) * BB, -(-t.shape[1] // BL) * BL
        t = torch.nn.functional.pad(t, (0, 0, 0, Lp - t.shape[1], 0, 0))
        t = torch.cat([t, t.new_zeros(Bp - t.shape[0], *t.shape[1:])]) if Bp > t.shape[0] else t
        return t.reshape(Bp // BB, BB, Lp // BL, BL, t.shape[2]).permute(0, 2, 1, 3, 4).reshape(-1, BB * BL, t.shape[2])
    for sel in _batch_chunks(B, pitch * C, align=BB):
        sel = sel.to(xa.device)
        x = xa.index_select(0, sel)
        with emu.compute(torch.float64):
            r1 = emu.unit_stage1(x, snap["w3t"], dil, pad_l, args["slope_mid"], L,
                                 out_act=torch.zeros(x.shape, dtype=torch.float64, device=x.device))
            S1 = emu.conv1d_tc(x.abs(), snap["w3t"].abs(), None, None, 1, dil, (pad_l, 2 * dil - pad_l), 0, 0.2,
                               want_f32=True, Lout=L, Lin=L)[0]
            b1 = (n1 * 17 / 16 + 1) * U23 * S1
            if a1 is not None:        # stage 2 from the kernel's own intermediate: the tight bound holds
                g1 = a1.index_select(0, sel)
                ck.elementwise(op, args, "a1", g1[:, :L], r1[:, :L], b1, bf16_out=True, stat=st)
                if pitch > L:
                    ck.exact(op, args, "a1 slack rows", g1[:, L:], torch.zeros_like(g1[:, L:]))
                mid, e1 = g1, 0.0
            else:                     # the kernel's bf16 intermediate may differ by b1 + one ulp from the reference's
                mid, e1 = r1.to(torch.bfloat16), b1 + ulp_bf16(S1 + b1)
            r32 = torch.zeros(x.shape, dtype=torch.float64, device=x.device) if out_f32 is not None else None
            ra = torch.zeros(x.shape, dtype=torch.float64, device=x.device) if out_act is not None else None
            emu.unit_stage2(mid, x, snap["w1t"], args["slope_in"], args["act_out"], args["slope_out"], L, r32, ra)
            S2 = emu.conv1d_tc(f64(mid).abs().to(torch.bfloat16) if a1 is not None else (S1 + e1).to(torch.float32).to(
                torch.bfloat16), snap["w1t"].abs(), None, None, want_f32=True, Lout=L, Lin=L)[0]
            if a1 is None:
                S2 = S2 * (1 + 2.0 ** -7)            # the bf16 rounding of the magnitudes above
            T = unleaky(f64(x[:, :L]), args["slope_in"]).abs()
            bound = (n2 * 17 / 16 + 2) * U23 * S2 + 2 * U23 * T
            if a1 is None:                           # + what the intermediate's difference carries through conv1x1
                bound = bound + emu.conv1d_tc(e1, snap["w1t"].abs(), None, None, want_f32=True, Lout=L, Lin=L)[0]
        if out_f32 is not None:
            g = out_f32.index_select(0, sel)[:, :L]
            ck.elementwise(op, args, "out_f32", g, r32[:, :L], bound, stat=st)
            if a1 is not None:
                ck.tiles(op, args, "out_f32", g, r32[:, :L], S2, n2, tile_rows, stat=st)
        if out_act is not None:
            g = out_act.index_select(0, sel)[:, :L]
            ck.elementwise(op, args, "out_act", g, ra[:, :L], bound, bf16_out=True, stat=st)
    ck.records.append((op, "unit", st, (B, C, L, dil)))


# ---------------------------------------------------------------------------------------------- conv1d_tc_wgrad
def check_wgrad(ck, op, args, snap, dwt):
    P, Q = snap["P_cl"], snap["Q_cl"]
    B, p_pitch, Cm = P.shape
    Cn = Q.shape[2]
    K = args["K"]
    Lp = p_pitch if args["Lp"] is None else args["Lp"]
    st = Stat()
    if bool(torch.isnan(dwt).any()):
        nz = torch.isnan(dwt).reshape(dwt.shape[0], -1).any(1).nonzero().reshape(-1).tolist()
        ck.fail(op, args, "coverage", f"dwt: split slice(s) {nz} of {dwt.shape[0]} left unwritten")
    ref = torch.zeros(K, Cm, Cn, dtype=torch.float64, device=P.device)
    S = torch.zeros_like(ref)
    db = f64(snap["dbias"]).clone() if snap["dbias"] is not None else None
    dbS = torch.zeros(Cm, dtype=torch.float64, device=P.device)
    kw = dict(stride=args["stride"], dil=args["dil"], pad_l=args["pad_l"], Lp=args["Lp"], Lq=args["Lq"])
    for sel in _batch_chunks(B, p_pitch * max(Cm, Cn), align=1):
        sel = sel.to(P.device)
        p, q = P.index_select(0, sel), Q.index_select(0, sel)
        with emu.compute(torch.float64):
            ref += emu.conv1d_tc_wgrad(p, q, K, dbias=db, **kw).sum(0)
            S += emu.conv1d_tc_wgrad(p.abs(), q.abs(), K, dbias=dbS if db is not None else None, **kw).sum(0)
    n = B * Lp
    got = f64(dwt).sum(0)
    ck.elementwise(op, args, "dwt (slices summed)", got, ref, (n * 17 / 16 + 1) * U23 * S, stat=st)
    ck.tiles(op, args, "dwt", got, ref, S, n, lambda t: _wg_tiles(t), stat=st, n_acc=-(-n // dwt.shape[0]))
    if db is not None:
        ck.elementwise(op, args, "dbias", args["dbias"], db, (n + dwt.shape[0] + 2) * U23 * (dbS + f64(snap["dbias"]).abs()),
                       stat=st)
    ck.records.append((op, "wgrad", st, (B, Cm, Cn, Lp, K, dwt.shape[0])))


def _wg_tiles(t):
    """[K, Cm, Cn] -> [K * m-tiles, 128, Cn]: one tap's 128 output rows per tile."""
    K, Cm, Cn = t.shape
    Mp = -(-Cm // TILE_M) * TILE_M
    t = torch.nn.functional.pad(t, (0, 0, 0, Mp - Cm))
    return t.reshape(K * (Mp // TILE_M), TILE_M, Cn)


# ---------------------------------------------------------------------------------------------- elementwise kernels
def _f64args(snap, keys):
    return [f64(snap[k]) if torch.is_tensor(snap[k]) and snap[k].dtype == torch.float32 else snap[k] for k in keys]


def check_snake_fwd(ck, op, args, snap, out):
    h, al = f64(snap["h_cl"]), f64(snap["alpha"]).reshape(-1)
    with emu.compute(torch.float64):
        ref = emu.snake_cl_fwd(snap["h_cl"], al)
    # fp32 evaluation: sin's argument carries |alpha h| 2^-24, so sin^2 / alpha carries ~2 |sin| |h| 2^-24
    sn = torch.sin(al * h)
    bound = 16 * U23 * (h.abs() + sn.square() / (al + 1e-9).abs() + 2 * sn.abs() * h.abs())
    st = Stat()
    ck.elementwise(op, args, "a", out, f64(ref), bound, bf16_out=True, stat=st)
    ck.records.append((op, "snake", st, tuple(h.shape)))


def check_snake_bwd(ck, op, args, snap, out):
    gh, dal = out
    h, g, al = f64(snap["h_cl"]), f64(snap["ga_cl"]), f64(snap["alpha"]).reshape(-1)
    add = f64(snap["add"]) if snap["add"] is not None else None
    with emu.compute(torch.float64):
        rgh, rdal = emu.snake_cl_bwd(snap["ga_cl"], snap["h_cl"], al, snap["add"], args["want_dalpha"])
    ae = (al + 1e-9).abs()
    st = Stat()
    mag = g.abs() * (2 + 4 * (al * h).abs()) + (add.abs() if add is not None else 0)
    ck.elementwise(op, args, "g_h", gh, f64(rgh), 16 * U23 * mag, bf16_out=True, stat=st)
    if dal is not None:
        terms = (g.abs() * (h.abs() * (1 + 4 * (al * h).abs()) / ae + torch.sin(al * h) ** 2 / ae.square())
                 ).reshape(-1, h.shape[-1])
        n = terms.shape[0]
        ck.elementwise(op, args, "dalpha", dal, rdal, (n + 16) * U23 * terms.sum(0), stat=st)
    ck.records.append((op, "snake", st, tuple(h.shape)))


def check_ncl_to_cl(ck, op, args, snap, out):
    yb, yf = out
    x = snap["x"]
    st = Stat()
    if yf is not None:
        ck.exact(op, args, "f32", yf, x.permute(0, 2, 1))
    if yb is not None:
        with emu.compute(torch.float64):
            rb, _ = emu.ncl_to_cl(f64(x), args["act"], args["slope"], want_bf16=True)
        if args["act"] == 0:
            ck.exact(op, args, "bf16", yb, x.permute(0, 2, 1).to(torch.bfloat16))
        else:                         # LeakyReLU in fp32, then bf16
            ck.elementwise(op, args, "bf16", yb, f64(rb), U23 * f64(x).abs().permute(0, 2, 1), bf16_out=True, stat=st)
    ck.records.append((op, "layout", st, tuple(x.shape)))


def check_ncl_to_cl_x3(ck, op, args, snap, out):
    x = snap["x"].float()
    xt = x.permute(0, 2, 1)
    hi = xt.to(torch.bfloat16)
    lo = (xt - hi.float()).to(torch.bfloat16)
    ck.exact(op, args, "[hi | lo]", out, torch.cat([hi, lo], -1))
    ck.records.append((op, "layout", Stat(), tuple(x.shape)))


def check_cl_to_ncl(ck, op, args, snap, out):
    ck.exact(op, args, "ncl", out, snap["x_cl"].permute(0, 2, 1))
    ck.records.append((op, "layout", Stat(), tuple(snap["x_cl"].shape)))


# ---------------------------------------------------------------------------------------------- first-layer kernels
def check_im2col(ck, op, args, snap, out):
    keys = ("Lin", "Lout", "out_pitch", "K", "stride", "pad_l", "period", "pool")
    src = f64(snap["src"])
    with emu.compute(torch.float64):
        ref = (emu.im2col_c1 if op == "im2col_c1" else emu.im2col_cin)(src, *[args[k] for k in keys])
    st = Stat()
    if args["pool"] == 1:
        ck.exact(op, args, "X", out, ref)
    else:                             # average pooling: a mean of `pool` fp32 values, then bf16
        with emu.compute(torch.float64):
            S = (emu.im2col_c1 if op == "im2col_c1" else emu.im2col_cin)(src.abs(), *[args[k] for k in keys])
        ck.elementwise(op, args, "X", out, f64(ref), (args["pool"] + 2) * U23 * f64(S), bf16_out=True, stat=st)
    ck.records.append((op, "first_layer", st, tuple(src.shape)))


def check_gather(ck, op, args, snap, out):
    keys = ("src_shape", "Lin", "Lout", "K", "stride", "pad_l", "period", "pool", "batch0")
    P = f64(snap["P_cl"])
    fn = emu.gather_c1 if op == "gather_c1" else emu.gather_cin
    with emu.compute(torch.float64):
        ref = fn(P, *[args[k] for k in keys])
        S = fn(P.abs(), *[args[k] for k in keys])
    n = args["K"] * args["pool"] + 2
    st = Stat()
    ck.elementwise(op, args, "dsrc", out, ref, n * U23 * S, stat=st)
    ck.records.append((op, "first_layer", st, tuple(P.shape)))


def check_c1_fwd(ck, op, args, snap, out):
    out_f32, out_act = out
    x, w, bias = _f64args(snap, ("x_rows", "w", "bias"))
    Lout = args["Lout"]
    K = w.numel() // w.shape[0]
    rows = (out_f32 if out_f32 is not None else out_act).shape[1]
    R, Cout = x.shape[0], w.shape[0]
    r32 = torch.zeros(R, rows, Cout, dtype=torch.float64, device=x.device)
    ra = torch.zeros_like(r32)
    S = torch.zeros_like(r32)
    with emu.compute(torch.float64):
        emu.conv1d_c1(x, w, bias, args["Lin"], args["stride"], args["pad"], args["act"], args["slope"], r32, ra, Lout)
        emu.conv1d_c1(x.abs(), w.abs(), bias.abs() if bias is not None else None, args["Lin"], args["stride"],
                      args["pad"], 0, 0.2, S, None, Lout)
    bound = (K + 3) * U23 * S
    st = Stat()
    for key, t, r, bf in (("out_f32", out_f32, r32, False), ("out_act", out_act, ra, True)):
        if t is None:
            continue
        ck.elementwise(op, args, key, t[:, :Lout], r[:, :Lout], bound[:, :Lout], bf16_out=bf, stat=st)
        if snap.get(key) is not None:
            wm = torch.zeros(t.shape, dtype=torch.bool, device=t.device)
            wm[:, :Lout] = True
            ck.mark_written(t, wm)
    ck.records.append((op, "first_layer", st, (R, Cout, Lout, K)))


def check_c1_wgrad(ck, op, args, snap, dwt):
    g, x = snap["g_cl"], f64(snap["x_rows"])
    keys = ("Cout", "K", "Lin", "Lout", "stride", "pad_l")
    with emu.compute(torch.float64):
        ref = emu.conv1d_c1_wgrad(g, x, *[args[k] for k in keys]).sum(0)
        S = emu.conv1d_c1_wgrad(g.abs(), x.abs(), *[args[k] for k in keys]).sum(0)
    n = g.shape[0] * args["Lout"]
    st = Stat()
    if bool(torch.isnan(dwt).any()):
        ck.fail(op, args, "coverage", "dwt: slices left unwritten")
    ck.elementwise(op, args, "dwt (slices summed)", f64(dwt).sum(0), ref, (n + dwt.shape[0]) * U23 * S, stat=st)
    ck.records.append((op, "first_layer", st, tuple(g.shape)))


def check_c1_dgrad(ck, op, args, snap, dx):
    g, w = snap["g_cl"], f64(snap["w"])
    keys = ("x_pitch", "Lin", "Lout", "stride", "pad_l")
    with emu.compute(torch.float64):
        ref = emu.conv1d_c1_dgrad(g, w, *[args[k] for k in keys])
        S = emu.conv1d_c1_dgrad(g.abs(), w.abs(), *[args[k] for k in keys])
    n = w.shape[0] * (w.numel() // w.shape[0])
    st = Stat()
    ck.elementwise(op, args, "dx", dx, ref, (n + 1) * U23 * S, stat=st)
    ck.records.append((op, "first_layer", st, tuple(g.shape)))


def check_colsum(ck, op, args, snap, out):
    g = snap["g_cl"]
    L, C = args["L"], args["C"]
    with emu.compute(torch.float64):
        ref = emu.colsum_bf16(g, L, C)
        S = emu.colsum_bf16(g.abs(), L, C)
    st = Stat()
    ck.elementwise(op, args, "colsum", out, ref, (g.shape[0] * L + 2) * U23 * S, stat=st)
    ck.records.append((op, "reduction", st, tuple(g.shape)))


# ---------------------------------------------------------------------------------------------- loss taps
def check_fm_stats(ck, op, args, snap, out):
    a = snap["a_cl"]
    L, slope = args["L"], args["slope"]
    ref = f64(snap["stats_row"]).clone()
    with emu.compute(torch.float64):
        emu.fm_stats(a, ref, L, slope)
        h = unleaky(f64(a[:, :L]), slope).abs()
    hh = h.shape[0] // 2
    S = torch.stack([(h[:hh] + h[hh:]).sum(), h[:hh].sum()]) + f64(snap["stats_row"]).abs()
    n = hh * L * a.shape[2]
    st = Stat()
    ck.elementwise(op, args, "stats", args["stats_row"], ref, (n + 3) * U23 * S, stat=st)
    ck.records.append((op, "reduction", st, tuple(a.shape)))


def check_fm_grad(ck, op, args, snap, g):
    a = snap["a_cl"]
    with emu.compute(torch.float64):
        ref = emu.fm_grad(a, f64(snap["dstats_row"]), args["L"], args["slope"])
    # sign terms are exact; d0 * s + d1 * s' is formed in fp32 and rounded to bf16
    d = f64(snap["dstats_row"]).abs()
    st = Stat()
    ck.elementwise(op, args, "g", g, f64(ref), 2 * U23 * (d[0] + d[1]) * torch.ones_like(f64(g)), bf16_out=True,
                   stat=st)
    ck.records.append((op, "reduction", st, tuple(a.shape)))


def check_score_stats(ck, op, args, snap, out):
    s = snap["score_cl"]
    L = args["L"]
    ref = f64(snap["stats6"]).clone()
    with emu.compute(torch.float64):
        emu.score_stats(s, ref, L)
    v = f64(s[:, :L, 0])
    h = v.shape[0] // 2
    sr, sf = v[:h].abs(), v[h:].abs()
    S = torch.stack([(sr + sf).sum(), sr.sum(), (1 + sr).sum(), (1 + sf).sum(), sr.sum(), sf.sum()])
    S = S.reshape(ref.shape) + f64(snap["stats6"]).abs()
    st = Stat()
    ck.elementwise(op, args, "stats6", args["stats6"], ref, (h * L + 3) * U23 * S, stat=st)
    ck.records.append((op, "reduction", st, tuple(s.shape)))


def check_score_grad(ck, op, args, snap, g):
    with emu.compute(torch.float64):
        ref = emu.score_grad(snap["score_cl"], snap["dstats6"], args["L"])
    d = f64(snap["dstats6"]).abs().reshape(-1)
    st = Stat()
    # reference rounded to the gradient dtype from fp64; the kernel rounds its fp32 sum of <= 4 terms
    ck.elementwise(op, args, "g", g, f64(ref), 4 * U23 * d.sum() * torch.ones_like(f64(g)), bf16_out=True, stat=st)
    ck.records.append((op, "reduction", st, tuple(snap["score_cl"].shape)))


# ---------------------------------------------------------------------------------------------- weights
def check_weight_prep(ck, op, args, snap, out):
    items = snap["items"]
    x3 = args["x3"]
    st = Stat()
    for i, (it, got) in enumerate(zip(items, out)):
        v, g = f64(it[0]), f64(it[1]) if it[1] is not None else None
        with emu.compute(torch.float64):
            saved = emu.OPERAND_DTYPE
            emu.OPERAND_DTYPE = torch.float64            # the unrounded weights; rounding is allowed for below
            try:
                norm, A, Bm = emu.weight_prep_tc(v, g, *it[2:])
            finally:
                emu.OPERAND_DTYPE = saved
        m = v.reshape(v.shape[0], -1).shape[1]
        rel = (m + 8) * U23                              # norm: a sum of m squares, a sqrt, a divide, a multiply
        if norm is not None:
            ck.elementwise(op, args, f"item {i} norm", got[0], norm, rel * norm.abs(), stat=st)
        for name, r, gt in (("A", A, got[1]), ("B", Bm, got[2])):
            if r is None:
                continue
            if x3:                   # [hi slabs | lo slabs]: hi + lo carries the weight to ~2^-16
                h = gt.shape[0] // 2
                gs = f64(gt[:h]) + f64(gt[h:])
                ck.elementwise(op, args, f"item {i} {name}(hi+lo)", gs, r, (rel + 2.0 ** -15) * r.abs(), stat=st)
            else:
                ck.elementwise(op, args, f"item {i} {name}", gt, r, rel * r.abs(), bf16_out=True, stat=st)
    ck.records.append((op, "weights", st, len(items)))


def check_weight_norm_bwd(ck, op, args, snap, out):
    st = Stat()
    for i, (it, (dv, dg)) in enumerate(zip(snap["items"], out)):
        dwt, v, g, norm = (f64(t) if t is not None else None for t in it[:4])
        extra = it[4] if len(it) > 4 else None
        with emu.compute(torch.float64):
            (rdv, rdg), = emu.weight_norm_bwd_multi([(dwt, v, g, norm) + ((extra,) if len(it) > 4 else ())])
            (adv, _), = emu.weight_norm_bwd_multi([(dwt.abs(), v.abs(), g.abs() if g is not None else None, norm)
                                                   + ((extra,) if len(it) > 4 else ())])
        S_dw = adv if g is None else None
        m = v.reshape(v.shape[0], -1).shape[1]
        n = dwt.shape[0] + m + 8
        if g is None:
            ck.elementwise(op, args, f"item {i} dv", dv, rdv, n * U23 * S_dw, stat=st)
            continue
        # |dv| <= |g|/||v|| (|dw| + |v| sum|dw v| / ||v||^2): the magnitudes of every term
        C0 = v.shape[0]
        v2 = v.reshape(C0, -1)
        with emu.compute(torch.float64):
            (adw, _), = emu.weight_norm_bwd_multi([(dwt.abs(), v, None, norm) + ((extra,) if len(it) > 4 else ())])
        adw2 = adw.reshape(C0, -1)
        dot = (adw2 * v2.abs()).sum(1, keepdim=True)
        gn = g.reshape(C0, 1).abs() / norm.reshape(C0, 1)
        Sdv = gn * (adw2 + v2.abs() * dot / norm.reshape(C0, 1) ** 2)
        ck.elementwise(op, args, f"item {i} dv", dv, rdv, n * U23 * Sdv.reshape(v.shape), stat=st)
        ck.elementwise(op, args, f"item {i} dg", dg, rdg, n * U23 * (dot / norm.reshape(C0, 1)).reshape(g.shape), stat=st)
    ck.records.append((op, "weights", st, len(snap["items"])))


CHECKS = {
    "conv1d_tc": check_conv1d_tc,
    "dilated_unit_tc": check_unit,
    "conv1d_tc_wgrad": check_wgrad,
    "snake_cl_fwd": check_snake_fwd,
    "snake_cl_bwd": check_snake_bwd,
    "conv1d_c1": check_c1_fwd,
    "conv1d_c1_wgrad": check_c1_wgrad,
    "conv1d_c1_dgrad": check_c1_dgrad,
    "im2col_c1": check_im2col,
    "im2col_cin": check_im2col,
    "gather_c1": check_gather,
    "gather_cin": check_gather,
    "colsum_bf16": check_colsum,
    "fm_stats": check_fm_stats,
    "fm_grad": check_fm_grad,
    "score_stats": check_score_stats,
    "score_grad": check_score_grad,
    "weight_prep_tc_multi": check_weight_prep,
    "weight_norm_bwd_multi": check_weight_norm_bwd,
    "ncl_to_cl": check_ncl_to_cl,
    "ncl_to_cl_x3": check_ncl_to_cl_x3,
    "cl_to_ncl": check_cl_to_ncl,
}

OUTPUTS = {                       # caller-provided outputs and accumulators of each entry point
    "conv1d_tc": ("out_f32", "out_act"),
    "dilated_unit_tc": ("out_f32", "out_act"),
    "conv1d_c1": ("out_f32", "out_act"),
    "conv1d_tc_wgrad": ("dbias",),
    "fm_stats": ("stats_row",),
    "score_stats": ("stats6",),
}

PREPARE = {
    "conv1d_tc": _prep_conv,
    "dilated_unit_tc": _prep_unit,
}

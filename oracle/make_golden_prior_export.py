"""TEST INFRASTRUCTURE -- generates the fixture of the exported model's `prior(temp)` (scripts/export.py TraceModel,
lines 411-466, at a `--streaming` export) by EXECUTING THE UNMODIFIED REFERENCE's prior modules (rave/prior/{core,model}.py
under oracle/make_golden_prior.load_reference_prior).  Writes a new file only:

    python -m oracle.make_golden_prior_export

  tests/golden/prior_export.pt   per case (D, B, the prior's seeded parameters): several consecutive calls of different
                                 lengths, each with its temperature input, uniforms, dither, classes and output latents

What runs the reference's code, in float64 except the decode:
  * Prior.forward: the cached convs' one-frame steps equal the dense causal forward over the whole history from zero
    padding, so each step runs the dense forward on every class frame so far and keeps the last logits;
  * QuantizedNormal.decode with dither on, in float32 as the export runs it; its rand_like draw is recorded by seeding
    the global generator before it;
  * DiagonalShift.inverse of the D - 1 cached decoded frames (initially the value 0.0, as CachedPadding1d pads) and the
    new one.
`torch.multinomial` is replaced by the inverse CDF (first class whose running softmax probability exceeds u) at recorded
float32 uniforms; a uniform within 1e-3 of a float64 CDF edge is redrawn from the same seeded generator, so every class
is unambiguous in float32.  The temperature lines are restated below with their line numbers.
"""
import math
import os

import torch
import torch.nn as nn

from oracle import prior_oracle as P
from oracle.make_golden import GOLDEN
from oracle.make_golden_prior import TINY, build_ref_prior, load_reference_prior

PARAM_SEED = 4321
EDGE = 1e-3
# (D, B, the row temperature levels of the input, call lengths)
CASES = [(4, 1, [0.0], [1, 3, 6, 2]),
         (4, 3, [-2.0, 0.0, 2.5], [2, 1, 5, 4]),
         (8, 3, [-1.0, 0.0, 3.0], [3, 7, 1, 5])]


def _pick(lg, gen):
    """Inverse-CDF class of each row of lg [N, R] (float64) at a float32 uniform at least EDGE from every CDF edge."""
    p = torch.softmax(lg - torch.logsumexp(lg, -1, keepdim=True), -1)      # model.py:147, post_process_prediction
    cum = p.cumsum(-1)
    us, ks = [], []
    for n in range(lg.shape[0]):
        while True:
            u = torch.rand(1, generator=gen)[0]
            if (cum[n] - u.double()).abs().min() >= EDGE:
                break
        over = (cum[n] > u.double()).nonzero()
        us.append(u)
        ks.append(int(over[0]) if len(over) else int((p[n] > 0).nonzero()[-1]))
    return torch.stack(us), torch.tensor(ks)


def golden_case(R, D, B, levels, lengths, seed):
    print(f"prior export: D {D}, B {B}, calls {lengths}")
    res = TINY["resolution"]
    prior = build_ref_prior(R, None, latent_size=D, sr=48000, **TINY)
    shapes = [(k, tuple(v.shape)) for k, v in prior.named_parameters()]
    prior.load_state_dict(P.seeded_params(shapes, PARAM_SEED + D), strict=False)
    prior = prior.double().eval()
    qn = R.prior.core.QuantizedNormal(res)
    ds = R.prior.core.DiagonalShift()
    gen = torch.Generator().manual_seed(seed)

    # TraceModel.__init__: previous_step = quantized_normal.encode(zeros(1, D, 1)), pre_diag_cache of D - 1 zero frames
    history = qn.encode(torch.zeros(1, D, 1)).double().repeat(B, 1, 1)     # stacked one-hot [B, D R, 1]
    cache = torch.zeros(B, D, D - 1)
    calls = []
    for ci, T in enumerate(lengths):
        temp_in = (torch.tensor(levels)[:, None, None] + 0.5 * torch.randn(B, 1, T, generator=gen)).float()
        # scripts/export.py:460-461
        temp = temp_in.double().mean(-1, keepdim=True)
        temp = nn.functional.softplus(temp) / math.log(2)
        uni, dit, cls, out = [], [], [], []
        for i in range(T):
            with torch.no_grad():
                x = prior.forward(history)[..., -1:]                       # export.py:441, dense causal forward
            x = x / temp                                                   # export.py:442
            lg = prior.split_classes(x).reshape(B * D, res)                # [B, D, 1, R]
            u, k = _pick(lg, gen)
            k = k.reshape(B, D)
            onehot = qn.to_stack_one_hot(k[:, :, None])                    # export.py:443-444, previous_step
            history = torch.cat([history, onehot.double()], -1)
            s = int(torch.randint(0, 2 ** 31, (1,), generator=gen))
            torch.manual_seed(s)
            d = torch.rand(B, 1, D)                                        # the rand_like of decode, recorded
            torch.manual_seed(s)
            y = qn.decode(onehot.float())                                  # export.py:447, [B, D, 1]
            seq = torch.cat([cache, y], -1)                                # export.py:448, pre_diag_cache
            out.append(ds.inverse(seq))                                    # export.py:449
            cache = seq[..., 1:]
            uni.append(u.reshape(B, D))
            dit.append(d[:, 0])
            cls.append(k)
        calls.append(dict(temp_in=temp_in, temperature=temp.float(), uniform=torch.stack(uni, 1),
                          dither=torch.stack(dit, 1), classes=torch.stack(cls, 1), out=torch.cat(out, -1)))
        print(f"  call {ci}: T {T}, temperatures {temp.flatten().tolist()}")
    return dict(D=D, B=B, param_seed=PARAM_SEED + D, param_shapes=shapes, calls=calls)


def main():
    R = load_reference_prior()
    cases = [golden_case(R, D, B, lv, ln, seed=100 + i) for i, (D, B, lv, ln) in enumerate(CASES)]
    torch.save(dict(prior_cfg=TINY, edge=EDGE, cases=cases), os.path.join(GOLDEN, "prior_export.pt"))


if __name__ == "__main__":
    main()

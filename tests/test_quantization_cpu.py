"""CPU: the RVQ head of the `discrete` configuration (rave_b200/quantization.py runs on torch; SURVEY K18)
against the unmodified reference under the same RNG seed (build container) and basic invariants."""
import pytest
import torch

from rave_b200 import quantization as Q


def test_rvq_shapes_and_state_dict_names():
    torch.manual_seed(0)
    rvq = Q.ResidualVectorQuantization(num_quantizers=3, dim=8, codebook_size=16)
    keys = set(rvq.state_dict())
    assert {"layers.0._codebook.inited", "layers.0._codebook.cluster_size", "layers.0._codebook.embed",
            "layers.0._codebook.embed_avg"} <= keys
    x = torch.randn(4, 8, 32)
    rvq.train()
    q, loss, idx = rvq(x)
    assert q.shape == x.shape and idx.shape == (4, 3, 32) and idx.dtype == torch.int64
    assert torch.isfinite(loss)
    # residual quantisation: more stages -> smaller error
    errs = []
    rvq.eval()
    codes = rvq.encode(x)
    for n in (1, 2, 3):
        part = sum(rvq.layers[i].decode(codes[:, i]) for i in range(n))
        errs.append(float((x - part).pow(2).mean()))
    assert errs[0] >= errs[1] >= errs[2]
    assert torch.allclose(rvq.decode(codes), sum(rvq.layers[i].decode(codes[:, i]) for i in range(3)))


def test_rvq_matches_reference_bit_for_bit():
    """Against the unmodified reference's ResidualVectorQuantization (tests/golden/reference_pins.pt)."""
    import os
    from oracle.make_reference_pins import rvq_run
    g = torch.load(os.path.join(os.path.dirname(__file__), "golden", "reference_pins.pt"), weights_only=False)["rvq"]
    got = rvq_run(Q, g["x"])
    assert len(got) == len(g["out"])
    for a, b in zip(got, g["out"]):
        assert torch.equal(a, b)

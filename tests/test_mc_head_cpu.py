"""The host restatement of the Monte-Carlo head (mc._generic_mc_forward, mc.chan_merge) against the float64 reference
tests/mc_head_ref.py, on the CPU: the epistemic variance is centred (Welford over a rank's samples, Chan's merge over
the ranks), so it is never negative and keeps its relative accuracy when the samples agree; and the reference's own
bounds are finite at every case of the GPU sweep."""
import math

import pytest
import torch

from tests import mc_head_ref as R


def _close_logits(S, B, C, spread, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (4 * torch.randn(1, B, C, generator=g) + spread * torch.randn(S, B, C, generator=g)).float()


@pytest.mark.parametrize("S,spread", [(10, 1e-2), (100, 1e-2), (25, 1e-1), (7, 0.0)])
def test_generic_mc_forward_epistemic_is_centred(S, spread):
    from pytorch_bayesiancnn_b200 import mc
    L = _close_logits(S, 256, 10, spread)
    lo, kl, (pred, epi, ale, ent) = mc.mc_forward(lambda x, j: (L[j], torch.tensor(2.0)), torch.zeros(256, 1), S,
                                                  want_uncertainty=True)
    ref = R.head(L, None, [2.0])
    assert bool((epi >= 0).all())
    if spread == 0.0:
        assert bool((epi == 0).all())
    p = torch.softmax(L.double(), 2)
    # torch's fp32 softmax on the CPU, not the kernel: bound the per-sample error by a C-term sum (k = C), as the module
    # doc derives for the kernel with its lane sums
    delta = p.amax(0) * R.U * (4 * 10 + 40 + 6 * S)
    bound = (2 * S + 6) * R.U * ref["epi"] + 2 * delta * ref["epi"].sqrt() + delta ** 2
    assert bool(((epi.double() - ref["epi"]).abs() <= bound).all())
    assert bool(((ale.double() - ref["ale"]).abs() <= delta + bound + 3 * R.U).all())
    assert float((pred.double() - ref["pred"]).abs().max()) < 1e-5
    assert float((lo.double() - ref["lo"]).abs().max()) < 1e-5


def test_chan_merge_equals_one_pass_over_all_samples():
    """Groups of 0, 1, 4 and 7 samples merged in order == Welford over all 12, in float64 exactly to rounding; fp32
    groups of nearly equal samples keep a relative error of a few hundred u (E[x^2] - mean^2 would lose all digits)."""
    from pytorch_bayesiancnn_b200 import mc
    x = 0.5 + 1e-4 * torch.randn(12, 1000, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    groups = [x[:0], x[:1], x[1:5], x[5:]]
    counts = [len(g) for g in groups]
    means = [g.mean(0) if len(g) else torch.zeros(1000, dtype=torch.float64) for g in groups]
    m2s = [((g - g.mean(0)) ** 2).sum(0) if len(g) else torch.zeros(1000, dtype=torch.float64) for g in groups]
    mean, m2 = mc.chan_merge(counts, means, m2s)
    ref = ((x - x.mean(0)) ** 2).sum(0)
    assert float((mean - x.mean(0)).abs().max()) < 1e-15
    assert float(((m2 - ref) / ref).abs().max()) < 1e-9
    f = [t.float() for t in means], [t.float() for t in m2s]
    mean32, m232 = mc.chan_merge(counts, *f)
    assert float(((m232.double() - ref) / ref).abs().max()) < 1e-3
    naive = (x.float() ** 2).sum(0) - 12 * x.float().mean(0) ** 2
    assert float(((naive.double() - ref) / ref).abs().max()) > 1e-1


def test_reference_bounds_finite_at_every_sweep_case():
    """mc_head_ref.bounds at every case of the GPU sweep: finite and non-negative wherever the reference is finite, and
    the float64 work of a case stays in the tens of millions of elements."""
    from tests.test_gpu_mc_head_geometry import CASES, _local, _logits
    for cs in CASES:
        assert cs.S * cs.B * cs.C <= 5_000_000, cs.name
        L, labels, kl = _logits(cs)
        ref = R.head(L, labels, kl, cs.normalized, 50000.0, 0.1)
        rs = cs.world // cs.rb
        b = R.bounds(L, labels, kl, max(_local(cs.S, rs, g) for g in range(rs)), rs, cs.normalized, 50000.0, 0.1,
                     ref=ref)
        for k in ("lo", "pred", "epi", "ale", "ent", "ee", "mi"):
            fin = torch.isfinite(ref[k])
            assert bool(fin[..., :].any()), (cs.name, k)
            assert bool(torch.isfinite(b[k][fin]).all() and (b[k][fin] >= 0).all()), (cs.name, k)
        assert math.isfinite(ref["head"][1]), cs.name

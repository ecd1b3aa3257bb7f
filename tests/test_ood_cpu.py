"""Ranking metrics of out-of-distribution detection and selective prediction (mc.ood_metrics, mc.selective_metrics) on
CPU tensors against the float64 restatement tests/ood_ref.py, the host checks of bbb_mc_score_log, and ScoreLog's
bookkeeping.  No GPU needed."""
import ctypes
import math

import numpy as np
import pytest
import torch

from tests import ood_ref as R


def _close(a, b, tol=1e-12):
    return (math.isnan(a) and math.isnan(b)) or abs(a - b) <= tol


def _check_ood(s_in, s_out):
    from pytorch_bayesiancnn_b200 import mc
    got = mc.ood_metrics(torch.as_tensor(s_in), torch.as_tensor(s_out))
    ref = R.ood(s_in, s_out)
    for k in ref:
        assert _close(got[k], ref[k]), (k, got[k], ref[k])
    assert got["n_in"] == len(s_in) and got["n_out"] == len(s_out)
    return got


def _check_selective(s, ok):
    from pytorch_bayesiancnn_b200 import mc
    got = mc.selective_metrics(torch.as_tensor(s), torch.as_tensor(ok))
    ref = R.selective(s, ok)
    for k in ("aurc", "eaurc", "auroc", "accuracy"):
        assert _close(got[k], ref[k]), (k, got[k], ref[k])
    np.testing.assert_allclose(got["coverage"].numpy(), ref["coverage"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(got["risk"].numpy(), ref["risk"], rtol=0, atol=1e-12)
    for c in R.COVERAGES:
        assert _close(got["accuracy_at"][c], ref["accuracy_at"][c]), c
    return got


CASES = {
    "random": lambda g: (g.standard_normal(200), g.standard_normal(150) + 0.7),
    "heavy ties": lambda g: (g.integers(0, 4, 300).astype(float), g.integers(1, 5, 120).astype(float)),
    "all tied": lambda g: (np.full(17, 0.25), np.full(9, 0.25)),
    "one each": lambda g: (np.array([0.3]), np.array([0.7])),
    "one each tied": lambda g: (np.array([0.3]), np.array([0.3])),
    "one in": lambda g: (np.array([1.0]), g.standard_normal(40)),
    "float32 scores": lambda g: (g.random(500).astype(np.float32), (g.random(64) ** 0.5).astype(np.float32)),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_ood_metrics_match_reference(case):
    s_in, s_out = CASES[case](np.random.default_rng(len(case)))
    _check_ood(s_in, s_out)


@pytest.mark.parametrize("case", sorted(CASES))
def test_auroc_is_the_mann_whitney_u(case):
    from scipy.stats import mannwhitneyu
    from pytorch_bayesiancnn_b200 import mc
    s_in, s_out = CASES[case](np.random.default_rng(len(case)))
    u = mannwhitneyu(np.asarray(s_out, np.float64), np.asarray(s_in, np.float64)).statistic
    assert _close(mc.ood_metrics(torch.as_tensor(s_in), torch.as_tensor(s_out))["auroc"], u / (len(s_in) * len(s_out)))


def test_ood_metrics_separated_and_inverted():
    s_in, s_out = np.linspace(0, 1, 30), np.linspace(2, 3, 20)
    m = _check_ood(s_in, s_out)
    assert m["auroc"] == 1.0 and m["fpr_at_95_tpr"] == 0.0 and m["aupr_out"] == 1.0 and m["aupr_in"] == 1.0
    m = _check_ood(s_out, s_in)
    assert m["auroc"] == 0.0 and m["fpr_at_95_tpr"] == 1.0
    m = _check_ood(np.full(5, 1.0), np.full(7, 1.0))
    assert m["auroc"] == 0.5 and m["fpr_at_95_tpr"] == 1.0 and _close(m["aupr_out"], 7 / 12)


@pytest.mark.parametrize("case", ["random", "heavy ties", "all tied", "one", "all correct", "all wrong", "perfect"])
def test_selective_metrics_match_reference(case):
    from pytorch_bayesiancnn_b200 import mc
    g = np.random.default_rng(7)
    n = 301
    s = {"heavy ties": g.integers(0, 5, n).astype(float), "all tied": np.zeros(n), "one": np.array([0.5])}.get(
        case, g.standard_normal(n))
    n = s.size
    ok = {"all correct": np.ones(n), "all wrong": np.zeros(n), "one": np.array([1.0]),
          "perfect": (s < np.sort(s)[n // 3]).astype(float)}.get(case, (g.random(n) < 0.7).astype(float))
    m = _check_selective(s, ok)
    if case == "perfect":                     # every wrong image has a larger score than every correct one
        assert m["auroc"] == 1.0 and _close(m["eaurc"], 0.0)
    if case in ("all correct", "all wrong", "one"):
        assert math.isnan(m["auroc"])
    assert m["n"] == n


def test_selective_accuracy_at_coverage_breaks_ties_by_index():
    from pytorch_bayesiancnn_b200 import mc
    s = torch.zeros(10, dtype=torch.float64)
    ok = torch.tensor([1, 0, 1, 1, 1, 0, 1, 1, 1, 1], dtype=torch.float64)
    m = mc.selective_metrics(s, ok)
    assert m["accuracy_at"][0.5] == 0.8                   # images 0..4
    assert m["accuracy_at"][0.8] == 6 / 8                 # ceil(0.8 * 10) = 8, exactly
    assert m["accuracy_at"][0.99] == 0.8                  # all ten
    assert m["coverage"].tolist() == [1.0] and m["risk"].tolist() == [0.2]


def test_nan_and_empty_raise():
    from pytorch_bayesiancnn_b200 import mc
    x = torch.tensor([0.1, 0.2])
    for a, b in ((torch.tensor([]), x), (x, torch.tensor([])), (torch.tensor([float("nan"), 1.0]), x),
                 (x, torch.tensor([0.0, float("nan")]))):
        with pytest.raises(ValueError):
            mc.ood_metrics(a, b)
    with pytest.raises(ValueError, match="empty"):
        mc.selective_metrics(torch.tensor([]), torch.tensor([]))
    with pytest.raises(ValueError, match="NaN"):
        mc.selective_metrics(torch.tensor([float("nan")]), torch.tensor([1.0]))
    with pytest.raises(ValueError, match="NaN"):
        mc.selective_metrics(x, torch.tensor([1.0, float("nan")]))       # a log without labels
    with pytest.raises(ValueError, match="0 or 1"):
        mc.selective_metrics(x, torch.tensor([1.0, 0.5]))
    with pytest.raises(ValueError, match="correct flags"):
        mc.selective_metrics(x, torch.tensor([1.0]))


def test_score_log_host_checks():
    """bbb_mc_score_log refuses bad arguments before any device work."""
    import __graft_entry__ as g
    g.build()
    from pytorch_bayesiancnn_b200 import _lib as L
    lib = L.lib()
    p = ctypes.c_void_p(0x1000)                  # never dereferenced: every call below fails its host checks

    def call(lo=p, B=4, Cc=10, planes=p, pred=p, cap=8, cursor=p):
        return lib.bbb_mc_score_log(lo, None, None, None, None, None, B, Cc, planes, pred, cap, cursor, None)
    for kw in (dict(lo=None), dict(planes=None), dict(pred=None), dict(cursor=None), dict(B=0), dict(B=-1),
               dict(Cc=0), dict(cap=-1), dict(cap=1 << 48)):
        assert call(**kw) == -1, kw             # BBB_E_INVALID
    assert "bbb_mc_score_log" in L.SYMBOLS and L.MC_SCORE_PLANES == 6


def test_score_log_sizes_and_reset():
    from pytorch_bayesiancnn_b200 import EngineError, mc
    log = mc.ScoreLog("cpu", 5)
    assert len(log) == 0 and log.dropped == 0 and log.capacity == 5
    assert log._planes.shape == (6, 5) and log._planes.dtype == torch.float32
    assert log._pred.shape == (5,) and log._pred.dtype == torch.int32 and log._cursor.tolist() == [0, 0]
    r = log.read()
    assert set(r) == set(mc.ScoreLog.PLANES) | {"pred"} and all(v.numel() == 0 for v in r.values())
    log._cursor.copy_(torch.tensor([3, 0]))         # what three logged images leave behind
    log._planes[0, :3] = torch.tensor([0.5, 0.25, 1.0])
    assert len(log) == 3 and log.read()["confidence"].tolist() == [0.5, 0.25, 1.0]
    log._cursor.copy_(torch.tensor([9, 4]))         # nine appended, four past the end
    assert len(log) == 5 and log.dropped == 4
    with pytest.raises(EngineError, match="4 images did not fit"):
        log.read()
    log.reset()
    assert len(log) == 0 and log.dropped == 0
    empty = mc.ScoreLog("cpu", 0)
    assert len(empty) == 0 and empty._planes.data_ptr() != 0       # the kernel refuses a NULL plane pointer
    with pytest.raises(ValueError):
        mc.ScoreLog("cpu", -1)


def test_score_log_append_and_engines_need_cuda():
    from pytorch_bayesiancnn_b200 import EngineError, mc
    log = mc.ScoreLog("cpu", 4)
    with pytest.raises(EngineError, match="CUDA"):
        log.append(torch.zeros(2, 3))


def test_detect_ood_rejects_unknown_score():
    from pytorch_bayesiancnn_b200 import mc
    with pytest.raises(ValueError, match="unknown score"):
        mc.detect_ood(torch.nn.Linear(2, 2), [], [], 2, score="variation_ratio")

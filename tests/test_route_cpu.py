"""Routing between task experts without a GPU: the float64 restatement (tests/route_ref.py) against the reference's
two-expert formulas (Mixtures/utils_mixture.py:119-187, restated) and against independent formulations for any K, on
random planes, exact ties, NaN scores, out-of-range labels and task labels; the host checks of ExpertStep, route and
the routing log."""
import numpy as np
import pytest
import torch

from tests import route_ref as R


def _random_planes(rng, K, B, C):
    out = []
    for _ in range(K):
        logits = rng.normal(size=(B, C)) * 2
        lo = logits - np.log(np.exp(logits).sum(1, keepdims=True))
        out.append({"pred": rng.normal(size=(B, C)).astype(np.float32),
                    "epistemic": (rng.random((B, C)) * 1e-2).astype(np.float32),
                    "aleatoric": (rng.random((B, C)) * 1e-1).astype(np.float32),
                    "log_outputs": lo.astype(np.float32),
                    "mutual_info": (rng.random(B) * 1e-2).astype(np.float32)})
    return out


def _reference_two_experts(batches, kind):
    """predict_using_uncertainty_separate_models for K = 2 (and, for kind == "confidence", the confidence baseline on
    p_bar), restated: per batch np.sum(..., axis=1), set1_preferred = u2 > u1 (max1 > max2), np.where, the batch
    accuracy of the chosen rows' argmax against the task-local labels; np.mean(accs), the selected counts and total_u."""
    accs, total_u1, total_u2, set1, set2 = [], 0.0, 0.0, 0, 0
    for (p1, p2), labels in batches:
        if kind == "confidence":
            max1 = np.exp(p1["log_outputs"].astype(np.float64)).max(axis=1)
            max2 = np.exp(p2["log_outputs"].astype(np.float64)).max(axis=1)
            set1_preferred = max1 > max2
            u1, u2 = -max1, -max2
        else:
            def u(p):
                epi, ale = p["epistemic"].astype(np.float64), p["aleatoric"].astype(np.float64)
                return {"epistemic": np.sum(epi, axis=1), "aleatoric": np.sum(ale, axis=1),
                        "both": np.sum(epi, axis=1) + np.sum(ale, axis=1)}[kind]
            u1, u2 = u(p1), u(p2)
            set1_preferred = u2 > u1
        total_u1 += np.sum(u1).item()
        total_u2 += np.sum(u2).item()
        preds = np.where(np.expand_dims(set1_preferred, 1), p1["pred"], p2["pred"])
        set1 += int(np.sum(set1_preferred))
        set2 += int(np.sum(~set1_preferred))
        accs.append(np.mean(preds.argmax(axis=1) == labels))
    return np.mean(accs), set1, set2, total_u1, total_u2


@pytest.mark.parametrize("kind", ["epistemic", "aleatoric", "both", "confidence"])
@pytest.mark.parametrize("task", [0, 1])
def test_two_experts_pinned_to_the_reference_formulas(kind, task):
    rng = np.random.default_rng(11 + task)
    B, C, n = 64, 5, 6
    batches = []
    for i in range(n):
        planes = _random_planes(rng, 2, B, C)
        if kind == "confidence":                       # the baseline's class is the argmax of p_bar
            for p in planes:
                p["pred"] = p["log_outputs"].copy()
        if i == 1:                                     # exact ties: the reference keeps expert 2 (u2 > u1 is false)
            for name in ("epistemic", "aleatoric", "log_outputs"):
                planes[1][name][:8] = planes[0][name][:8]
        batches.append((planes, rng.integers(0, C, B)))
    mean_acc, set1, set2, tu1, tu2 = _reference_two_experts(batches, kind)
    acc = R.new_acc(2)
    for planes, labels in batches:
        R.accumulate(acc, planes, kind, labels, task=task)
    assert acc["sum_local_acc"] / acc["steps"] == pytest.approx(mean_acc, rel=1e-15, abs=0)
    assert acc["selected"].tolist() == [set1, set2]
    assert acc["total_score"] == pytest.approx([tu1, tu2], rel=1e-12)
    assert acc["invalid"] == 0 and acc["images"] == n * B
    assert acc["own"] == (set1 if task == 0 else set2)


@pytest.mark.parametrize("K", [2, 3, 7, 16])
@pytest.mark.parametrize("kind", R.SCORES)
def test_choice_matches_independent_formulations(K, kind):
    """Without ties or NaN: np.argmin; with exact ties: the last of the minimal experts; NaN scores: never chosen while
    a number is there, every score NaN: K - 1."""
    rng = np.random.default_rng(K * 7 + len(kind))
    B, C = 200, 4
    planes = _random_planes(rng, K, B, C)
    S = R.scores(planes, kind)
    assert S.shape == (B, K) and np.isfinite(S).all()
    assert np.array_equal(R.choose(S), np.argmin(S, axis=1))
    # ties: copy expert 0's planes onto a random subset of experts for the first 50 rows
    for e in rng.choice(np.arange(1, K), size=max(1, K // 2), replace=False):
        for name in planes[0]:
            planes[e][name][:50] = planes[0][name][:50]
    # NaN: rows 50..99 lose a random expert's score, rows 100..109 every expert's
    for b in range(50, 100):
        e = rng.integers(0, K)
        planes[e]["epistemic"][b, 0] = planes[e]["aleatoric"][b, 0] = np.nan
        planes[e]["log_outputs"][b, 1] = planes[e]["mutual_info"][b] = np.nan
    for p in planes:
        p["epistemic"][100:110, 2] = p["aleatoric"][100:110, 2] = np.nan
        p["log_outputs"][100:110, 3] = p["mutual_info"][100:110] = np.nan
    S = R.scores(planes, kind)
    got = R.choose(S)
    filled = np.where(np.isnan(S), np.inf, S)
    last_min = K - 1 - np.argmin(filled[:, ::-1], axis=1)
    assert np.array_equal(got[:100], last_min[:100])
    assert (got[100:110] == K - 1).all()
    assert np.array_equal(got[110:], np.argmin(S[110:], axis=1))
    assert not np.isnan(S[np.arange(100), got[:100]]).any()


def test_local_class_is_the_first_maximal_and_nan_rows_give_zero():
    rows = np.array([[1, 3, 3, 0], [np.nan, 2, 5, 5], [np.nan] * 4, [-np.inf] * 4, [0.5] * 4], dtype=np.float32)
    assert R.first_argmax(rows).tolist() == [1, 2, 0, 0, 0]


def test_labels_tasks_and_out_of_range():
    K, C = 3, 4
    y = np.array([0, 3, 4, 11, 12, -1, 7])
    tk, ly, gy, ok = R.label_tasks(y, K, C)
    assert tk.tolist() == [0, 0, 1, 2, -1, -1, 1] and ly.tolist() == [0, 3, 0, 3, -1, -1, 3]
    assert ok.tolist() == [True] * 4 + [False, False, True]
    # task given: labels are local classes of that expert; labels that are already global fall out of range
    tk, ly, gy, ok = R.label_tasks(y, K, C, task=2)
    assert ok.tolist() == [True, True, False, False, False, False, False]
    assert gy[:2].tolist() == [8, 11] and (tk[:2] == 2).all()
    # offsets with gaps and a first match
    tk, ly, gy, ok = R.label_tasks(np.array([0, 10, 12, 30]), 2, C, offsets=[10, 30])
    assert tk.tolist() == [-1, 0, 0, 1] and ly.tolist() == [-1, 0, 2, 0]


def test_accumulator_counts_invalid_labels_as_wrong():
    rng = np.random.default_rng(3)
    K, C, B = 2, 5, 40
    planes = _random_planes(rng, K, B, C)
    e, local, pred, S = R.route(planes, "epistemic")
    labels = pred.copy()                                   # every image right
    labels[:5] = 10                                        # out of range: wrong, never an index
    acc = R.new_acc(K)
    R.accumulate(acc, planes, "epistemic", labels)
    assert acc["invalid"] == 5 and acc["global"] == B - 5 and acc["sum_local_acc"] == (B - 5) / B
    assert acc["own"] == B - 5
    # the same labels as task-1 local classes: global labels >= C are out of range
    acc = R.new_acc(K)
    R.accumulate(acc, planes, "epistemic", labels, task=1)
    assert acc["invalid"] == int(np.sum((labels < 0) | (labels >= C)))


# --------------------------------------------------------------------------- #
# host checks (no device needed)
# --------------------------------------------------------------------------- #
def _lenets(classes, n=2):
    from pytorch_bayesiancnn_b200.models import BBBLeNet
    from tests.util import CFG_PRIORS
    return [BBBLeNet(c, 1, CFG_PRIORS, "lrt", "softplus") for c in ([classes] * n if np.isscalar(classes) else classes)]


def test_expert_step_host_checks(monkeypatch):
    from pytorch_bayesiancnn_b200 import EngineError, mc
    x = torch.zeros(8, 1, 32, 32)
    with pytest.raises(ValueError, match="unknown routing score"):
        mc.ExpertStep(_lenets(5), x, 2, score="entropy")
    with pytest.raises(EngineError, match="2 to 16"):
        mc.ExpertStep(_lenets(5, 1), x, 2)
    with pytest.raises(EngineError, match="2 to 16"):
        mc.ExpertStep(_lenets(2, 17), x, 2)
    with pytest.raises(EngineError, match="different numbers of classes"):
        mc.ExpertStep(_lenets([5, 4]), x, 2)
    with pytest.raises(ValueError, match="offsets"):
        mc.ExpertStep(_lenets(5), x, 2, offsets=[0])
    with pytest.raises(ValueError, match="offsets"):
        mc.ExpertStep(_lenets(5), x, 2, offsets=[0, -1])
    with pytest.raises(EngineError, match="one device"):
        mc.ExpertStep(_lenets(5), x.to("meta"), 2)
    with pytest.raises(EngineError, match="CUDA"):
        mc.ExpertStep(_lenets(5), x, 2)
    monkeypatch.setattr(mc, "_dist_info", lambda group: (None, 2, 0))
    with pytest.raises(EngineError, match="one rank"):
        mc.ExpertStep(_lenets(5), x, 2, group=object())


def test_route_host_checks():
    from pytorch_bayesiancnn_b200 import EngineError, mc
    loader = [(torch.zeros(8, 1, 32, 32), torch.zeros(8, dtype=torch.int64))]
    with pytest.raises(ValueError, match="unknown routing score"):
        mc.route(_lenets(5), loader, 2, score="variance")
    with pytest.raises(ValueError, match="task"):
        mc.route(_lenets(5), loader, 2, task=2)
    with pytest.raises(EngineError, match="CUDA"):
        mc.route(_lenets(5), loader, 2, task=1)
    with pytest.raises(EngineError, match="different numbers of classes"):
        mc.route(_lenets([5, 4]), loader, 2)
    with pytest.raises(ValueError, match="unknown routing score"):
        mc.route_batch([{}, {}], "bald")
    with pytest.raises(ValueError, match="num_experts"):
        mc.RouteLog("cpu", 4, 1)
    with pytest.raises(ValueError, match="capacity"):
        mc.RouteLog("cpu", -1, 2)
    assert mc.ROUTE_SCORES == R.SCORES


def test_read_route_metrics_hand_counts():
    from pytorch_bayesiancnn_b200 import _lib as L, mc
    t = torch.zeros(6 + 2 * L.ROUTE_MAX_EXPERTS + 2, dtype=torch.float64)
    t[:6] = torch.tensor([4, 100, 3.0, 70, 80, 0], dtype=torch.float64)
    t[6:9] = torch.tensor([50, 30, 20], dtype=torch.float64)
    t[22:25] = torch.tensor([1.5, 2.5, 3.5], dtype=torch.float64)
    m = mc.read_route_metrics(t, 3)
    assert m["steps"] == 4 and m["images"] == 100 and m["local_accuracy"] == 0.75 and m["accuracy"] == 0.7
    assert m["routing_accuracy"] == 0.8 and m["selected"] == [0.5, 0.3, 0.2] and m["total_score"] == [1.5, 2.5, 3.5]
    assert m["selected_count"] == [50, 30, 20] and m["invalid"] == 0

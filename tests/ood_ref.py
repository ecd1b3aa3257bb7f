"""Float64 numpy restatement of the ranking metrics of mc.ood_metrics / mc.selective_metrics, straight from their
definitions (pairs and thresholds enumerated one by one, no ranks or cumulative sums), and of one score-log entry
(bbb_mc_score_log) from the exchange outputs it reads.  Larger score = more likely OOD / wrong."""
import math
from fractions import Fraction

import numpy as np

COVERAGES = (0.5, 0.8, 0.9, 0.95, 0.99)


def auroc(neg, pos):
    """mean over pairs of [pos > neg] + 1/2 [pos == neg]."""
    neg, pos = np.asarray(neg, np.float64), np.asarray(pos, np.float64)
    gt = (pos[:, None] > neg[None, :]).sum()
    eq = (pos[:, None] == neg[None, :]).sum()
    return (gt + 0.5 * eq) / (pos.size * neg.size)


def average_precision(s, pos):
    """sum_k (R_k - R_{k-1}) P_k over the distinct thresholds t_1 > t_2 > ..., flagging s >= t_k, R_0 = 0."""
    s, pos = np.asarray(s, np.float64), np.asarray(pos, bool)
    ap, r_prev = 0.0, 0.0
    for t in sorted(set(s.tolist()), reverse=True):
        flag = s >= t
        tp = float((flag & pos).sum())
        r = tp / pos.sum()
        ap += (r - r_prev) * tp / flag.sum()
        r_prev = r
    return ap


def fpr_at_tpr(s_in, s_out, level=0.95):
    s_in, s_out = np.asarray(s_in, np.float64), np.asarray(s_out, np.float64)
    best = math.inf
    for t in set(np.concatenate([s_in, s_out]).tolist()):
        tpr = (s_out >= t).sum() / s_out.size
        if tpr >= level:
            best = min(best, (s_in >= t).sum() / s_in.size)
    return best


def ood(s_in, s_out):
    s_in, s_out = np.asarray(s_in, np.float64), np.asarray(s_out, np.float64)
    s = np.concatenate([s_in, s_out])
    out = np.concatenate([np.zeros(s_in.size, bool), np.ones(s_out.size, bool)])
    return {"auroc": auroc(s_in, s_out), "aupr_out": average_precision(s, out), "aupr_in": average_precision(-s, ~out),
            "fpr_at_95_tpr": fpr_at_tpr(s_in, s_out)}


def selective(score, correct):
    s, ok = np.asarray(score, np.float64), np.asarray(correct, np.float64)
    n = s.size
    cov, risk = [], []
    for t in sorted(set(s.tolist())):
        acc = s <= t
        cov.append(acc.sum() / n)
        risk.append((1.0 - ok[acc]).sum() / acc.sum())
    aurc = sum((c - cp) * r for c, cp, r in zip(cov, [0.0] + cov[:-1], risk))
    n_ok = int(ok.sum())
    ideal = sum(max(0, k - n_ok) / k for k in range(1, n + 1)) / n
    bad = ok == 0
    au = auroc(s[~bad], s[bad]) if 0 < n_ok < n else math.nan
    order = sorted(range(n), key=lambda i: (s[i], i))
    at = {c: float(np.mean(ok[order[:max(1, math.ceil(Fraction(str(c)) * n))]])) for c in COVERAGES}
    return {"coverage": np.array(cov), "risk": np.array(risk), "aurc": aurc, "eaurc": aurc - ideal, "auroc": au,
            "accuracy": n_ok / n, "accuracy_at": at}


def score_entry(lo_row, labels_b=None, epistemic_row=None):
    """(confidence, epistemic sum in float64, correct, pred) of one image as bbb_mc_score_log forms them: the argmax is
    the first maximal class (NaN never maximal; a row of -inf gives 0); confidence = float32 expf of that value."""
    lo = np.asarray(lo_row, np.float32)
    finite = [(v, c) for c, v in enumerate(lo.tolist()) if not math.isnan(v)]
    pred = 0
    if finite:
        best = max(v for v, _ in finite)
        pred = next(c for v, c in finite if v == best)
    conf = np.float32(np.exp(np.float32(lo[pred]))) if finite else np.float32(0.0)
    epi = float(np.asarray(epistemic_row, np.float64).sum()) if epistemic_row is not None else math.nan
    correct = (1.0 if int(labels_b) == pred else 0.0) if labels_b is not None else math.nan
    return conf, epi, correct, pred

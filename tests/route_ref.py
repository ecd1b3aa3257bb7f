"""Float64 restatement of the routing between task experts (include/bbb_b200.h, bbb_mc_route), for any K.

``planes``: one dict per expert of numpy float32 arrays, pred / epistemic / aleatoric / log_outputs [B, C] and
mutual_info [B] (the keys the score reads)."""
import numpy as np

SCORES = ("epistemic", "aleatoric", "both", "mutual_info", "confidence")
MAX_EXPERTS = 16


def _row_sum(p):
    """sum_c in class order, in double (the kernel's order)."""
    s = np.zeros(p.shape[0])
    for c in range(p.shape[1]):
        s = s + p[:, c].astype(np.float64)
    return s


def scores(planes, score):
    """[B, K] float64, smaller = preferred."""
    cols = []
    for pl in planes:
        if score == "epistemic":
            s = _row_sum(pl["epistemic"])
        elif score == "aleatoric":
            s = _row_sum(pl["aleatoric"])
        elif score == "both":
            s = _row_sum(pl["epistemic"]) + _row_sum(pl["aleatoric"])
        elif score == "mutual_info":
            s = pl["mutual_info"].astype(np.float64)
        elif score == "confidence":
            lo = pl["log_outputs"]
            with np.errstate(invalid="ignore"):
                s = -np.exp(np.max(lo, axis=1).astype(np.float64))
            s[np.isnan(lo).any(axis=1)] = np.nan
        else:
            raise ValueError(score)
        cols.append(s)
    return np.stack(cols, axis=1)


def choose(S):
    """The routed expert per row of S [B, K]: the smallest score, ties to the highest index, NaN never chosen while a
    number is there (all NaN: K - 1)."""
    B, K = S.shape
    out = np.full(B, K - 1, dtype=np.int64)
    for b in range(B):
        best = None
        for e in range(K):
            v = S[b, e]
            if np.isnan(v):
                continue
            if best is None or v <= S[b, best]:
                best = e
        if best is not None:
            out[b] = best
    return out


def first_argmax(rows):
    """The first maximal class of each row; NaN never maximal, a row of NaN gives 0."""
    r = np.where(np.isnan(rows), -np.inf, rows.astype(np.float64))
    out = np.argmax(r, axis=1)
    out[np.isnan(rows).all(axis=1)] = 0
    return out


def offsets_of(K, C, offsets=None):
    return np.arange(K, dtype=np.int64) * C if offsets is None else np.asarray(offsets, dtype=np.int64)


def route(planes, score, offsets=None):
    """(expert, local, pred, scores) of one batch."""
    K, C = len(planes), planes[0]["pred"].shape[1]
    off = offsets_of(K, C, offsets)
    S = scores(planes, score)
    e = choose(S)
    B = S.shape[0]
    local = np.array([first_argmax(planes[e[b]]["pred"][b:b + 1])[0] for b in range(B)], dtype=np.int64)
    return e, local, off[e] + local, S


def label_tasks(labels, K, C, task=-1, offsets=None):
    """(task, local label, global label, valid) per image (bbb_mc_route's label rules)."""
    off = offsets_of(K, C, offsets)
    y = np.asarray(labels, dtype=np.int64)
    tk = np.full(y.shape, -1)
    ly = np.full(y.shape, -1)
    gy = np.full(y.shape, -1)
    for b in range(y.size):
        if task >= 0:
            if 0 <= y[b] < C:
                tk[b], ly[b], gy[b] = task, y[b], off[task] + y[b]
        else:
            for e in range(K):
                if off[e] <= y[b] < off[e] + C:
                    tk[b], ly[b], gy[b] = e, y[b] - off[e], y[b]
                    break
    return tk, ly, gy, tk >= 0


def new_acc(K):
    return {"steps": 0, "images": 0, "sum_local_acc": 0.0, "global": 0, "own": 0, "invalid": 0,
            "selected": np.zeros(K, dtype=np.int64), "total_score": np.zeros(K)}


def accumulate(acc, planes, score, labels, task=-1, offsets=None):
    """Add one batch to a new_acc() dict; returns route()'s tuple."""
    K, C = len(planes), planes[0]["pred"].shape[1]
    e, local, pred, S = route(planes, score, offsets)
    tk, ly, gy, ok = label_tasks(labels, K, C, task, offsets)
    B = e.size
    acc["steps"] += 1
    acc["images"] += B
    acc["sum_local_acc"] += float(np.sum(ok & (local == ly))) / B
    acc["global"] += int(np.sum(ok & (pred == gy)))
    acc["own"] += int(np.sum(ok & (e == tk)))
    acc["invalid"] += int(np.sum(~ok))
    acc["selected"] += np.bincount(e, minlength=K)
    acc["total_score"] += S.sum(axis=0)
    return e, local, pred, S

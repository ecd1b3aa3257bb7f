"""Split conformal prediction without a GPU: the float64 reference (tests/conformal_ref.py) against brute-force set
definitions, its Philox against known answers, mc.conformal_quantile at its edges, conformal_metrics against hand
counts, the host checks of ConformalLog, and the coverage guarantee on exchangeable synthetic data."""
import math

import numpy as np
import pytest
import torch

from oracle import bbb_oracle as O
from tests import conformal_ref as R


def _rows(B, C, seed, conc=1.0):
    g = np.random.default_rng(seed)
    return np.log(g.dirichlet(np.full(C, conc), size=B)).astype(np.float32)


# --------------------------------------------------------------------------- #
# the reference
# --------------------------------------------------------------------------- #
def test_philox_known_answers_and_oracle():
    """Random123's known-answer vectors, and the oracle's independent restatement at many counters."""
    assert tuple(int(v) for v in R.philox4x32_10(0, 0, 0, 0, 0, 0)) == (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)
    m = 0xFFFFFFFF
    assert tuple(int(v) for v in R.philox4x32_10(m, m, m, m, m, m)) == (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)
    g = np.random.default_rng(0)
    ctr = g.integers(0, 1 << 32, size=(64, 4), dtype=np.uint64).astype(np.uint32)
    key = g.integers(0, 1 << 32, size=2, dtype=np.uint64).astype(np.uint32)
    ours = np.stack(R.philox4x32_10(ctr[:, 0], ctr[:, 1], ctr[:, 2], ctr[:, 3], int(key[0]), int(key[1])), axis=1)
    assert np.array_equal(ours, O.philox4x32_10(ctr, key))


def test_u_depends_on_index_and_is_in_the_open_unit_interval():
    seed, stream = 0x0123456789ABCDEF, (1 << 40) + 5
    idx = np.array([0, 1, 2, (1 << 32) - 1, 1 << 32, (1 << 47) + 3])
    u = R.u_of(seed, stream, idx)
    assert ((u > 0) & (u < 1)).all() and len(set(u.tolist())) == len(idx)
    r = R.philox4x32_10(1 << 32 & 0xFFFFFFFF, 1, stream & 0xFFFFFFFF, stream >> 32, seed & 0xFFFFFFFF, seed >> 32)
    assert u[4] == (float(r[0]) + 0.5) * 2.0 ** -32
    assert np.array_equal(R.u_of(seed, stream, idx[2:]), u[2:])          # a function of the index alone


def _brute(lo_row, method, randomized, lam, k_reg, u):
    """E_c by direct definition: the classes ranked before c, one at a time."""
    C = lo_row.size
    if np.isnan(lo_row).any():
        return np.full(C, np.nan)
    p = np.exp(lo_row.astype(np.float64))
    E = np.empty(C)
    for c in range(C):
        before = [d for d in range(C) if lo_row[d] > lo_row[c] or (lo_row[d] == lo_row[c] and d < c)]
        S, o = sum(p[d] for d in before), len(before)
        if method == R.LAC:
            E[c] = 1.0 - p[c]
        else:
            E[c] = S + (u * p[c] if randomized else p[c])
            if method == R.RAPS:
                E[c] += lam * max(0, o + 1 - k_reg)
    return E


def _special_rows(C, seed):
    lo = _rows(8, C, seed)
    lo[0] = math.log(1.0 / C)                                   # every class tied
    lo[1, C // 2:] = -np.inf                                    # probabilities exactly 0
    lo[2] = -np.inf
    lo[2, C - 1] = 0.0                                          # peaked: one class at log 0
    lo[3] = -1e30
    lo[3, 0] = 0.0
    lo[4, 1] = np.nan
    lo[5, 0], lo[5, C - 1] = -0.0, 0.0                          # signed zeros tie
    lo[6, :] = lo[6, 0]
    lo[6, 1] = lo[6, 0] + 1
    return lo


@pytest.mark.parametrize("method,randomized,lam,k_reg", [
    (R.LAC, False, 0.0, 0), (R.APS, False, 0.0, 0), (R.APS, True, 0.0, 0), (R.RAPS, True, 0.3, 2),
    (R.RAPS, False, 0.01, 0), (R.RAPS, True, 0.0, 5)])
@pytest.mark.parametrize("C", [2, 3, 10, 33])
def test_reference_scores_match_brute_force(C, method, randomized, lam, k_reg):
    lo = _special_rows(C, C)
    u = R.u_of(7, 3, np.arange(lo.shape[0]))
    E = R.scores(lo, method, randomized, lam, k_reg, u)
    for b in range(lo.shape[0]):
        ref = _brute(lo[b], method, randomized, lam, k_reg, u[b])
        assert np.array_equal(np.isnan(E[b]), np.isnan(ref)), b
        assert np.allclose(E[b][~np.isnan(ref)], ref[~np.isnan(ref)], rtol=0, atol=1e-13), b
    assert np.isnan(E[4]).all()


@pytest.mark.parametrize("C", [3, 10, 100])
def test_reference_sets_are_the_textbook_sets(C):
    """LAC keeps {c : p_c >= 1 - q}; non-randomised APS keeps the shortest prefix of the ranking whose mass reaches
    q (every class whose cumulative mass up to and including it is <= q); RAPS with lam = 0 is APS; larger q never
    removes a class."""
    lo = _rows(200, C, C + 1, conc=0.3)
    p = np.exp(lo.astype(np.float64))
    srt, pos = R.order(lo)
    for q in (0.05, 0.5, 0.9, 0.999):
        lac = R.sets(R.scores(lo, R.LAC, False), q)
        assert np.array_equal(lac, p >= 1.0 - q)
        aps = R.sets(R.scores(lo, R.APS, False), q)
        cum = np.cumsum(np.take_along_axis(p, srt, -1), -1)
        assert np.array_equal(aps, np.take_along_axis(cum, pos, -1) <= q)
        assert (np.diff(np.take_along_axis(aps, srt, -1).astype(int), axis=-1) <= 0).all()     # a prefix
        raps0 = R.sets(R.scores(lo, R.RAPS, False, lam=0.0, k_reg=3), q)
        assert np.array_equal(raps0, aps)
    u = R.u_of(1, 2, np.arange(200))
    E = R.scores(lo, R.RAPS, True, 0.05, 2, u)
    small, big = R.sets(E, 0.4), R.sets(E, 0.8)
    assert (big | ~small).all()
    assert not R.sets(E, np.nan).any()


def test_reference_entries():
    lo = _special_rows(10, 2)
    y = np.array([0, 9, 9, 0, 3, 7, 1, 11])                     # the last label is outside [0, C)
    e = R.entries(lo, y, R.APS, True, 0.0, 0, 5, 1, 100, 0.7)
    assert e["label"].tolist() == [0, 9, 9, 0, 3, 7, 1, -1]
    assert np.isnan(e["score"][4]) and np.isnan(e["score"][7]) and e["covered"][7] == -1
    assert e["score"][2] == e["u"][2]                           # peaked row, label on the peak: E_y = u exactly
    assert e["size"][4] == 0 and e["covered"][4] == 0          # a NaN row has an empty set
    none = R.entries(lo, y, R.APS, True, 0.0, 0, 5, 1, 100, np.nan)
    assert (none["size"] == -1).all() and (none["covered"] == -1).all() and not none["sets"].any()


# --------------------------------------------------------------------------- #
# conformal_quantile
# --------------------------------------------------------------------------- #
def test_quantile_rank_and_edges():
    from pytorch_bayesiancnn_b200 import mc
    s = torch.tensor([0.5, 0.1, 0.9, 0.3, 0.7], dtype=torch.float64)
    # n = 5: ceil(6 * 0.9) = 6 > 5 -> +inf; ceil(6 * 0.5) = 3 -> the 3rd smallest; ceil(6 * 0.8) = 5 (exactly 4.8 up)
    assert math.isinf(float(mc.conformal_quantile(s, 0.1)))
    assert float(mc.conformal_quantile(s, 0.5)) == 0.5
    assert float(mc.conformal_quantile(s, 0.2)) == 0.9
    # alpha is read as its shortest decimal, 0.3333333333333333: 6 (1 - alpha) is a hair above 4 and rounds up to 5,
    # the conservative side
    assert float(mc.conformal_quantile(s, 1.0 / 3.0)) == 0.9
    assert float(mc.conformal_quantile(s, 0.999999)) == 0.1        # rank 1
    assert math.isinf(float(mc.conformal_quantile(s, 1e-300)))
    assert math.isinf(float(mc.conformal_quantile(torch.zeros(0, dtype=torch.float64), 0.5)))
    assert float(mc.conformal_quantile(torch.tensor([0.25]), 0.5)) == 0.25      # n = 1: ceil(2 * 0.5) = 1
    # (n + 1)(1 - alpha) an exact integer: no rounding up past it (alpha = 0.1, n = 9: rank 9)
    s9 = torch.arange(9, dtype=torch.float64)
    assert float(mc.conformal_quantile(s9, 0.1)) == 8.0
    # ties
    t = torch.tensor([1.0, 1.0, 1.0, 2.0, 2.0, 3.0, 3.0, 3.0, 3.0], dtype=torch.float64)
    assert float(mc.conformal_quantile(t, 0.5)) == 2.0
    for bad in (0.0, 1.0, -0.1, 1.5, float("nan")):
        with pytest.raises(ValueError, match="alpha"):
            mc.conformal_quantile(s, bad)
    with pytest.raises(ValueError, match="NaN"):
        mc.conformal_quantile(torch.tensor([0.1, float("nan")]), 0.1)


@pytest.mark.parametrize("alpha", [0.05, 0.1, 0.2, 0.5, 0.9])
@pytest.mark.parametrize("n", [1, 2, 9, 19, 100, 1001])
def test_quantile_matches_reference(n, alpha):
    from pytorch_bayesiancnn_b200 import mc
    g = np.random.default_rng(n)
    s = np.round(g.random(n), 2)                               # plenty of ties
    got = float(mc.conformal_quantile(torch.from_numpy(s), alpha))
    ref = R.quantile(s, alpha)
    assert got == ref or (math.isinf(got) and math.isinf(ref))


def test_quantile_mondrian_few_images():
    from pytorch_bayesiancnn_b200 import mc
    s = torch.tensor([0.9, 0.1, 0.4, 0.3, 0.2, 0.8, 0.5], dtype=torch.float64)
    cls = torch.tensor([0, 0, 2, 2, 2, 2, 2])
    q = mc.conformal_quantile(s, 0.4, classes=cls, num_classes=4)
    # class 0: n = 2, ceil(3 * 0.6) = 2 -> 0.9; class 1, 3: no images -> +inf; class 2: n = 5, ceil(3.6) = 4 -> 0.5
    assert q.dtype == torch.float64 and q.shape == (4,)
    assert q[0] == 0.9 and math.isinf(q[1]) and q[2] == 0.5 and math.isinf(q[3])
    g = np.random.default_rng(3)
    s = g.random(500)
    c = g.integers(0, 7, 500)
    c[c == 5] = 4                                              # class 5 empty
    got = mc.conformal_quantile(torch.from_numpy(s), 0.1, classes=torch.from_numpy(c), num_classes=7).numpy()
    assert np.array_equal(got, R.quantile(s, 0.1, c, 7))
    assert mc.conformal_quantile(torch.from_numpy(s), 0.1, classes=torch.from_numpy(c)).shape == (7,)
    with pytest.raises(ValueError, match="classes"):
        mc.conformal_quantile(torch.from_numpy(s), 0.1, classes=torch.from_numpy(c), num_classes=4)
    with pytest.raises(ValueError, match="classes"):
        mc.conformal_quantile(torch.from_numpy(s), 0.1, classes=torch.from_numpy(c[:10]))


# --------------------------------------------------------------------------- #
# conformal_metrics
# --------------------------------------------------------------------------- #
def test_conformal_metrics_hand_counts():
    from pytorch_bayesiancnn_b200 import mc
    C = 12
    sizes = [0, 1, 1, 2, 3, 4, 10, 11, 12, 1]
    labels = [0, 1, 1, 2, 2, 3, 3, 3, 5, -1]
    covered = [0, 1, 0, 1, 1, 0, 1, 1, 1, -1]
    sets = torch.zeros(len(sizes), C, dtype=torch.bool)
    for i, k in enumerate(sizes):
        sets[i, :k] = True
    r = {"size": torch.tensor(sizes, dtype=torch.int32), "covered": torch.tensor(covered, dtype=torch.int32),
         "label": torch.tensor(labels, dtype=torch.int32), "score": torch.zeros(len(sizes), dtype=torch.float64),
         "sets": sets}
    m = mc.conformal_metrics(r)
    assert m["n"] == 10
    assert m["coverage"] == 6 / 9                              # the unlabelled image does not count
    assert m["mean_size"] == sum(sizes) / 10
    assert m["empty_fraction"] == 0.1
    hist = [0] * (C + 1)
    for k in sizes:
        hist[k] += 1
    assert m["size_histogram"].tolist() == hist
    assert m["class_count"].tolist() == [1, 2, 2, 3, 0, 1] + [0] * 6
    cc = m["class_coverage"].tolist()
    assert cc[:4] == [0.0, 0.5, 1.0, 2 / 3] and math.isnan(cc[4]) and cc[5] == 1.0
    assert m["min_class_coverage"] == 0.0
    st = m["size_stratified"]
    assert {k: v["count"] for k, v in st.items()} == {"0": 1, "1": 3, "2-3": 2, "4-10": 2, "11+": 2}
    assert st["0"]["coverage"] == 0.0 and st["1"]["coverage"] == 0.5 and st["2-3"]["coverage"] == 1.0
    assert st["4-10"]["coverage"] == 0.5 and st["11+"]["coverage"] == 1.0
    with pytest.raises(ValueError, match="threshold"):
        mc.conformal_metrics(dict(r, size=torch.full((10,), -1, dtype=torch.int32)))


# --------------------------------------------------------------------------- #
# host checks
# --------------------------------------------------------------------------- #
def test_conformal_log_host_checks():
    from pytorch_bayesiancnn_b200 import mc
    for kw, match in ((dict(method="thr"), "method"), (dict(num_classes=1), "num_classes"),
                      (dict(num_classes=1025), "num_classes"), (dict(lam=-0.1), "lam"),
                      (dict(lam=float("inf")), "lam"), (dict(lam=float("nan")), "lam"), (dict(k_reg=-1), "k_reg"),
                      (dict(capacity=-1), "capacity"), (dict(stream=-1), "stream")):
        args = dict(device="cpu", capacity=4, num_classes=10)
        args.update(kw)
        with pytest.raises(ValueError, match=match):
            mc.ConformalLog(**args)
    log = mc.ConformalLog("cpu", 4, 10, method="raps", lam=0.2, k_reg=1, seed=3, stream=1)
    assert log.threshold is None and log._empty().capacity == 0 and log._empty()._options() == log._options()
    log.set_threshold(0.5)
    assert float(log.threshold) == 0.5 and log._qhat.tolist() == [0.5] * 10
    q = torch.linspace(0, 1, 10, dtype=torch.float64)
    log.set_threshold(q)
    assert torch.equal(log.threshold, q) and torch.equal(log._qhat, q)
    with pytest.raises(ValueError, match="one value or 10"):
        log.set_threshold(torch.zeros(3))


def test_mc_train_step_refuses_a_conformal_log():
    from pytorch_bayesiancnn_b200 import EngineError, mc
    with pytest.raises(EngineError, match="conformal"):
        mc.MCTrainStep(None, None, 2, 1.0, conformal=mc.ConformalLog("cpu", 1, 10))


# --------------------------------------------------------------------------- #
# the guarantee
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("method,randomized,lam,k_reg", [(R.LAC, False, 0.0, 0), (R.APS, True, 0.0, 0),
                                                         (R.RAPS, True, 0.1, 2)])
def test_coverage_on_exchangeable_data(method, randomized, lam, k_reg):
    """Rows p ~ Dirichlet, labels drawn from a distorted p (a miscalibrated net): over 200 seeds of n = 500 calibration
    and 2000 test images the mean coverage lies in [1 - alpha, 1 - alpha + 1/(n + 1)] within 4 standard errors.
    The per-seed variance is that of the Beta(k, n + 1 - k) coverage given the calibration set plus the test
    binomial: k(n + 1 - k) / ((n + 1)^2 (n + 2)) + 0.09 / 2000."""
    alpha, n, m, C, seeds = 0.1, 500, 2000, 10, 200
    covs = []
    for seed in range(seeds):
        g = np.random.default_rng(1000 + seed)
        p = g.dirichlet(np.full(C, 0.5), size=n + m)
        q = p ** 2
        q /= q.sum(1, keepdims=True)                           # the truth is sharper than the net says
        y = (q.cumsum(1) > g.random((n + m, 1))).argmax(1)
        lo = np.log(p).astype(np.float32)
        u = R.u_of(seed, 0, np.arange(n + m))                  # one log index per image: independent u
        E = R.scores(lo, method, randomized, lam, k_reg, u)
        ey = E[np.arange(n + m), y]
        qhat = R.quantile(ey[:n], alpha)
        covs.append(np.mean(R.sets(E[n:], qhat)[np.arange(m), y[n:]]))
    k = R.rank(n, alpha)
    var = k * (n + 1 - k) / ((n + 1) ** 2 * (n + 2)) + alpha * (1 - alpha) / m
    tol = 4 * math.sqrt(var / seeds)
    mean = float(np.mean(covs))
    print(method, mean, tol)
    assert 1 - alpha - tol <= mean <= 1 - alpha + 1 / (n + 1) + tol, (mean, tol)

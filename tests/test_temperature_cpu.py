"""Temperature scaling on the host: the float64 restatement (tests/temperature_ref.py) against a brute-force evaluation,
the search planner mc.temperature_grid (round 0, the narrowing rounds, ties and clamping at the ends), the search's
recovery of a planted temperature, and the argument checks of the pure-host functions."""
import math

import numpy as np
import pytest
from scipy.special import logsumexp

from pytorch_bayesiancnn_b200 import mc
from tests import temperature_ref as R


def _bank(n, S, C, scale, seed):
    rng = np.random.default_rng(seed)
    z = (rng.standard_normal((n, S, C)) * scale).astype(np.float32)
    y = rng.integers(0, C, n)
    return z, y


def _brute(z, y, T):
    tot = 0.0
    for i in range(z.shape[0]):
        lps = []
        for s in range(z.shape[1]):
            row = z[i, s].astype(np.float64) / T
            lps.append(row[y[i]] - logsumexp(row))
        tot += logsumexp(lps) - math.log(len(lps))
    return -tot / z.shape[0]


@pytest.mark.parametrize("n,S,C,scale", [(1, 1, 2, 1.0), (7, 3, 10, 5.0), (20, 25, 4, 1e-3), (5, 2, 100, 1e3)])
@pytest.mark.parametrize("T", [0.05, 0.37, 1.0, 2.5, 20.0])
def test_reference_nll_is_brute_force(n, S, C, scale, T):
    z, y = _bank(n, S, C, scale, n + S + C)
    assert R.nll(z, y, T) == pytest.approx(_brute(z, y, T), rel=1e-12, abs=1e-12)


def test_bound_is_small_and_grows_with_scale():
    z, y = _bank(50, 10, 10, 1.0, 1)
    b1 = R.bound(z, y, 1.0)
    assert 0 < b1 < 1e-4
    assert R.bound(z * 1000, y, 0.05) > R.bound(z, y, 1.0)


def test_grid_round_zero():
    g = mc.temperature_grid(0.05, 20.0, 32)
    lo, hi = math.log(0.05), math.log(20.0)
    assert len(g) == 32 and g[0] == lo
    assert g == [lo + (hi - lo) * k / 31 for k in range(32)]
    assert all(b > a for a, b in zip(g, g[1:]))
    assert abs(g[-1] - hi) < 1e-15
    odd = mc.temperature_grid(0.25, 4.0, 5)
    assert odd[2] == 0.0                              # a symmetric odd grid holds T = 1 itself


@pytest.mark.parametrize("k", [0, 1, 7, 30, 31])
def test_grid_next_round_spans_the_neighbours(k):
    g = mc.temperature_grid(0.05, 20.0, 32)
    nxt = mc.temperature_grid(0.05, 20.0, 32, prev=g, argmin=k)
    lo, hi = g[max(k - 1, 0)], g[min(k + 1, 31)]     # clamped at the ends
    assert nxt[0] == lo and len(nxt) == 32
    assert nxt == [lo + (hi - lo) * j / 31 for j in range(32)]
    step0, step1 = g[1] - g[0], nxt[1] - nxt[0]
    assert step1 == pytest.approx(step0 * (1 if k in (0, 31) else 2) / 31, rel=1e-9)


def test_first_argmin_ties_and_nan():
    assert R.first_argmin([3.0, 1.0, 1.0, 2.0]) == 1
    assert R.first_argmin([float("nan"), 2.0, 2.0]) == 1
    assert R.first_argmin([float("nan")] * 3) == 0


def test_search_schedule_and_t_one():
    z, y = _bank(200, 4, 10, 3.0, 2)
    r = R.search(z, y, 0.05, 20.0, 8, 3)
    assert len(r["trace"]) == 3
    t0 = r["trace"][0]
    assert t0["tau"] == mc.temperature_grid(0.05, 20.0, 8)
    for a, b in zip(r["trace"], r["trace"][1:]):
        k = R.first_argmin(a["nll"])
        assert b["tau"] == mc.temperature_grid(0.05, 20.0, 8, prev=a["tau"], argmin=k)
    assert r["nll_at_one"] == R.nll(z, y, 1.0)
    assert r["nll"] <= r["nll_at_one"]
    assert r["nll"] == pytest.approx(R.nll(z, y, r["temperature"]), rel=1e-12)
    # a bank where T = 1 is best and the grid misses it: the result is T = 1 itself
    rng = np.random.default_rng(3)
    zz = (rng.standard_normal((4000, 1, 5)) * 2).astype(np.float32)
    p = np.exp(zz[:, 0] - logsumexp(zz[:, 0], axis=1, keepdims=True))
    yy = np.array([rng.choice(5, p=pi / pi.sum()) for pi in p])
    r1 = R.search(zz, yy, 0.5, 3.0, 3, 1)               # grid 0.5, 1.22, 3.0 -- T = 1 is not on it
    assert r1["temperature"] == 1.0 and r1["tau"] == 0.0 and r1["nll"] == r1["nll_at_one"]


def test_search_at_bound():
    z, y = _bank(300, 3, 10, 1.0, 4)
    y = z.astype(np.float64).mean(1).argmax(1)        # labels that make T -> 0 best
    assert R.search(z, y, 0.5, 20.0, 8, 2)["at_bound"]


@pytest.mark.parametrize("T0", [0.5, 2.0])
def test_search_recovers_planted_temperature(T0):
    """Labels drawn from p_bar_T0 = mean_s softmax(z_s / T0): the fit finds ln T0 within 4 standard errors of the
    maximum-likelihood estimate (from the observed information n l''(tau)) plus the search's resolution."""
    rng = np.random.default_rng(int(T0 * 10))
    n, S, C = 20000, 4, 10
    z = (rng.standard_normal((n, S, C)) * 3 + rng.standard_normal((n, 1, C)) * 2).astype(np.float32)
    x = z.astype(np.float64) / T0
    p = np.exp(x - logsumexp(x, axis=2, keepdims=True)).mean(1)
    cum = np.cumsum(p, 1)
    y = np.minimum((rng.random((n, 1)) * cum[:, -1:] > cum).sum(1), C - 1)
    r = R.search(z, y, 0.05, 20.0, 32, 4)
    tau0, h = math.log(T0), 1e-3
    curv = (R.nll(z, y, math.exp(tau0 + h)) - 2 * R.nll(z, y, T0) + R.nll(z, y, math.exp(tau0 - h))) / h ** 2
    se = 1.0 / math.sqrt(n * curv)
    step = (math.log(20.0) - math.log(0.05)) / 31 * (2 / 31) ** 3
    assert abs(r["tau"] - tau0) <= 4 * se + step, (r["tau"], tau0, se)
    assert not r["at_bound"]


def test_host_argument_checks():
    with pytest.raises(ValueError, match="t_min < t_max"):
        mc.temperature_grid(2.0, 1.0)
    with pytest.raises(ValueError, match="t_min < t_max"):
        mc.temperature_grid(0.0, 1.0)
    with pytest.raises(ValueError, match="t_min < t_max"):
        mc.temperature_grid(0.1, float("inf"))
    with pytest.raises(ValueError, match="grid must be"):
        mc.temperature_grid(0.1, 10.0, 2)
    with pytest.raises(ValueError, match="grid must be"):
        mc.temperature_grid(0.1, 10.0, 64)
    with pytest.raises(ValueError, match="grid must be"):
        mc.temperature_grid(0.1, 10.0, 4.5)
    g = mc.temperature_grid(0.1, 10.0, 5)
    with pytest.raises(ValueError, match="prev holds"):
        mc.temperature_grid(0.1, 10.0, 5, prev=g[:4], argmin=0)
    with pytest.raises(ValueError, match="argmin"):
        mc.temperature_grid(0.1, 10.0, 5, prev=g, argmin=5)
    with pytest.raises(ValueError, match="argmin"):
        mc.temperature_grid(0.1, 10.0, 5, prev=g)
    with pytest.raises(ValueError, match="rounds"):
        mc._check_search(0.1, 10.0, 5, 0)
    with pytest.raises(ValueError, match="num_ens"):
        mc.LogitBank("cpu", 4, 0, 10)
    with pytest.raises(ValueError, match="num_ens"):
        mc.LogitBank("cpu", 4, 257, 10)
    with pytest.raises(ValueError, match="num_classes"):
        mc.LogitBank("cpu", 4, 2, 1025)
    with pytest.raises(ValueError, match="capacity"):
        mc.LogitBank("cpu", -1, 2, 10)
    with pytest.raises(ValueError, match="normalized"):
        mc._temperature_tensor(2.0, "cpu", True, "MCForward")
    for bad in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="finite and > 0"):
            mc._temperature_tensor(bad, "cpu", False, "MCForward")
    with pytest.raises(ValueError, match="one per expert"):
        mc._expert_temperatures([1.0], 2)
    assert mc._expert_temperatures(None, 3) == [None] * 3

"""Vector scaling on the CPU: the float64 restatement (tests/scaling_ref.py) -- its gradient against central finite
differences, its fit on banks with planted scales and biases against the planted values and scipy's L-BFGS-B, the bound
-- and the host argument rules of mc.LogitScaling, fit_scaling, calibrate_scaling and the engine keywords."""
import math

import numpy as np
import pytest
import torch

from tests import scaling_ref as R


def planted(n, S, C, seed, b_scale=0.7):
    """A bank whose labels are drawn from mean_s softmax(a* z_s + b*): (z fp32 [n, S, C], y [n], a*, b*)."""
    rng = np.random.default_rng(seed)
    z = (rng.standard_normal((n, S, C)) * 2 + rng.standard_normal((n, 1, C)) * 2).astype(np.float32)
    a = rng.uniform(0.4, 1.6, C)
    b = rng.standard_normal(C) * b_scale
    t = z.astype(np.float64) * a + b
    p = np.exp(t - t.max(2, keepdims=True))
    p = (p / p.sum(2, keepdims=True)).mean(1)
    cum = np.cumsum(p, 1)
    y = np.minimum((rng.random((n, 1)) * cum[:, -1:] > cum).sum(1), C - 1)
    return z, y, a, b


@pytest.mark.parametrize("S,C,mu", [(1, 2, 0.0), (3, 5, 0.0), (4, 10, 0.3)])
def test_gradient_is_central_differences(S, C, mu):
    z, y, _, _ = planted(60, S, C, S * 10 + C)
    rng = np.random.default_rng(3)
    a, b = rng.uniform(0.5, 1.5, C), rng.standard_normal(C) * 0.5
    ga, gb = R.gradient(z, y, a, b, mu)
    h = 1e-6
    for c in range(C):
        e = np.zeros(C)
        e[c] = h
        fa = (R.objective(z, y, a + e, b, mu) - R.objective(z, y, a - e, b, mu)) / (2 * h)
        fb = (R.objective(z, y, a, b + e, mu) - R.objective(z, y, a, b - e, mu)) / (2 * h)
        assert abs(fa - ga[c]) <= 1e-7 * (1 + abs(fa)), (c, fa, ga[c])
        assert abs(fb - gb[c]) <= 1e-7 * (1 + abs(fb)), (c, fb, gb[c])
    # the softmax does not see a shift of every bias: the bias gradient sums to 0 without the penalty
    if mu == 0.0:
        assert abs(gb.sum()) < 1e-12


def test_identity_and_temperature_are_special_cases():
    z, y, _, _ = planted(50, 3, 6, 1)
    from tests import temperature_ref as TR
    assert R.objective(z, y, np.ones(6), np.zeros(6)) == pytest.approx(TR.nll(z, y, 1.0), rel=1e-13)
    assert R.objective(z, y, np.full(6, 1 / 2.5), np.zeros(6)) == pytest.approx(TR.nll(z, y, 2.5), rel=1e-13)
    assert np.array_equal(R.apply(z, np.ones(6), np.zeros(6)), z + np.float32(0.0))


def _fisher_se(z, y, a, b):
    """Standard errors of (a, b - mean b) at the optimum: the inverse of n times the Hessian of J (central differences
    of the analytic gradient), on the subspace the softmax identifies (b up to a common shift)."""
    n, _, C = z.shape
    x = np.concatenate([a, b])
    h = 1e-5
    H = np.zeros((2 * C, 2 * C))
    for k in range(2 * C):
        e = np.zeros(2 * C)
        e[k] = h
        gp = np.concatenate(R.gradient(z, y, (x + e)[:C], (x + e)[C:]))
        gm = np.concatenate(R.gradient(z, y, (x - e)[:C], (x - e)[C:]))
        H[:, k] = (gp - gm) / (2 * h)
    cov = np.linalg.pinv(0.5 * (H + H.T) * n, rcond=1e-10)
    P = np.eye(2 * C)
    P[C:, C:] -= 1.0 / C                                            # b -> b - mean b
    cov = P @ cov @ P.T
    return np.sqrt(np.maximum(np.diag(cov), 0.0))


@pytest.mark.parametrize("seed", [1, 2])
def test_fit_recovers_planted_scaling(seed):
    """The fit mc.fit_scaling runs (300 Adam passes with the default steps) recovers the planted a*, b* within 4
    standard errors, and its NLL is within 1e-4 of scipy's L-BFGS-B on the float64 objective."""
    z, y, a0, b0 = planted(1500, 3, 6, seed)
    r = R.fit(z, y)
    la, lb, lJ = R.lbfgs(z, y)
    assert r["nll"] <= r["nll_start"]
    assert r["nll"] - lJ <= 1e-4, (r["nll"], lJ)
    se = _fisher_se(z, y, la, lb)
    est = np.concatenate([r["a"], r["b"] - r["b"].mean()])
    want = np.concatenate([a0, b0 - b0.mean()])
    assert bool((np.abs(est - want) <= 4 * se + 1e-3).all()), (est - want) / se


def test_fit_beats_temperature_on_a_per_class_problem():
    """A class the net predicts too often needs its own bias: vector scaling's NLL is clearly below the best
    temperature's."""
    from tests import temperature_ref as TR
    z, y, _, _ = planted(1500, 3, 6, 7, b_scale=1.5)
    r = R.fit(z, y)
    t = TR.search(z, y, 0.05, 20.0, 32, 4)
    assert r["nll"] < t["nll"] - 0.01, (r["nll"], t["nll"])
    # started from the fitted temperature, it is never worse than that temperature
    r2 = R.fit(z, y, T=t["temperature"])
    assert r2["nll_start"] == pytest.approx(TR.nll(z, y, t["temperature"]), abs=1e-6)
    assert r2["nll"] <= r2["nll_start"]


def test_fit_keeps_the_best_iterate():
    """A step size that diverges: the result is the start, never worse."""
    z, y, _, _ = planted(200, 2, 4, 5)
    r = R.fit(z, y, iters=20, lr=50.0)
    assert r["nll"] <= r["nll_start"] and r["nll_last"] > r["nll"]


def test_bound_is_small_and_grows_with_the_logits():
    z, y, _, _ = planted(100, 4, 10, 9)
    a, b = np.full(10, 1.2), np.linspace(-1, 1, 10)
    bJ, ba, bb = R.bound(z, y, a, b)
    assert 0 < bJ < 1e-4 and bool((ba > 0).all()) and bool((bb > 0).all()) and float(ba.max()) < 1e-3
    bJ2 = R.bound(z * 100, y, a, b)[0]
    assert bJ2 > bJ


def test_schedule_matches_host():
    from pytorch_bayesiancnn_b200 import mc
    assert mc.scaling_schedule(0.1, 300) == R.schedule(0.1, 300)
    s = mc.scaling_schedule(0.2, 4)
    assert s[0] == 0.2 and s == sorted(s, reverse=True) and s[-1] > 0


def test_host_argument_rules():
    from pytorch_bayesiancnn_b200 import EngineError, mc
    with pytest.raises(ValueError, match="kind must be 'vector' or 'matrix'"):
        mc.LogitScaling("cpu", 10, kind="diagonal")
    with pytest.raises(ValueError, match="at most 128 classes"):
        mc.LogitScaling("cpu", 129, kind="matrix")
    m = mc.LogitScaling("cpu", 5, kind="matrix")
    assert torch.equal(m.W, torch.eye(5)) and torch.equal(m.b, torch.zeros(5)) and m.params.shape == (6, 5)
    with pytest.raises(AttributeError):
        m.a
    with pytest.raises(AttributeError):
        mc.LogitScaling("cpu", 5).W
    with pytest.raises(ValueError, match="num_classes"):
        mc.LogitScaling("cpu", 1)
    with pytest.raises(ValueError, match="num_classes"):
        mc.LogitScaling("cpu", 1025)
    s = mc.LogitScaling("cpu", 10)
    assert torch.equal(s.a, torch.ones(10)) and torch.equal(s.b, torch.zeros(10))
    with torch.no_grad():
        s.a.mul_(2.0)
    assert torch.equal(s.reset().params, torch.stack([torch.ones(10), torch.zeros(10)]))
    # the one slot in front of the exchange: a temperature or a scaling, never both, never normalized
    assert mc._logit_map(None, None, "cpu", True, 10, "MCForward") == (None, None)
    with pytest.raises(ValueError, match="not both"):
        mc._logit_map(2.0, s, "cpu", False, 10, "MCForward")
    with pytest.raises(ValueError, match="normalized"):
        mc._logit_map(None, s, "cpu", True, 10, "MCForward")
    with pytest.raises(ValueError, match="normalized"):
        mc._logit_map(2.0, None, "cpu", True, 10, "MCForward")
    with pytest.raises(EngineError, match="holds 10 classes"):
        mc._logit_map(None, s, "cpu", False, 100, "MCForward")
    with pytest.raises(TypeError, match="LogitScaling"):
        mc._logit_map(None, torch.ones(2, 10), "cpu", False, 10, "MCForward")
    assert mc._logit_map(None, s, "cpu", False, 10, "MCForward") == (None, s)
    t, none = mc._logit_map(2.0, None, "cpu", False, 10, "MCForward")
    assert none is None and float(t) == 2.0
    # engine keys: by object for tensors and scalings, by value for floats
    assert mc._map_key(s) == mc._map_key(s) != mc._map_key(mc.LogitScaling("cpu", 10))
    assert mc._map_key(2.0) == 2.0 and mc._map_key(None) is None
    with pytest.raises(ValueError, match="2 scalings for 3 experts"):
        mc._expert_temperatures([s, None], 3, "scalings")
    with pytest.raises(EngineError, match="MCTrainStep does not scale logits"):
        mc.MCTrainStep(None, None, 2, 1000.0, scaling=s)
    # the fit's arguments
    bank = mc.LogitBank("cpu", 4, 2, 10)
    with pytest.raises(ValueError, match="kind must be 'vector' or 'matrix'"):
        mc.fit_scaling(bank, "diagonal")
    with pytest.raises(ValueError, match="at most 128 classes"):
        mc.fit_scaling(mc.LogitBank("cpu", 4, 2, 200), "matrix")
    with pytest.raises(ValueError, match="0 for vector scaling"):
        mc.fit_scaling(bank, l2_offdiag=0.1)
    with pytest.raises(ValueError, match="l2_offdiag"):
        mc.fit_scaling(bank, "matrix", l2_offdiag=-1.0)
    with pytest.raises(TypeError, match="LogitBank"):
        mc.fit_scaling(mc.ProbBank("cpu", 4, 2, 10))
    for kw, msg in ((dict(iters=-1), "iters"), (dict(iters=2.5), "iters"), (dict(lr=float("nan")), "lr"),
                    (dict(lr=-1.0), "lr"), (dict(l2_bias=-0.1), "l2_bias"), (dict(l2_bias=math.inf), "l2_bias")):
        with pytest.raises(ValueError, match=msg):
            mc.fit_scaling(bank, **kw)
    with pytest.raises(EngineError, match="CUDA"):
        mc.fit_scaling(bank)
    with pytest.raises(TypeError):
        mc.fit_scaling(bank, "vector", 300)                         # the arguments after kind are keyword-only
    with pytest.raises(ValueError, match="init must be"):
        mc.calibrate_scaling(None, [], 2, init="matrix")


# --------------------------------------------------------------------------- #
# matrix scaling
# --------------------------------------------------------------------------- #
def planted_m(n, S, C, seed):
    """A bank whose labels are drawn from mean_s softmax(W* z_s + b*), W* near the identity with off-diagonal mass."""
    rng = np.random.default_rng(seed)
    z = (rng.standard_normal((n, S, C)) * 2 + rng.standard_normal((n, 1, C)) * 2).astype(np.float32)
    W = np.diag(rng.uniform(0.4, 1.4, C)) + rng.standard_normal((C, C)) * 0.15
    b = rng.standard_normal(C) * 0.7
    t = R.apply_matrix(z, W, b)
    p = np.exp(t - t.max(2, keepdims=True))
    p = (p / p.sum(2, keepdims=True)).mean(1)
    cum = np.cumsum(p, 1)
    y = np.minimum((rng.random((n, 1)) * cum[:, -1:] > cum).sum(1), C - 1)
    return z, y, W, b


@pytest.mark.parametrize("S,C,lam,mu", [(1, 2, 0.0, 0.0), (3, 5, 0.5, 0.0), (4, 6, 0.2, 0.3)])
def test_matrix_gradient_is_central_differences(S, C, lam, mu):
    z, y, _, _ = planted_m(40, S, C, S + C)
    rng = np.random.default_rng(4)
    W, b = np.eye(C) + rng.standard_normal((C, C)) * 0.3, rng.standard_normal(C) * 0.5
    gW, gb = R.gradient_m(z, y, W, b, lam, mu)
    h = 1e-6
    for j in range(C):
        for k in range(C):
            E = np.zeros((C, C))
            E[j, k] = h
            f = (R.objective_m(z, y, W + E, b, lam, mu) - R.objective_m(z, y, W - E, b, lam, mu)) / (2 * h)
            assert abs(f - gW[j, k]) <= 1e-7 * (1 + abs(f)), (j, k, f, gW[j, k])
        e = np.zeros(C)
        e[j] = h
        f = (R.objective_m(z, y, W, b + e, lam, mu) - R.objective_m(z, y, W, b - e, lam, mu)) / (2 * h)
        assert abs(f - gb[j]) <= 1e-7 * (1 + abs(f)), (j, f, gb[j])
    # the identity is the untransformed predictive, and a diagonal W = I / T the temperature's
    from tests import temperature_ref as TR
    assert R.objective_m(z, y, np.eye(C), np.zeros(C)) == pytest.approx(TR.nll(z, y, 1.0), rel=1e-13)
    assert R.objective_m(z, y, np.eye(C) / 2.5, np.zeros(C)) == pytest.approx(TR.nll(z, y, 2.5), rel=1e-13)


def test_matrix_fit_matches_lbfgs_and_beats_vector():
    """The matrix fit mc.fit_scaling runs (300 Adam passes, ODIR) is within 1e-3 of scipy's L-BFGS-B on the same float64
    objective, never worse than its start, and on a bank planted with off-diagonal mass clearly below vector
    scaling's NLL."""
    z, y, _, _ = planted_m(1500, 3, 6, 2)
    lam = 0.01
    r = R.fit_m(z, y, lam=lam)
    lJ = R.lbfgs_m(z, y, lam=lam)[2]
    assert r["nll"] <= r["nll_start"]
    assert r["nll"] - lJ <= 1e-3, (r["nll"], lJ)
    v = R.fit(z, y)
    nll_m = R.objective_m(z, y, r["W"], r["b"])
    assert nll_m < v["nll"] - 0.005, (nll_m, v["nll"])


def test_matrix_bounds_are_small():
    z, y, _, _ = planted_m(100, 4, 10, 9)
    W, b = np.eye(10) * 1.1 + 0.05, np.linspace(-1, 1, 10)
    bJ, bW, bb = R.bound_m(z, y, W, b, 0.1, 0.1)
    assert 0 < bJ < 0.05 and float(bW.max()) < 0.05 and float(bb.max()) < 0.05        # tf32 operands: ~2^-10
    ab = R.apply_bound(z, W, b)
    assert float(ab.max()) < 1e-4

"""Float64 restatement of vector scaling of the Monte-Carlo predictive (include/bbb_b200.h, bbb_mc_logit_scale /
bbb_scaling_nll_grad; mc.fit_scaling), with the error bounds of the kernel's objective and gradient (helpers, not a test
module).

  apply(z, a, b)            z' = a * z + b per class, as fp32 (fl(fl(z a) + b): the bits of torch's z * a + b)
  objective(z, y, a, b, mu) J = -(1/n) sum_i log( (1/S) sum_s softmax(a z_is + b)[y_i] ) + mu sum_c b_c^2 / C
  gradient(z, y, a, b, mu)  dJ/da, dJ/db: with p_sc = softmax(z'_is)[c] and w_s = p_s[y] / sum_s' p_s'[y],
                            dL_i/dz'_sc = w_s (1[c = y] - p_sc), dJ/da_c = -(1/n) sum_is dL_i/dz'_sc z_sc, dJ/db_c likewise
                            without z, plus 2 mu b_c / C
  fit(z, y, ...)            mc.fit_scaling's passes: Adam on the double iterate, every pass at its fp32 rounding, the
                            best pass kept (the start included)
  bound(z, y, a, b, mu)     |kernel J - J| and |kernel dJ - dJ| per parameter, derived below with u = 2^-24.

The map: the kernel's z'_c = fl(fl(z_c a_c) + b_c) differs from the exact a_c z_c + b_c by
delta_c <= u (|a_c z_c| + |z'_c|); log softmax is 2-Lipschitz in the max-norm of its argument, so lp moves by 2 max delta.
Per row the kernel then forms, as temperature_ref.py derives for the temperature, with x_c = z'_c - max z' (fp32
d_c = x_c (u), times fp32 log2 e (2u)): exponent errors 3u |x_c|, ex2.approx's 4u, one lane's sum of the C terms in
order (C - 1) u, and the flushes below 2^-126:
    rho = sum_c w_c (3u |x_c| + 4u) + (C - 1) u + C 2^-126,      (w = softmax(x))
    e_s = rho + u (3 |x_y| + 3 |ln E| + |lp|) + 2 max_c delta_c            (log2f 2u, the ln 2 product, the difference)
The logmeanexp over s and everything after it is double: the image's term errs by max_s e_s (1-Lipschitz), plus
1e-12 |J| for the double sums.  For the gradient, the kernel's p_sc errs relatively by
    eps_c = 3u |x_c| + 4u + 3u |ln E| + rho + 2 max delta,
its weight w_s (fp32 from a double formed from the lp's) by 2 max_s e_s + u, so a term w_s (1[c=y] - p_sc) z_sc errs by
    |z_sc| w_s ((2 max_s e_s + u) |1[c=y] - p_sc| + p_sc eps_c),
summed over (i, s) and divided by n, plus n S 2^-52 of the sum of the terms' magnitudes for the double sums."""
import math

import numpy as np
from scipy.special import logsumexp

U = 2.0 ** -24
BETA1, BETA2, EPS = 0.9, 0.999, 1e-8


def apply(z, a, b):
    """The kernel's map in fp32: fl(fl(z * a) + b) (numpy float32 arithmetic rounds each operation)."""
    z = np.asarray(z, dtype=np.float32)
    return (z * np.asarray(a, dtype=np.float32)) + np.asarray(b, dtype=np.float32)


def _parts(z, y, a, b):
    z = np.asarray(z, dtype=np.float64)
    y = np.asarray(y, dtype=np.int64)
    t = z * np.asarray(a, dtype=np.float64) + np.asarray(b, dtype=np.float64)
    lse = logsumexp(t, axis=2)
    logp = t - lse[..., None]
    lp = np.take_along_axis(logp, y[:, None, None].repeat(z.shape[1], 1), 2)[:, :, 0]
    L = logsumexp(lp, axis=1) - math.log(z.shape[1])
    w = np.exp(lp - logsumexp(lp, axis=1, keepdims=True))
    return z, y, t, logp, lp, L, w


def objective(z, y, a, b, mu=0.0):
    b64 = np.asarray(b, dtype=np.float64)
    L = _parts(z, y, a, b)[5]
    return float(-L.mean() + mu * (b64 ** 2).sum() / b64.size)


def gradient(z, y, a, b, mu=0.0):
    """(dJ/da [C], dJ/db [C]) in float64."""
    z, y, t, logp, lp, L, w = _parts(z, y, a, b)
    n, S, C = z.shape
    g = -np.exp(logp)
    g[np.arange(n), :, y] += 1.0
    g *= w[..., None]                                               # dL_i/dz'_sc
    b64 = np.asarray(b, dtype=np.float64)
    return -(g * z).sum((0, 1)) / n, -g.sum((0, 1)) / n + 2.0 * mu * b64 / C


def schedule(lr, iters):
    return [lr * 0.5 * (1.0 + math.cos(math.pi * t / iters)) for t in range(iters)]


def fit(z, y, iters=300, lr=0.1, mu=0.0, T=None):
    """mc.fit_scaling in float64: {"a", "b", "nll", "nll_start", "nll_last"}."""
    C = np.asarray(z).shape[2]
    x = np.concatenate([np.full(C, 1.0 if T is None else 1.0 / float(np.float32(T))), np.zeros(C)])
    m, v = np.zeros(2 * C), np.zeros(2 * C)
    steps = schedule(lr, iters)
    best, best_theta, start = math.inf, None, None
    for t in range(iters + 1):
        theta = x.astype(np.float32).astype(np.float64)
        J = objective(z, y, theta[:C], theta[C:], mu)
        if start is None:
            start, best, best_theta = J, J, theta
        elif J < best:
            best, best_theta = J, theta
        if t == iters:
            break
        ga, gb = gradient(z, y, theta[:C], theta[C:], mu)
        g = np.concatenate([ga, gb])
        m = BETA1 * m + (1 - BETA1) * g
        v = BETA2 * v + (1 - BETA2) * g * g
        x = x - steps[t] * (m / (1 - BETA1 ** (t + 1))) / (np.sqrt(v / (1 - BETA2 ** (t + 1))) + EPS)
    return {"a": best_theta[:C], "b": best_theta[C:], "nll": best, "nll_start": start, "nll_last": J}


def lbfgs(z, y, mu=0.0, a0=None):
    """scipy's L-BFGS-B on the float64 objective: (a, b, J)."""
    from scipy.optimize import minimize
    C = np.asarray(z).shape[2]
    x0 = np.concatenate([np.ones(C) if a0 is None else np.asarray(a0, dtype=np.float64), np.zeros(C)])

    def f(x):
        ga, gb = gradient(z, y, x[:C], x[C:], mu)
        return objective(z, y, x[:C], x[C:], mu), np.concatenate([ga, gb])
    r = minimize(f, x0, jac=True, method="L-BFGS-B", options={"maxiter": 5000, "gtol": 1e-10, "ftol": 1e-15})
    return r.x[:C], r.x[C:], float(r.fun)


def bound(z, y, a, b, mu=0.0):
    """(the bound on |J|'s error, the bound on dJ/da's [C], on dJ/db's [C]) of bbb_scaling_nll_grad (module doc)."""
    a32, b32 = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    z, y, t, logp, lp, L, w = _parts(z, y, a32, b32)
    n, S, C = z.shape
    delta = U * (np.abs(z * a32.astype(np.float64)) + np.abs(t))
    dmax = delta.max(2)                                             # [n, S]
    x = t - t.max(2, keepdims=True)
    lse = logsumexp(x, axis=2)                                      # ln E
    p = np.exp(logp)
    xy = np.take_along_axis(x, y[:, None, None].repeat(S, 1), 2)[:, :, 0]
    rho = (p * (3 * U * np.abs(x) + 4 * U)).sum(2) + (C - 1) * U + C * 2.0 ** -126
    e_s = rho + U * (3 * np.abs(xy) + 3 * np.abs(lse) + np.abs(lp)) + 2 * dmax
    e_i = e_s.max(1)
    J = objective(z, y, a32, b32, mu)
    bJ = float(e_i.mean()) + 1e-12 * abs(J)
    eps = 3 * U * np.abs(x) + 4 * U + (3 * U * np.abs(lse) + rho + 2 * dmax)[..., None]
    one = np.zeros_like(p)
    one[np.arange(n), :, y] = 1.0
    dw = (2 * e_i[:, None, None] + U) * np.abs(one - p) + p * eps
    term = w[..., None] * np.abs(one - p)
    dsum = n * S * 2.0 ** -52
    bb = (w[..., None] * dw).sum((0, 1)) / n + dsum * term.sum((0, 1)) / n + 1e-12 * 2 * mu * np.abs(b32) / C
    ba = (w[..., None] * dw * np.abs(z)).sum((0, 1)) / n + dsum * (term * np.abs(z)).sum((0, 1)) / n
    return bJ, ba, bb


# --------------------------------------------------------------------------------------------------------------------
# Matrix scaling, z' = W z + b (C <= 128), with the ODIR penalty lam sum_{j != k} W_jk^2 / (C (C - 1)).
#
# The apply forms output j as an fmaf chain over k = 0 .. C-1 from 0, then + b_j: |err| <= gamma_C sum_k |W_jk z_k|
# + u |z'_j| with gamma_C = C u / (1 - C u) (apply_bound).
#
# The fit pass forms z' on tf32 wgmma: W and z rounded to tf32 (round to nearest, 2^-11 relative each), products
# exact in fp32 and summed in fp32 over K = C in an unspecified order, then + b in fp32.  So
#     delta_j <= (2^-10 + 2^-22 + gamma_C) sum_k |W_jk z_k| + u |z'_j|,
# and the objective errs as in the vector bound with this delta.  The gradient G^T Z takes G and Z rounded to tf32
# (2^-10 relative per product) and accumulates in fp32 over at most MX_ROWS (2048) rows of a CTA (gamma_2048 of the
# magnitudes), the bias gradient the tf32 G (2^-11) in double.
# --------------------------------------------------------------------------------------------------------------------
U_TF32 = 2.0 ** -11
MX_ROWS = 2048


def _gamma(k):
    return k * U / (1 - k * U)


def apply_matrix(z, W, b):
    """Float64 W z + b over the last axis."""
    return np.asarray(z, dtype=np.float64) @ np.asarray(W, dtype=np.float64).T + np.asarray(b, dtype=np.float64)


def apply_bound(z, W, b):
    z = np.asarray(z, dtype=np.float64)
    C = z.shape[-1]
    return _gamma(C) * (np.abs(z) @ np.abs(np.asarray(W, dtype=np.float64)).T) + U * np.abs(apply_matrix(z, W, b))


def _parts_m(z, y, W, b):
    z64 = np.asarray(z, dtype=np.float64)
    y = np.asarray(y, dtype=np.int64)
    t = apply_matrix(z64, W, b)
    lse = logsumexp(t, axis=2)
    logp = t - lse[..., None]
    lp = np.take_along_axis(logp, y[:, None, None].repeat(z64.shape[1], 1), 2)[:, :, 0]
    L = logsumexp(lp, axis=1) - math.log(z64.shape[1])
    w = np.exp(lp - logsumexp(lp, axis=1, keepdims=True))
    return z64, y, t, logp, lp, L, w


def _odir(W, lam):
    W = np.asarray(W, dtype=np.float64)
    C = W.shape[0]
    off = W - np.diag(np.diag(W))
    return lam * (off ** 2).sum() / (C * (C - 1)), 2.0 * lam * off / (C * (C - 1))


def objective_m(z, y, W, b, lam=0.0, mu=0.0):
    b64 = np.asarray(b, dtype=np.float64)
    L = _parts_m(z, y, W, b)[5]
    return float(-L.mean() + _odir(W, lam)[0] + mu * (b64 ** 2).sum() / b64.size)


def gradient_m(z, y, W, b, lam=0.0, mu=0.0):
    """(dJ/dW [C, C], dJ/db [C]) in float64."""
    z, y, t, logp, lp, L, w = _parts_m(z, y, W, b)
    n, S, C = z.shape
    g = -np.exp(logp)
    g[np.arange(n), :, y] += 1.0
    g *= w[..., None]                                               # dL_i/dz'_sc
    b64 = np.asarray(b, dtype=np.float64)
    gW = -np.einsum("isj,isk->jk", g, z) / n + _odir(W, lam)[1]
    return gW, -g.sum((0, 1)) / n + 2.0 * mu * b64 / C


def bound_m(z, y, W, b, lam=0.0, mu=0.0):
    """(bound on |J|'s error, on dJ/dW's [C, C], on dJ/db's [C]) of bbb_scaling_nll_grad's matrix pass (above)."""
    W32, b32 = np.asarray(W, dtype=np.float32), np.asarray(b, dtype=np.float32)
    z, y, t, logp, lp, L, w = _parts_m(z, y, W32, b32)
    n, S, C = z.shape
    mag = np.abs(z) @ np.abs(W32.astype(np.float64)).T
    delta = (2 * U_TF32 + 2.0 ** -22 + _gamma(C)) * mag + U * np.abs(t)
    dmax = delta.max(2)
    x = t - t.max(2, keepdims=True)
    lse = logsumexp(x, axis=2)
    p = np.exp(logp)
    xy = np.take_along_axis(x, y[:, None, None].repeat(S, 1), 2)[:, :, 0]
    rho = (p * (3 * U * np.abs(x) + 4 * U)).sum(2) + (C - 1) * U + C * 2.0 ** -126
    e_s = rho + U * (3 * np.abs(xy) + 3 * np.abs(lse) + np.abs(lp)) + 2 * dmax
    e_i = e_s.max(1)
    J = objective_m(z, y, W32, b32, lam, mu)
    bJ = float(e_i.mean()) + 1e-12 * abs(J)
    eps = 3 * U * np.abs(x) + 4 * U + (3 * U * np.abs(lse) + rho + 2 * dmax)[..., None]
    one = np.zeros_like(p)
    one[np.arange(n), :, y] = 1.0
    dw = (2 * e_i[:, None, None] + U) * np.abs(one - p) + p * eps      # the kernel's g before rounding
    term = w[..., None] * np.abs(one - p)                           # |g|
    err_g = w[..., None] * dw + U_TF32 * (term + w[..., None] * dw)   # and its tf32 rounding
    rows = min(n * S, MX_ROWS)
    dsum = n * S * 2.0 ** -52
    bW = (np.einsum("isj,isk->jk", err_g, np.abs(z)) + (2 * U_TF32 + _gamma(rows) + dsum)
          * np.einsum("isj,isk->jk", term, np.abs(z))) / n
    bb = (err_g.sum((0, 1)) + dsum * term.sum((0, 1))) / n
    return bJ, bW + 1e-12 * np.abs(_odir(W32, lam)[1]), bb + 1e-12 * 2 * mu * np.abs(b32) / C


def fit_m(z, y, iters=300, lr=0.1, lam=0.0, mu=0.0, T=None):
    """mc.fit_scaling(kind="matrix") in float64: {"W", "b", "nll", "nll_start", "nll_last"}."""
    C = np.asarray(z).shape[2]
    x = np.concatenate([(np.eye(C) * (1.0 if T is None else 1.0 / float(np.float32(T)))).ravel(), np.zeros(C)])
    m, v = np.zeros_like(x), np.zeros_like(x)
    steps = schedule(lr, iters)
    best, best_theta, start = math.inf, None, None
    for t in range(iters + 1):
        theta = x.astype(np.float32).astype(np.float64)
        W, b = theta[:C * C].reshape(C, C), theta[C * C:]
        J = objective_m(z, y, W, b, lam, mu)
        if start is None:
            start, best, best_theta = J, J, theta
        elif J < best:
            best, best_theta = J, theta
        if t == iters:
            break
        gW, gb = gradient_m(z, y, W, b, lam, mu)
        g = np.concatenate([gW.ravel(), gb])
        m = BETA1 * m + (1 - BETA1) * g
        v = BETA2 * v + (1 - BETA2) * g * g
        x = x - steps[t] * (m / (1 - BETA1 ** (t + 1))) / (np.sqrt(v / (1 - BETA2 ** (t + 1))) + EPS)
    return {"W": best_theta[:C * C].reshape(C, C), "b": best_theta[C * C:], "nll": best, "nll_start": start,
            "nll_last": J}


def lbfgs_m(z, y, lam=0.0, mu=0.0):
    """scipy's L-BFGS-B on the float64 matrix objective: (W, b, J)."""
    from scipy.optimize import minimize
    C = np.asarray(z).shape[2]

    def f(x):
        W, b = x[:C * C].reshape(C, C), x[C * C:]
        gW, gb = gradient_m(z, y, W, b, lam, mu)
        return objective_m(z, y, W, b, lam, mu), np.concatenate([gW.ravel(), gb])
    x0 = np.concatenate([np.eye(C).ravel(), np.zeros(C)])
    r = minimize(f, x0, jac=True, method="L-BFGS-B", options={"maxiter": 5000, "gtol": 1e-10, "ftol": 1e-15})
    return r.x[:C * C].reshape(C, C), r.x[C * C:], float(r.fun)

"""Float64 restatement of temperature scaling of the Monte-Carlo predictive (include/bbb_b200.h, bbb_temperature_nll;
mc.fit_temperature), with the error bound of the kernel's NLL (helpers, not a test module).

  nll(z, y, T)   l(T) = -(1/n) sum_i log( (1/S) sum_s softmax(z_is / T)[y_i] ),  z [n, S, C], y [n]
  search(...)    the grid search on tau = ln T: round 0 on mc.temperature_grid(t_min, t_max, grid) plus tau = 0, then
                 every round on the grid around the first minimal point; never worse than T = 1
  bound(z, y, tau)   |kernel nll - nll| at each tau, derived below with u = 2^-24 (fp32 unit roundoff) to first order.

Per (i, s) the kernel forms, in fp32, d_c = z_c - m (m = max_c z_c; u |d_c|), a = (float)(log2(e) / T) (u), d_c a (u):
the exponent of each term errs by 3u |x_c| with x_c = (z_c - m) / T, which moves the term by 3u |x_c| relative;
ex2.approx adds 2 ulp = 4u, and a term below 2^-126 flushes to 0 (C 2^-126 of a sum >= 1); the sum of C terms in order
(C - 1) u.  So the sum E = sum_c exp(x_c) errs by rho = sum_c w_c (3u |x_c| + 4u) + (C - 1) u + C 2^-126 relative
(w = softmax(x)); log2f adds 1 ulp = 2u |ln E| (in natural units); d_y a 3u |x_y|; the difference u |lp|:
    e_s = rho + u (3 |x_y| + 2 |ln E| + |lp|),      lp = x_y - ln E = log softmax(z_s / T)[y].
The logmeanexp over s is 1-Lipschitz in the lp's, and its own fp32 online (max, sum) over a lane's n_loc = ceil(S/32)
samples and the five levels of the warp tree carries at most 11u of the total per update (each term and rescale:
the argument's rounding, ex2's 4u, the multiply and the add), so the image's term errs by
    e_i = max_s e_s + 11u (n_loc + 5),
and the mean over images by mean_i e_i; the double sums after it add n 2^-53 relative, covered by 1e-12 |l|."""
import math

import numpy as np
from scipy.special import logsumexp

U = 2.0 ** -24


def _x(z, T):
    z = np.asarray(z, dtype=np.float64)
    return (z - z.max(2, keepdims=True)) / T


def image_ll(z, y, T):
    """[n] log( (1/S) sum_s softmax(z_is / T)[y_i] ) in float64."""
    x = _x(z, T)
    y = np.asarray(y, dtype=np.int64)
    lp = np.take_along_axis(x, y[:, None, None].repeat(x.shape[1], 1), 2)[:, :, 0] - logsumexp(x, axis=2)
    return logsumexp(lp, axis=1) - math.log(x.shape[1])


def nll(z, y, T):
    return float(-image_ll(z, y, T).mean())


def first_argmin(v):
    """The first minimal value's index; NaN never minimal (all NaN: 0)."""
    best, kb = math.inf, 0
    for k, x in enumerate(v):
        if x < best:
            best, kb = x, k
    return kb


def search(z, y, t_min=0.05, t_max=20.0, grid=32, rounds=4):
    """The search mc.fit_temperature runs, in float64: {"temperature", "tau", "nll", "nll_at_one", "at_bound", "trace"}."""
    from pytorch_bayesiancnn_b200 import mc
    taus = mc.temperature_grid(t_min, t_max, grid)
    at_one = nll(z, y, 1.0)
    trace = []
    for r in range(rounds):
        v = [nll(z, y, math.exp(t)) for t in taus]
        trace.append({"tau": list(taus), "nll": v})
        k = first_argmin(v)
        if r == 0:
            at_bound = k in (0, grid - 1)
        if r + 1 < rounds:
            taus = mc.temperature_grid(t_min, t_max, grid, prev=taus, argmin=k)
    best, tau = v[k], taus[k]
    if best > at_one:
        best, tau = at_one, 0.0
    return {"temperature": math.exp(tau), "tau": tau, "nll": best, "nll_at_one": at_one, "at_bound": at_bound,
            "trace": trace}


def bound(z, y, T):
    """The bound on |bbb_temperature_nll - nll(z, y, T)| (module doc)."""
    x = _x(z, T)
    n, S, C = x.shape
    y = np.asarray(y, dtype=np.int64)
    lse = logsumexp(x, axis=2)                                   # ln E
    w = np.exp(x - lse[..., None])
    xy = np.take_along_axis(x, y[:, None, None].repeat(S, 1), 2)[:, :, 0]
    lp = xy - lse
    rho = (w * (3 * U * np.abs(x) + 4 * U)).sum(2) + (C - 1) * U + C * 2.0 ** -126
    e_s = rho + U * (3 * np.abs(xy) + 2 * np.abs(lse) + np.abs(lp))
    e_i = e_s.max(1) + 11 * U * (math.ceil(S / 32) + 5)
    return float(e_i.mean()) + 1e-12 * abs(nll(z, y, T))

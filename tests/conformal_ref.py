"""float64 numpy restatement of split conformal prediction as bbb_mc_conformal_log and mc.conformal_quantile define it
(include/bbb_b200.h), with a numpy Philox4x32-10 that reproduces the kernel's randomisation u bit for bit."""
from fractions import Fraction

import numpy as np

LAC, APS, RAPS = "lac", "aps", "raps"
M32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """common.cuh's philox4x32_10 on uint32 arrays (broadcast); returns (x, y, z, w)."""
    c = [np.asarray(v, dtype=np.uint64) & M32 for v in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0) & M32, np.uint64(k1) & M32
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        hi0, lo0, hi1, lo1 = p0 >> np.uint64(32), p0 & M32, p1 >> np.uint64(32), p1 & M32
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
        k0 = (k0 + np.uint64(0x9E3779B9)) & M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & M32
    return tuple(v.astype(np.uint32) for v in c)


def u_of(seed, stream, idx):
    """u of the images at log indices idx: (r.x + 0.5) 2^-32, r = philox(counter (i_lo, i_hi, stream_lo, stream_hi),
    key seed)."""
    i = np.asarray(idx, dtype=np.uint64)
    r = philox4x32_10(i & M32, i >> np.uint64(32), stream & 0xFFFFFFFF, stream >> 32, seed & 0xFFFFFFFF, seed >> 32)
    return (r[0].astype(np.float64) + 0.5) * 2.0 ** -32


def order(lo):
    """[B, C] positions of the classes: log p descending, ties to the smaller class, -inf last."""
    lo = np.asarray(lo, dtype=np.float32)
    B, C = lo.shape
    srt = np.lexsort((np.broadcast_to(np.arange(C), (B, C)), -lo.astype(np.float64)), axis=-1)
    pos = np.empty_like(srt)
    np.put_along_axis(pos, srt, np.broadcast_to(np.arange(C), (B, C)), axis=-1)
    return srt, pos


def scores(lo, method, randomized, lam=0.0, k_reg=0, u=None):
    """E [B, C] in float64 (every E of a row that holds a NaN is NaN)."""
    lo = np.asarray(lo, dtype=np.float32)
    B, C = lo.shape
    p = np.exp(lo.astype(np.float64))
    if method == LAC:
        E = 1.0 - p
    else:
        srt, pos = order(lo)
        ps = np.take_along_axis(p, srt, axis=-1)
        S_sorted = np.cumsum(ps, axis=-1) - ps                     # mass before each position
        S = np.take_along_axis(S_sorted, pos, axis=-1)
        uu = np.ones(B) if (not randomized or u is None) else np.asarray(u, dtype=np.float64)
        E = S + (uu[:, None] * p if randomized else p)
        if method == RAPS:
            E = E + lam * np.maximum(0, pos + 1 - k_reg)
    E[np.isnan(lo).any(axis=1)] = np.nan
    return E


def sets(E, qhat):
    """bool [B, C]: E_c <= q_hat_c; none at all while q_hat holds a NaN."""
    q = np.broadcast_to(np.asarray(qhat, dtype=np.float64).reshape(-1), (E.shape[1],))
    if np.isnan(q).any():
        return np.zeros(E.shape, dtype=bool)
    with np.errstate(invalid="ignore"):
        return E <= q[None, :]


def entries(lo, labels, method, randomized, lam, k_reg, seed, stream, first_index, qhat):
    """The entries one launch appends at first_index .. first_index + B - 1."""
    lo = np.asarray(lo, dtype=np.float32)
    B, C = lo.shape
    u = u_of(seed, stream, first_index + np.arange(B))
    E = scores(lo, method, randomized, lam, k_reg, u)
    y = np.full(B, -1, dtype=np.int64) if labels is None else np.asarray(labels, dtype=np.int64).copy()
    y[(y < 0) | (y >= C)] = -1
    st = sets(E, qhat)
    no_q = np.isnan(np.asarray(qhat, dtype=np.float64)).any()
    has = y >= 0
    score = np.full(B, np.nan)
    score[has] = E[has, y[has]]
    covered = np.full(B, -1, dtype=np.int64)
    if not no_q:
        covered[has] = st[has, y[has]]
    return {"score": score, "E": E, "u": u, "sets": st, "size": np.full(B, -1) if no_q else st.sum(1),
            "covered": covered, "label": y}


def rank(n, alpha):
    a = Fraction(repr(float(alpha)))
    return -(-(n + 1) * (a.denominator - a.numerator) // a.denominator)


def quantile(s, alpha, classes=None, num_classes=None):
    """ceil((n + 1)(1 - alpha))-th smallest score (+inf past n), per class with classes."""
    s = np.asarray(s, dtype=np.float64)
    if classes is None:
        k = rank(s.size, alpha)
        return np.sort(s)[k - 1] if k <= s.size else np.inf
    classes = np.asarray(classes)
    return np.array([quantile(s[classes == c], alpha) for c in range(num_classes)])

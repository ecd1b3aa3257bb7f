"""Float64 restatement of BatchBALD (Kirsch et al. 2019) as the engine computes it (include/bbb_b200.h,
bbb_joint_entropy; mc.batchbald): the joint entropy by brute-force enumeration, the normalised-column estimator
H(y_A, y_i) = sum_m omega_m h_m(i) + const, and the greedy loop.  probs: [N, S, C] float64 per-sample probabilities."""
import itertools

import numpy as np


def _xlogx(x):
    x = np.asarray(x, dtype=np.float64)
    return np.where(x > 0, x * np.log(np.where(x > 0, x, 1.0)), 0.0)


def expected_entropy(probs):
    """E_s H[p_s(y_i)] per candidate: [N]."""
    return -_xlogx(probs).sum(2).mean(1)


def joint_entropy_brute(probs, idx):
    """H(y_idx) by enumerating every label tuple: P(y) = (1/S) sum_s prod_j p_s(y_j)."""
    N, S, C = probs.shape
    h = 0.0
    for ys in itertools.product(range(C), repeat=len(idx)):
        p = np.ones(S)
        for j, y in zip(idx, ys):
            p = p * probs[j, :, y]
        h -= float(_xlogx(p.mean()))
    return h


def exact_configs(probs, chosen):
    """The exact configurations of the labels of ``chosen``: (pt [M, S] normalised columns, omega [M], const,
    configs [M, n]) in the engine's order (the last label varies fastest)."""
    N, S, C = probs.shape
    pt, omega, configs = np.full((1, S), 1.0 / S), np.ones(1), np.zeros((1, 0), dtype=np.int64)
    for a in chosen:
        pa = probs[a].T                                     # [C, S]
        q = pt @ pa.T                                       # [M, C]
        col = (pt[:, None, :] * pa[None]).reshape(-1, S)
        qf = q.reshape(-1, 1)
        pt = np.where(qf > 0, col / np.where(qf > 0, qf, 1.0), 0.0)
        omega = (omega[:, None] * q).reshape(-1)
        configs = np.concatenate([np.repeat(configs, C, 0), np.tile(np.arange(C), len(configs))[:, None]], 1)
    return pt, omega, -float(_xlogx(omega).sum()), configs


def sampled_configs(probs, chosen, configs):
    """The sampled estimator's inputs for given label configurations [M, n] of ``chosen``: (pt, omega = 1/M, const =
    -(1/M) sum_m log P(y_A(m)))."""
    N, S, C = probs.shape
    M = configs.shape[0]
    p = np.ones((M, S))
    for j, a in enumerate(chosen):
        p = p * probs[a][:, configs[:, j]].T                # [M, S]
    tot = p.sum(1, keepdims=True)
    return p / tot, np.full(M, 1.0 / M), -float(np.log(tot[:, 0] / S).mean())


def h_m(probs, pt):
    """h_m(i) = -sum_c Q log Q, Q[m, c] = sum_s pt[m, s] p_s(y_i = c): [N, M]."""
    q = np.einsum("ms,nsc->nmc", pt, probs)
    return -_xlogx(q).sum(2)


def scores(probs, pt, omega, const, chosen, eh=None):
    """a(A u {i}) for every candidate i (chosen ones -inf) and the per-candidate h_m: (scores [N], h [N, M])."""
    eh = expected_entropy(probs) if eh is None else eh
    h = h_m(probs, pt)
    a = h @ omega + const - sum(eh[j] for j in chosen) - eh
    a[list(chosen)] = -np.inf
    return a, h


def greedy_exact(probs, k):
    """Greedy BatchBALD with exact enumeration in every round: (indices, scores)."""
    chosen, got = [], []
    for _ in range(k):
        pt, omega, const, _ = exact_configs(probs, chosen)
        a, _ = scores(probs, pt, omega, const, chosen)
        i = int(np.argmax(a))
        chosen.append(i)
        got.append(float(a[i]))
    return chosen, got

"""Float64 restatement of the Monte-Carlo head (the exchange kernel's outputs, include/bbb_b200.h bbb_mc_exchange*), with
a per-element error bound for each fp32 output (helpers, not a test module).

head(...) returns, from [S, B, C] logits, labels, the per-sample KL terms, ``normalized``, train_size and beta:
  lo [B, C]      logmeanexp_s log p_hat_s                       (main_bayesian.py:46-53, utils.py:14-22)
  kl             sum(kl_terms)                                  (one sample's KL; kl_out = S * kl / S)
  pred, epi, ale [B, C], ent [B]                                (oracle.uncertainty: the centred epistemic form)
  ee, mi [B]                                                    (tests/info_ref.information)
  head [4]       nll * train_size + beta * kl, nll, accuracy, beta * kl   (metrics.py:12-14, 23-24)
  sums           tests/eval_ref.batch_sums of lo                (the METRICS accumulator of one step)
and bounds(...) the matching error bounds, derived below with u = 2^-24 (fp32 unit roundoff; one ulp is at most 2u
relative) and first-order error analysis.  Device functions: expf <= 2 ulp, logf and log1pf <= 1 ulp, __fdividef <=
2 ulp (CUDA C Programming Guide, Mathematical Functions, default flags).  Notation per element (b, c) and sample s:
l the logit, r_s the row normaliser (log-sum-exp, or sum softplus with ``normalized``), lp = log p_hat, p = p_hat;
n_loc the most samples one sender holds, n_src the number of senders (ranks, or sample groups with row blocks),
k = ceil(C / 32) + 5 the length of one lane's sum plus the five levels of the warp tree.

  p_hat, softmax.  r = mx + logf(sum expf(l - mx)): each term carries 4u + u|l - mx|, which weighted by p_c sums to
    4u + u E_p|l - mx|; the sum adds k u; logf adds 2u |log se|; the final add u |r|.  lp = l - r adds u |lp|, and
    expf 4u more:  e_lp = u (|r| + |lp| + 2 log se + E_p|l - mx| + k + 9),  e_p = e_lp + 4u (relative error of p);
    a p below FLT_MIN is subnormal or 0: an absolute eta = 2^-148 as well.
  p_hat, normalized.  softplus: expf 4u, log1pf 2u (log1p(y) is no more sensitive than y); the sum k u; the
    division 2u:  e_p = u (k + 20); and fp32 subnormals add an absolute eta = 2^-148 max(1, 1 / sum softplus).
    lp = logf(p) (2u |lp|), or below FLT_MIN (l or logf(softplus l)) - logf(sum) (u |l| + 2u |lp|); the reference
    takes log softplus(l) = l below l = -30 as well, where float64's softplus underflows long before fp32's log does:
    e_lp = e_p + 2u |lp| + u |l|.
  lo.  The online logmeanexp over a sender's samples, then over the senders: every sample's term, every rescale and
    every add carries at most 11u of the (positive) total (the u|x| e^x terms of expf are <= u / e each), logf(tot / S)
    2u |log S| + 4u, the final add u |lo|:  |d lo| <= max_s e_lp,s + u (11 (n_loc + n_src) + 4 + 2 log S + |lo|).
  pred.  Recursive sums of the S logits:  |d pred| <= u (S + n_src + 1) mean_s |l_s|.
  epistemic.  Welford over each sender's samples, Chan's merge over the senders.  The per-sample errors e_p p and the
    mean updates (three roundings, __fdividef 4u: <= 6u p per update) move the centred values by at most
    delta = max_s e_p,s p_s + 6u (n_loc + n_src) max_s p_s + eta, and an RMS moved by delta moves by <= delta:
    |sqrt(got) - sqrt(ref)| <= delta.  The sums of the non-negative squares add (2 (S + n_src) + 4) u relative, and
    their at most 2 S + 1 terms round on fp32's subnormal grid (2^-150 each, 2^-148 after the division by S):
        |got - ref| <= (2 (S + n_src) + 4) u ref + 2 delta sqrt(ref) + delta^2 + 2^-148,   and got >= 0.
    (An epistemic variance below 2^-148, about 3e-45, is not representable: its bound is that floor.)
    The one-pass E[p^2] - p_bar^2 errs by ~S u p_bar^2 instead: far outside this bound when the samples agree.
  aleatoric = p_bar (1 - p_bar) - epi:  |d| <= delta |1 - 2 p_bar| + delta^2 + |d epi| + u (3 p_bar (1 - p_bar) + |ale|).
  entropy H[p_bar].  d(p log p) = (log p + 1) dp with |dp| <= delta; below delta p log p is not Lipschitz, so
    L = |log max(p_bar, delta)| + 1 and the factor 2:  |d H| <= sum_c 2 delta_c L_c + u (k + 3) sum_c p_bar |log p_bar|.
  expected entropy (1/S) sum_s H[p_hat_s]:  per term |d(p lp)| <= p (|lp| + 1)(e_p + 3u) + p e_lp + eta (|lp| + 1),
    plus the sums (n_loc k + n_src + 7) u ee.  (p e_lp where p > 0.)
  mutual information = ent - ee in fp32:  |d mi| <= |d ent| + |d ee| + u |mi|.  It stays a difference of two
    entropies, so a mutual information below about u H is not resolved: its bound is absolute, set by the entropies.
  kl_out = (sum over senders of S_loc * sum_i kl_i) / S:  |d| <= u (n_kl + n_src + 3) sum_i |kl_i|.
  head: nll = mean_b -lo[b, y_b] in double, rounded to fp32: |d nll| <= mean_b |d lo[b, y_b]| + u |nll|;
    loss = nll * train_size + beta * kl in fp32: |d| <= train_size |d nll| + beta |d kl| + 3u (train_size |nll| + |beta kl|).
"""
import math

import torch
import torch.nn.functional as F

from oracle import bbb_oracle as O
from tests import eval_ref as E
from tests.info_ref import information

U = 2.0 ** -24
ETA = 2.0 ** -148


def _per_sample(L, normalized):
    """float64 [S, B, C] p, lp and their relative / absolute fp32 error bounds e_p, e_lp, eta (see the module doc)."""
    C = L.shape[2]
    k = math.ceil(C / 32) + 5
    if normalized:
        sp = F.softplus(L)
        norm = sp.sum(2, keepdim=True)
        p = sp / norm
        lp = torch.where(L < -30, L, torch.log(sp)) - torch.log(norm)    # log softplus(l) = l below -30, past exp's range
        eta = ETA * torch.clamp(1.0 / norm, min=1.0)
        e_p = torch.full_like(L, U * (k + 20))
        e_lp = torch.where(torch.isfinite(lp), e_p + 2 * U * lp.abs() + U * L.abs(), torch.full_like(L, math.inf))
        return p, lp, e_p, e_lp, eta.expand_as(L)
    mx = L.amax(2, keepdim=True)
    se = torch.exp(L - mx).sum(2, keepdim=True)
    r = mx + torch.log(se)
    lp = L - r
    p = torch.exp(lp)
    ep_dist = torch.where(p > 0, p * (L - mx).abs(), torch.zeros_like(p)).sum(2, keepdim=True)
    e_lp = U * (r.abs() + lp.abs() + 2 * torch.log(se) + ep_dist + k + 9)
    fin = torch.isfinite(lp)
    return p, lp, torch.where(fin, e_lp + 4 * U, torch.zeros_like(L)), torch.where(fin, e_lp, torch.full_like(L, math.inf)), \
        torch.full_like(L, ETA)


def head(logits, labels, kl_terms, normalized=False, train_size=1.0, beta=0.0):
    """Every output of the exchange in float64 (see the module doc)."""
    L = torch.as_tensor(logits).double()
    p, lp, _, _, _ = _per_sample(L, normalized)
    pred, epi, ale, ent = O.uncertainty(list(L), normalized=normalized)
    ee, mi = information(list(L), normalized=normalized)
    lo = O.logmeanexp(lp.permute(1, 2, 0), 2)
    kl = float(torch.as_tensor(kl_terms).double().sum())
    out = {"lo": lo, "kl": kl, "pred": pred, "epi": epi, "ale": ale, "ent": ent, "ee": ee, "mi": mi}
    if labels is not None:
        y = torch.as_tensor(labels).long()
        nll = float(-lo.gather(1, y[:, None]).mean())
        acc = float((lo.argmax(1) == y).double().mean())
        out["head"] = [nll * train_size + beta * kl, nll, acc, beta * kl]
        out["sums"] = E.batch_sums(lo, y)
    return out


def bounds(logits, labels, kl_terms, n_loc, n_src, normalized=False, train_size=1.0, beta=0.0, ref=None):
    """Per-element error bounds of the fp32 outputs (module doc): a dict with the keys of head()."""
    L = torch.as_tensor(logits).double()
    S, B, C = L.shape
    k = math.ceil(C / 32) + 5
    ref = ref if ref is not None else head(L, labels, kl_terms, normalized, train_size, beta)
    p, lp, e_p, e_lp, eta = _per_sample(L, normalized)
    fin = torch.isfinite(lp)
    lo_b = torch.where(fin, e_lp, torch.zeros_like(e_lp)).amax(0) + U * (11 * (n_loc + n_src) + 4 + 2 * math.log(S)
                                                                       + ref["lo"].abs())
    labs = torch.where(torch.isfinite(L), L.abs(), torch.zeros_like(L))
    pred_b = U * (S + n_src + 1) * labs.mean(0) + U * torch.nan_to_num(ref["pred"].abs(), posinf=0.0)
    pmax = p.amax(0)
    delta = (e_p * p).amax(0) + 6 * U * (n_loc + n_src) * pmax + eta.amax(0)
    epi = ref["epi"]
    epi_b = (2 * (S + n_src) + 4) * U * epi + 2 * delta * epi.sqrt() + delta ** 2 + ETA
    pb = p.mean(0)
    ale_b = delta * (1 - 2 * pb).abs() + delta ** 2 + epi_b + U * (3 * pb * (1 - pb) + ref["ale"].abs())
    Lh = torch.log(torch.maximum(pb, delta).clamp_min(1e-300)).abs() + 1
    plogp = torch.where(pb > 0, pb * torch.log(pb.clamp_min(1e-300)).abs(), torch.zeros_like(pb))
    ent_b = (2 * delta * Lh).sum(1) + U * (k + 3) * plogp.sum(1)
    alp = torch.where(fin, lp.abs(), torch.zeros_like(lp))
    term = p * (alp + 1) * (e_p + 3 * U) + torch.where(p > 0, p * e_lp, torch.zeros_like(p)) + eta * (alp + 1)
    ee_b = term.sum(2).mean(0) + (n_loc * k + n_src + 7) * U * ref["ee"].abs()
    mi_b = ent_b + ee_b + U * ref["mi"].abs()
    kt = torch.as_tensor(kl_terms).double()
    kl_b = U * (kt.numel() + n_src + 3) * float(kt.abs().sum())
    out = {"lo": lo_b, "pred": pred_b, "epi": epi_b, "ale": ale_b, "ent": ent_b, "ee": ee_b, "mi": mi_b, "kl": kl_b}
    if labels is not None:
        y = torch.as_tensor(labels).long()
        nll = ref["head"][1]
        nll_b = float(lo_b.gather(1, y[:, None]).mean()) + U * abs(nll)
        out["nll"] = nll_b
        out["loss"] = train_size * nll_b + beta * kl_b + 3 * U * (train_size * abs(nll) + abs(beta * ref["kl"]))
        out["beta_kl"] = beta * kl_b + U * abs(beta * ref["kl"])
    return out

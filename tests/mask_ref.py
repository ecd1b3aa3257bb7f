"""float64 restatement of a Bayesian layer with a pruning mask (set_weight_mask), for its tests (not a test module itself).

A pruned element is a deterministic zero: BBB w = m ? mu + eps sigma : 0, LRT mean operand m ? mu : 0 and variance
operand m ? sigma^2 : 0.  Feeding the unmasked float64 references mu -> 0 and rho -> -inf at pruned elements states
exactly that, since log1p(exp(-inf)) = 0 in float64: the weight sample is 0 + eps * 0 = 0 and sigma^2 = 0, whatever the
pruned mu / rho held.  The KL has no such shortcut (log 0): ``kl_ref`` sums the terms of the kept elements only.
"""
import torch

from oracle import bbb_oracle as O
from tests import forward_ref as R


def masked_params(W_mu, W_rho, b_mu, b_rho, w_mask, b_mask=None):
    """float64 (W_mu, W_rho, b_mu, b_rho) with mu = 0 and rho = -inf at pruned elements (b_mask None: biases kept)."""
    d = lambda t: None if t is None else t.detach().double()
    W_mu, W_rho, b_mu, b_rho = d(W_mu), d(W_rho), d(b_mu), d(b_rho)
    w_mask = w_mask.to(W_mu.device)
    W_mu = W_mu.where(w_mask, 0.0)
    W_rho = W_rho.where(w_mask, float("-inf"))
    if b_mu is not None and b_mask is not None:
        b_mask = b_mask.to(b_mu.device)
        b_mu = b_mu.where(b_mask, 0.0)
        b_rho = b_rho.where(b_mask, float("-inf"))
    return W_mu, W_rho, b_mu, b_rho


def layer_ref(variant, x, W_mu, W_rho, b_mu, b_rho, w_mask, b_mask, eps, conv, sample=True, act="none"):
    """(ref, M, sd) of one masked layer call in float64: forward_ref.layer_ref on the masked parameters."""
    return R.layer_ref(variant, x, *masked_params(W_mu, W_rho, b_mu, b_rho, w_mask, b_mask), eps, conv, sample, act)


def kl_terms(mu, rho, pm, ps, convention="reference"):
    """float64 KL term of every element (the kernels' kl_term), against the scalar or element-wise prior (pm, ps)."""
    mu, rho = mu.detach().double(), rho.detach().double()
    pm = pm.detach().double() if torch.is_tensor(pm) else float(pm)
    ps = ps.detach().double() if torch.is_tensor(ps) else float(ps)
    s = O.softplus_sigma(rho)
    if convention == "reference":
        return 0.5 * (2.0 * torch.log(s / ps) - 1.0 + (ps / s) ** 2 + ((mu - pm) / s) ** 2)
    return torch.log(ps / s) + (s * s + (mu - pm) ** 2) / (2.0 * ps * ps) - 0.5


def kl_ref(W_mu, W_rho, b_mu, b_rho, w_mask, b_mask, pm, ps, convention="reference", prior=None):
    """float64 KL of a masked layer: the sum of the kept elements' terms (a pruned element's mu / rho are not read).
    ``prior``: None (the scalar pm, ps) or the tensor prior (w_mu, w_sigma, b_mu, b_sigma)."""
    wp = (pm, ps) if prior is None else (prior[0], prior[1])
    kl = kl_terms(W_mu, W_rho, *wp, convention)[w_mask.to(W_mu.device)].sum()
    if b_mu is not None:
        bp = (pm, ps) if prior is None else (prior[2], prior[3])
        t = kl_terms(b_mu, b_rho, *bp, convention)
        kl = kl + (t if b_mask is None else t[b_mask.to(b_mu.device)]).sum()
    return kl

"""float64 restatement of the Monte-Carlo KL against the scale-mixture prior (include/bbb_b200.h, bbb_kl_mc_forward):
the contract of the kernels, kept with the tests because the reference project has no such prior.

For q = N(mu, sigma^2), sigma = log1p(exp(rho)), the prior p(w) = pi N(0, sigma1^2) + (1 - pi) N(0, sigma2^2) and a
given standard normal eps per element:
    w    = mu + sigma eps
    term = -log sigma - 1/2 - logsumexp(log pi - log sigma1 - w^2 / (2 sigma1^2), log(1 - pi) - log sigma2 - w^2 / (2 sigma2^2))
"""
import math

import torch


def sigma_of(rho):
    return torch.log1p(torch.exp(rho))


def log_prior(w, pi, sigma1, sigma2):
    """log p(w) + 1/2 log 2 pi, element-wise (pi = 1: the slab alone)."""
    a = math.log(pi) - math.log(sigma1) - w * w / (2.0 * sigma1 ** 2)
    if pi >= 1.0:
        return a
    b = math.log1p(-pi) - math.log(sigma2) - w * w / (2.0 * sigma2 ** 2)
    return torch.logsumexp(torch.stack([a, b]), dim=0)


def kl_terms(mu, rho, eps, pi, sigma1, sigma2):
    """The per-element terms in float64 (differentiable in mu and rho)."""
    mu, rho, eps = mu.double(), rho.double(), eps.double()
    sg = sigma_of(rho)
    return -torch.log(sg) - 0.5 - log_prior(mu + sg * eps, pi, sigma1, sigma2)


def kl_mc(parts, pi, sigma1, sigma2):
    """One draw's KL of a layer: ``parts`` = [(mu, rho, eps), ...] (W, then the bias)."""
    return sum(kl_terms(m, r, e, pi, sigma1, sigma2).sum() for m, r, e in parts)


def kl_mc_grads(mu, rho, eps, pi, sigma1, sigma2):
    """(d/dmu, d/drho) of one draw's sum of terms, in closed form: responsibilities r1, r2 (softmax of the two logsumexp
    arguments), s = w (r1 / sigma1^2 + r2 / sigma2^2), d/dmu = s, d/dsigma = -1/sigma + s eps, d/drho = sigmoid(rho) d/dsigma."""
    mu, rho, eps = mu.double(), rho.double(), eps.double()
    sg = sigma_of(rho)
    w = mu + sg * eps
    a = math.log(pi) - math.log(sigma1) - w * w / (2.0 * sigma1 ** 2)
    if pi >= 1.0:
        r1, r2 = torch.ones_like(w), torch.zeros_like(w)
    else:
        b = math.log1p(-pi) - math.log(sigma2) - w * w / (2.0 * sigma2 ** 2)
        r1, r2 = torch.softmax(torch.stack([a, b]), dim=0)
    s = w * (r1 / sigma1 ** 2 + r2 / sigma2 ** 2)
    return s, torch.sigmoid(rho) * (-1.0 / sg + s * eps)


def draw_index(n_w, n, bias=False):
    """Which normal of the draw's Philox stream an element takes: element n of W takes n, bias element n takes |W| + n."""
    return n_w + n if bias else n


def gaussian_kl(mu, sigma, prior_sigma):
    """Textbook KL(N(mu, sigma^2) || N(0, prior_sigma^2)) per element: what pi = 1 converges to."""
    return math.log(prior_sigma / sigma) + (sigma ** 2 + mu ** 2) / (2.0 * prior_sigma ** 2) - 0.5

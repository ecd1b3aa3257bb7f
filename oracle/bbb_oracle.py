"""CPU oracle for the Bayes-by-Backprop layer hot path.  TEST INFRASTRUCTURE ONLY.

This file is a CPU restatement of the reference's algorithm
(kumar-shridhar/PyTorch-BayesianCNN) for the one path this repo accelerates:
BBBConv2d / BBBLinear forward (weight-space "BBB" and local-reparameterisation
"LRT" variants) plus the closed-form Gaussian KL, and the Monte-Carlo combine
that sits directly above it.  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may import it; the
product package never does.

Parity pin: the reference has NO golden vectors and its only test file does not
collect (SURVEY.md D4).  The oracle is therefore pinned against outputs of the
reference itself, run in the build container by ``tests/golden/make_golden.py``
(imports the original project unmodified, replays its CPU-generator eps draws) and
committed as ``tests/golden/*.npz``.  ``tests/test_oracle_golden.py`` checks the
oracle against those fixtures bit-for-bit in fp32.

The arithmetic the reference executes lives in PyTorch/ATen (oneDNN on CPU);
the restatement uses the same aten calls in the same order so that, given the
same eps, it is bitwise equal on the same torch build.  A float64 mode is
offered for tolerance budgeting.

Every function cites the reference file:line (relative to the original project's root).
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------- #
# elementwise pieces
# --------------------------------------------------------------------------- #
def softplus_sigma(rho: torch.Tensor) -> torch.Tensor:
    """sigma = log1p(exp(rho)) -- layers/BBB/BBBConv.py:64, BBB_LRT/BBBConv.py:64.

    NOT F.softplus: no threshold, overflows for rho > ~88 exactly like the
    reference (SURVEY.md H5).
    """
    return torch.log1p(torch.exp(rho))


def calculate_kl(mu_q, sig_q, mu_p, sig_p) -> torch.Tensor:
    """metrics.py:27-29, verbatim formula."""
    kl = 0.5 * (2 * torch.log(sig_p / sig_q) - 1 + (sig_q / sig_p).pow(2)
                + ((mu_p - mu_q) / sig_p).pow(2)).sum()
    return kl


def kl_loss(W_mu, W_rho, bias_mu, bias_rho, prior_mu, prior_sigma) -> torch.Tensor:
    """layer.kl_loss() -- layers/BBB/BBBConv.py:79-83 (same at BBBLinear.py:72-76,
    BBB_LRT/BBBConv.py:83-87, BBB_LRT/BBBLinear.py:75-79).

    Note the argument binding at the call site (SURVEY.md D1): the prior is
    passed as (mu_q, sig_q) and the learned posterior as (mu_p, sig_p), so the
    value is KL(prior || posterior).  Parity means reproducing that.
    """
    kl = calculate_kl(prior_mu, prior_sigma, W_mu, softplus_sigma(W_rho))
    if bias_mu is not None:
        kl = kl + calculate_kl(prior_mu, prior_sigma, bias_mu, softplus_sigma(bias_rho))
    return kl


def kl_textbook(W_mu, W_rho, bias_mu, bias_rho, prior_mu, prior_sigma) -> torch.Tensor:
    """Textbook KL(q||p), q = N(mu, sigma^2) posterior, p = prior.  No reference
    (opt-in convention only): log(sp/s) + (s^2 + (mu-mp)^2)/(2 sp^2) - 1/2."""
    def one(mu, rho):
        s = softplus_sigma(rho)
        return (torch.log(prior_sigma / s) + (s * s + (mu - prior_mu) ** 2)
                / (2.0 * prior_sigma * prior_sigma) - 0.5).sum()
    kl = one(W_mu, W_rho)
    if bias_mu is not None:
        kl = kl + one(bias_mu, bias_rho)
    return kl


# --------------------------------------------------------------------------- #
# layer forwards (eps supplied by the caller)
# --------------------------------------------------------------------------- #
def _contract(x, w, b, conv):
    if conv is None:
        return F.linear(x, w, b)
    stride, padding, dilation = conv
    return F.conv2d(x, w, b, stride, padding, dilation, 1)


def bbb_forward(x, W_mu, W_rho, bias_mu, bias_rho, W_eps, bias_eps, conv=None,
                sample=True) -> torch.Tensor:
    """Weight-space sampling forward.

    conv: layers/BBB/BBBConv.py:61-77; linear: layers/BBB/BBBLinear.py:54-70.
    W = mu + eps * log1p(exp(rho)); same for bias; one contraction.
    ``conv`` = (stride, padding, dilation) or None for the linear layer.
    """
    if sample:
        weight = W_mu + W_eps * softplus_sigma(W_rho)
        bias = None
        if bias_mu is not None:
            bias = bias_mu + bias_eps * softplus_sigma(bias_rho)
    else:
        weight, bias = W_mu, bias_mu
    return _contract(x, weight, bias, conv)


def lrt_forward(x, W_mu, W_rho, bias_mu, bias_rho, eps, conv=None, sample=True) -> torch.Tensor:
    """Local-reparameterisation forward.

    conv: layers/BBB_LRT/BBBConv.py:62-81; linear: layers/BBB_LRT/BBBLinear.py:56-73.
    act_mu = x (*) mu + b_mu ; act_var = 1e-16 + x^2 (*) sigma^2 + sigma_b^2 ;
    y = act_mu + sqrt(act_var) * eps, eps of the activation's shape.
    """
    W_sigma = softplus_sigma(W_rho)
    bias_var = None
    if bias_mu is not None:
        bias_var = softplus_sigma(bias_rho) ** 2
    act_mu = _contract(x, W_mu, bias_mu, conv)
    act_var = 1e-16 + _contract(x ** 2, W_sigma ** 2, bias_var, conv)
    act_std = torch.sqrt(act_var)
    if sample:
        return act_mu + act_std * eps
    return act_mu


def lrt_moments(x, W_mu, W_rho, bias_mu, bias_rho, conv=None):
    """(act_mu, act_var) of the LRT path -- BBB_LRT/BBBConv.py:71-74.  Used by the
    statistical tests: both variants share these first two moments."""
    W_sigma = softplus_sigma(W_rho)
    bias_var = softplus_sigma(bias_rho) ** 2 if bias_mu is not None else None
    return (_contract(x, W_mu, bias_mu, conv),
            1e-16 + _contract(x ** 2, W_sigma ** 2, bias_var, conv))


# --------------------------------------------------------------------------- #
# model-level restatement: the three reference architectures as data
# --------------------------------------------------------------------------- #
# (kind, args).  conv: (cin, cout, k, stride, pad); pool: (k, stride); fc: (in, out)
# BayesianAlexNet.py:34-53 / BayesianLeNet.py:34-49 / Bayesian3Conv3FC.py:36-55
def arch(name: str, outputs: int, inputs: int):
    if name == "alexnet":
        return [("conv", (inputs, 64, 11, 4, 5)), ("act",), ("pool", (2, 2)),
                ("conv", (64, 192, 5, 1, 2)), ("act",), ("pool", (2, 2)),
                ("conv", (192, 384, 3, 1, 1)), ("act",),
                ("conv", (384, 256, 3, 1, 1)), ("act",),
                ("conv", (256, 128, 3, 1, 1)), ("act",), ("pool", (2, 2)),
                ("flatten", 128), ("fc", (128, outputs))]
    if name == "lenet":
        return [("conv", (inputs, 6, 5, 1, 0)), ("act",), ("pool", (2, 2)),
                ("conv", (6, 16, 5, 1, 0)), ("act",), ("pool", (2, 2)),
                ("flatten", 400), ("fc", (400, 120)), ("act",),
                ("fc", (120, 84)), ("act",), ("fc", (84, outputs))]
    if name == "3conv3fc":
        return [("conv", (inputs, 32, 5, 1, 2)), ("act",), ("pool", (3, 2)),
                ("conv", (32, 64, 5, 1, 2)), ("act",), ("pool", (3, 2)),
                ("conv", (64, 128, 5, 1, 1)), ("act",), ("pool", (3, 2)),
                ("flatten", 512), ("fc", (512, 1000)), ("act",),
                ("fc", (1000, 1000)), ("act",), ("fc", (1000, outputs))]
    raise ValueError(name)


def init_params(name, outputs, inputs, priors, seed, dtype=torch.float32):
    """Draw parameters the way reset_parameters does (BBB/BBBConv.py:53-59): per
    Bayesian layer, in order, W_mu, W_rho, bias_mu, bias_rho ~ normal_(mean, std)
    from the CPU generator.  Returns a list of dicts (one per Bayesian layer)."""
    g = torch.Generator().manual_seed(seed)
    mu0, rho0 = priors["posterior_mu_initial"], priors["posterior_rho_initial"]
    out = []
    for item in arch(name, outputs, inputs):
        if item[0] == "conv":
            cin, cout, k, _, _ = item[1]
            shape = (cout, cin, k, k)
        elif item[0] == "fc":
            shape = (item[1][1], item[1][0])
        else:
            continue
        p = {
            "W_mu": torch.empty(shape).normal_(*mu0, generator=g),
            "W_rho": torch.empty(shape).normal_(*rho0, generator=g),
            "bias_mu": torch.empty(shape[0]).normal_(*mu0, generator=g),
            "bias_rho": torch.empty(shape[0]).normal_(*rho0, generator=g),
        }
        out.append({k_: v.to(dtype) for k_, v in p.items()})
    return out


def eps_shapes(name, outputs, inputs, variant, batch, hw=32):
    """Shapes of the eps tensors one net(x) draws, in the reference's draw order
    (SURVEY.md 8c): BBB -> (W_eps, bias_eps) per layer; LRT -> one activation
    shaped eps per layer."""
    shapes = []
    h = w = hw
    c = inputs
    rows = batch
    for item in arch(name, outputs, inputs):
        if item[0] == "conv":
            cin, cout, k, s, p = item[1]
            h = (h + 2 * p - k) // s + 1
            w = (w + 2 * p - k) // s + 1
            c = cout
            if variant == "bbb":
                shapes += [(cout, cin, k, k), (cout,)]
            else:
                shapes += [(batch, cout, h, w)]
        elif item[0] == "pool":
            k, s = item[1]
            h = (h - k) // s + 1
            w = (w - k) // s + 1
        elif item[0] == "flatten":
            rows = batch * c * h * w // item[1]     # view(-1, F), layers/misc.py:35
        elif item[0] == "fc":
            fin, fout = item[1]
            if variant == "bbb":
                shapes += [(fout, fin), (fout,)]
            else:
                shapes += [(rows, fout)]
    return shapes


def draw_eps_like_reference(shapes: Sequence[tuple], seed: int):
    """Seed-replay of the reference's noise: ``torch.manual_seed(seed)`` then
    ``torch.empty(shape).normal_(0, 1)`` per tensor in draw order
    (layers/BBB/BBBConv.py:63,68; BBB_LRT/BBBConv.py:78).  Uses the GLOBAL CPU
    generator exactly as the reference does."""
    torch.manual_seed(seed)
    return [torch.empty(s).normal_(0, 1) for s in shapes]


def net_forward(name, params, x, eps_list, variant, activation="softplus",
                prior_mu=0.0, prior_sigma=0.1, outputs=10, sample=True):
    """ModuleWrapper.forward (layers/misc.py:16-25) over one of the three model
    files: children in order, then kl = 0.0 + sum of kl_loss().  Returns
    (logits, kl)."""
    act = F.softplus if activation == "softplus" else F.relu
    inputs = x.shape[1]
    it = iter(eps_list)
    li = 0
    kl = 0.0
    for item in arch(name, outputs, inputs):
        kind = item[0]
        if kind in ("conv", "fc"):
            p = params[li]
            li += 1
            conv = None
            if kind == "conv":
                _, _, _, s, pad = item[1]
                conv = (s, pad, 1)
            if variant == "bbb":
                we = next(it) if sample else None
                be = next(it) if sample else None
                x = bbb_forward(x, p["W_mu"], p["W_rho"], p["bias_mu"], p["bias_rho"],
                                we, be, conv, sample)
            else:
                e = next(it) if sample else None
                x = lrt_forward(x, p["W_mu"], p["W_rho"], p["bias_mu"], p["bias_rho"],
                                e, conv, sample)
            kl = kl + kl_loss(p["W_mu"], p["W_rho"], p["bias_mu"], p["bias_rho"],
                              prior_mu, prior_sigma)
        elif kind == "act":
            x = act(x)
        elif kind == "pool":
            x = F.max_pool2d(x, item[1][0], item[1][1])
        elif kind == "flatten":
            x = x.view(-1, item[1])        # layers/misc.py:35 (no shape check, D2)
    return x, kl


# --------------------------------------------------------------------------- #
# what sits directly above the path: MC combine and uncertainty reductions
# --------------------------------------------------------------------------- #
def logmeanexp(x, dim):
    """utils.py:14-22."""
    x_max, _ = torch.max(x, dim, keepdim=True)
    x = x_max + torch.log(torch.mean(torch.exp(x - x_max), dim, keepdim=True))
    return x.squeeze(dim)


def mc_combine(logits_per_sample: Sequence[torch.Tensor]) -> torch.Tensor:
    """main_bayesian.py:46-53: outputs[:,:,j] = log_softmax(net_out); logmeanexp over j."""
    outs = torch.stack([F.log_softmax(l, dim=1) for l in logits_per_sample], dim=2)
    return logmeanexp(outs, 2)


def uncertainty(logits_per_sample: Sequence[torch.Tensor], normalized=False):
    """uncertainty_estimation.py:70-96 restated without the per-image python loop:
    pred = mean_t logits (:82-83); p_hat = softmax (or softplus-normalised :73-77);
    epistemic = diag((p_hat-p_bar)^T (p_hat-p_bar))/T (:89-91);
    aleatoric = diag(diag(p_bar) - p_hat^T p_hat / T) (:94-95).
    Also returns H[p_bar] (predictive entropy; NO reference -- SURVEY.md D3)."""
    L = torch.stack(list(logits_per_sample), 0).double()         # [T,B,C]
    if normalized:
        pr = F.softplus(L)
        p_hat = pr / pr.sum(2, keepdim=True)
    else:
        p_hat = F.softmax(L, dim=2)
    p_bar = p_hat.mean(0)
    epistemic = ((p_hat - p_bar) ** 2).mean(0)
    aleatoric = p_bar - (p_hat ** 2).mean(0)
    entropy = -(p_bar * torch.log(p_bar.clamp_min(1e-300))).sum(1)
    return L.mean(0), epistemic, aleatoric, entropy


# --------------------------------------------------------------------------- #
# Philox4x32-10 + Box-Muller: host restatement of the engine's in-kernel noise
# (csrc/philox.cuh).  Integer stream is bit-exact; normals agree to ~1e-5 abs
# (the device uses __logf/__sincosf).
# --------------------------------------------------------------------------- #
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)


def philox4x32_10(ctr: np.ndarray, key: np.ndarray) -> np.ndarray:
    """ctr: [n,4] uint32, key: [2] uint32 -> [n,4] uint32 (Salmon et al. 2011)."""
    c = ctr.astype(np.uint32).copy()
    k0, k1 = np.uint32(key[0]), np.uint32(key[1])
    mask = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0 = _M0 * c[:, 0].astype(np.uint64)
        p1 = _M1 * c[:, 2].astype(np.uint64)
        hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & mask).astype(np.uint32)
        hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & mask).astype(np.uint32)
        c = np.stack([hi1 ^ c[:, 1] ^ k0, lo1, hi0 ^ c[:, 3] ^ k1, lo0], axis=1)
        with np.errstate(over="ignore"):
            k0 = np.uint32(k0 + _W0)
            k1 = np.uint32(k1 + _W1)
    return c


def philox_normal(n: int, seed: int, stream: int, offset: int = 0) -> np.ndarray:
    """Element i (global index offset+i) = Box-Muller lane (i&3) of
    Philox(counter=(i>>2 lo, i>>2 hi, stream lo, stream hi), key=(seed lo, seed hi))."""
    idx = np.arange(offset, offset + n, dtype=np.uint64)
    grp = idx >> np.uint64(2)
    ctr = np.stack([(grp & np.uint64(0xFFFFFFFF)).astype(np.uint32),
                    (grp >> np.uint64(32)).astype(np.uint32),
                    np.full(n, stream & 0xFFFFFFFF, np.uint32),
                    np.full(n, (stream >> 32) & 0xFFFFFFFF, np.uint32)], axis=1)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], np.uint32)
    r = philox4x32_10(ctr, key)
    lane = (idx & np.uint64(3)).astype(np.int64)
    pair = lane >> 1
    a = np.where(pair == 0, r[:, 0], r[:, 2])
    b = np.where(pair == 0, r[:, 1], r[:, 3])
    u1 = ((a >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)
          + np.float32(2.0 ** -25)).astype(np.float32)
    u2 = ((b >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)
          + np.float32(2.0 ** -25)).astype(np.float32)
    rad = np.sqrt(np.float32(-2.0) * np.log(u1)).astype(np.float32)
    th = (np.float32(2.0 * math.pi) * u2).astype(np.float32)
    z = np.where((lane & 1) == 0, rad * np.cos(th), rad * np.sin(th))
    return z.astype(np.float32)

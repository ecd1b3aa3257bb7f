"""Plain restatements of the Bayesian layer backward, for its tests (not a test module itself).

- ``grads``: the gradients of x, W_mu, W_rho, bias_mu and bias_rho of the loss (y * gout).sum(), by torch autograd
  through oracle.bbb_forward / lrt_forward in float64 (no KL term).
- ``bounds``: the same function on (|x|, |W_mu|, W_rho, |bias_mu|, bias_rho, |eps|, |gout|).  Every term of every
  gradient is a product of these factors (BBB: |W| <= |mu| + |eps| sigma; LRT: act_std depends only on x^2 and sigma),
  so this is, element by element, the sum M of the absolute values of the terms that make up the gradient.  A kernel
  whose operands are rounded with unit roundoff u and which sums in fp32 is then off by at most a few u times M.
- ``round_bf16`` / ``round_tf32``: the operand rounding of the tensor-core layer kernel (fwd_tc.cuh, pack_chunk).
- ``CASES``: the layer geometries the three models train with, and the edge cases of the tensor-core backward
  (functional._tc_wgrad / _tc_dgrad), each with the reason it is in the table.
- ``contractions``: the contraction shapes the tensor-core backward of a case issues, recorded without computing.
"""
import collections
import contextlib

import torch
import torch.nn.functional as F

from oracle import bbb_oracle as O


# ---------------------------------------------------------------------------------------------------------------- #
# operand rounding
# ---------------------------------------------------------------------------------------------------------------- #
def round_bf16(t):
    """fp32, then bf16 round-to-nearest-even (__floats2bfloat162_rn); returned as float64."""
    return t.float().to(torch.bfloat16).double()


def round_tf32(t):
    """fp32, then tf32 round-to-nearest with ties away from zero (cvt.rna.tf32.f32): on the fp32 bits,
    (u + 0x1000) & ~0x1fff; returned as float64."""
    u = t.float().contiguous().view(torch.int32)
    r = (u + 0x1000) & ~0x1FFF
    return r.view(torch.float32).double()


ROUND = {"bf16": round_bf16, "tf32": round_tf32}


def contract(x, w, conv):
    """The plain contraction functional._tc_contract computes: conv2d with ((sh, sw), (ph, pw), (dh, dw)), or linear."""
    return O._contract(x, w, None, conv)


# ---------------------------------------------------------------------------------------------------------------- #
# float64 reference gradients and their magnitudes
# ---------------------------------------------------------------------------------------------------------------- #
def grads(variant, x, W_mu, W_rho, bias_mu, bias_rho, eps, gout, conv=None, sample=True):
    """[gx, gW_mu, gW_rho, gbias_mu, gbias_rho] of (y * gout).sum() in float64 (bias entries None without a bias; a
    parameter the output does not depend on, e.g. W_rho with sample=False, gets zeros).  ``eps``: BBB (W_eps, bias_eps),
    LRT the activation-shaped eps (ignored when not sampling)."""
    ins = [t.detach().double().clone().requires_grad_(True) if t is not None else None
           for t in (x, W_mu, W_rho, bias_mu, bias_rho)]
    if variant == "bbb":
        we, be = eps if sample else (None, None)
        y = O.bbb_forward(ins[0], *ins[1:], None if we is None else we.double(),
                          None if be is None else be.double(), conv, sample)
    else:
        y = O.lrt_forward(ins[0], *ins[1:], None if not sample else eps.double(), conv, sample)
    (y * gout.double()).sum().backward()
    return [None if t is None else (t.grad if t.grad is not None else torch.zeros_like(t)) for t in ins]


def bounds(variant, x, W_mu, W_rho, bias_mu, bias_rho, eps, gout, conv=None, sample=True):
    """Element by element, the sum of the absolute values of the terms of each gradient (see the module docstring)."""
    ab = lambda t: None if t is None else t.abs()
    if variant == "bbb":
        e = (ab(eps[0]), ab(eps[1])) if sample else (None, None)
    else:
        e = ab(eps) if sample else None
    return grads(variant, x.abs(), W_mu.abs(), W_rho, ab(bias_mu), bias_rho, e, gout.abs(), conv, sample)


# ---------------------------------------------------------------------------------------------------------------- #
# the case table
# ---------------------------------------------------------------------------------------------------------------- #
Case = collections.namedtuple("Case", "name why cin cout k s p d hw B fallback")


def _c(name, why, cin, cout, k=None, s=1, p=0, d=1, hw=None, B=1, fallback=None):
    """k = None: a linear layer of cin -> cout.  Otherwise k, s, p, d are ints or (h, w) pairs and hw = (H, W).
    fallback: None (the tensor-core backward runs), "wgrad" (a wgrad contraction is refused) or "dgrad" (_tc_dgrad
    returns None); either way the layer then runs on the CUDA-core kernels."""
    pair = lambda v: tuple(v) if isinstance(v, (tuple, list)) else (v, v)
    if k is None:
        return Case(name, why, cin, cout, None, None, None, None, None, B, fallback)
    return Case(name, why, cin, cout, pair(k), pair(s), pair(p), pair(d), pair(hw), B, fallback)


def _model(prefix, why, layers, B):
    out = []
    for (tag, cin, cout, k, s, p, hw) in layers:
        out.append(_c(f"{prefix}_{tag}_b{B}", f"{why}: {tag}", cin, cout, k, s, p, 1, hw, B))
    return out


_ALEXNET = [("conv1", 3, 64, 11, 4, 5, 32), ("conv2", 64, 192, 5, 1, 2, 4), ("conv3", 192, 384, 3, 1, 1, 2),
            ("conv4", 384, 256, 3, 1, 1, 2), ("conv5", 256, 128, 3, 1, 1, 2), ("fc", 128, 10, None, 1, 0, None)]
_LENET = [("conv1", 3, 6, 5, 1, 0, 32), ("conv2", 6, 16, 5, 1, 0, 14), ("fc1", 400, 120, None, 1, 0, None),
          ("fc2", 120, 84, None, 1, 0, None), ("fc3", 84, 10, None, 1, 0, None)]
_3CONV3FC = [("conv1", 1, 32, 5, 1, 2, 32), ("conv2", 32, 64, 5, 1, 2, 15), ("conv3", 64, 128, 5, 1, 1, 7),
             ("fc1", 512, 1000, None, 1, 0, None), ("fc2", 1000, 1000, None, 1, 0, None),
             ("fc3", 1000, 10, None, 1, 0, None)]

CASES = (
    _model("alexnet", "BBBAlexNet at the benchmark batch; conv1 wgrad is 4 chunks of K = 8192", _ALEXNET, 512)
    + _model("alexnet", "BBBAlexNet, ragged last wgrad chunk (conv1: 7 x 128 + 104 images, conv2: 512 + 488)",
             _ALEXNET, 1000)
    + _model("lenet", "BBBLeNet; conv1 wgrad in 26 chunks of 10 images (the last 6)", _LENET, 256)
    + _model("3conv3fc", "BBB3Conv3FC: 15x15 and 7x7 maps, N = 1000, conv1 wgrad 38 chunks (the last 4 images)",
             _3CONV3FC, 300)
    + [
        _c("edge_k2s3", "stride 3 > kernel 2: input pixels no output reads get no gradient; zero insertion",
           5, 7, 2, 3, 0, 1, (11, 10), 4),
        _c("edge_rect_asym", "3x2 kernel, stride (2, 1), padding (1, 2), dilation (1, 2): every axis differs",
           6, 5, (3, 2), (2, 1), (1, 2), (1, 2), (9, 8), 3),
        _c("edge_k4x2_s3_d2", "4x2 kernel, stride 3, dilation 2, padding (2, 1)", 4, 9, (4, 2), 3, (2, 1), 2, (13, 11), 5),
        _c("edge_1x1_p1", "1x1 conv with padding 1: pad > dil*(k-1), _tc_dgrad returns None", 8, 4, 1, 1, 1, 1, (6, 6), 2,
           fallback="dgrad"),
        _c("edge_1x1_130", "1x1 conv on 130x130: OH*OW = 16900 > 16384, the wgrad contraction is refused",
           4, 3, 1, 1, 0, 1, (130, 130), 2, fallback="wgrad"),
        _c("edge_lin_b16384", "linear wgrad with the batch as K = 16384: the largest accepted", 24, 5, B=16384),
        _c("edge_lin_b16385", "linear wgrad with K = 16385: refused", 24, 5, B=16385, fallback="wgrad"),
        _c("edge_conv_b1", "a single image", 16, 24, 3, 1, 1, 1, (5, 5), 1),
        _c("edge_lin_b1", "a single row", 100, 70, B=1),
        _c("edge_cout1", "Cout = 1: one output channel, dgrad with N = 1", 3, 1, 3, 1, 1, 1, (7, 7), 5),
        _c("edge_lin_k100_n70", "K = 100 and N = 70: neither a multiple of the 64-wide (bf16) or 32-wide (tf32) K block "
           "nor of the 64-column tile", 100, 70, B=33),
        _c("edge_conv_k45", "K = 5*3*3 = 45 < 64 with stride 2 on a non-square map", 5, 7, 3, 2, 1, 1, (9, 8), 6),
    ]
)
assert len({c.name for c in CASES}) == len(CASES)


def conv_of(cs):
    """The ((sh, sw), (ph, pw), (dh, dw)) geometry of a case, None for a linear layer."""
    return None if cs.k is None else (cs.s, cs.p, cs.d)


def x_shape(cs):
    return (cs.B, cs.cin) if cs.k is None else (cs.B, cs.cin) + cs.hw


def w_shape(cs):
    return (cs.cout, cs.cin) if cs.k is None else (cs.cout, cs.cin) + cs.k


def y_shape(cs):
    if cs.k is None:
        return (cs.B, cs.cout)
    (sh, sw), (ph, pw), (dh, dw) = conv_of(cs)
    oh = (cs.hw[0] + 2 * ph - dh * (cs.k[0] - 1) - 1) // sh + 1
    ow = (cs.hw[1] + 2 * pw - dw * (cs.k[1] - 1) - 1) // sw + 1
    return (cs.B, cs.cout, oh, ow)


@contextlib.contextmanager
def contract_with(fn):
    """functional._tc_contract replaced by fn(x, w, conv) inside the block."""
    from pytorch_bayesiancnn_b200 import functional as Fn
    prev = Fn._tc_contract
    Fn._tc_contract = fn
    try:
        yield
    finally:
        Fn._tc_contract = prev


def contractions(cs):
    """(role, x shape, w shape, conv) of every contraction _tc_wgrad and _tc_dgrad issue for the case, in order, and
    whether _tc_dgrad gave up (returned None).  Shapes are recorded on the meta device: nothing is computed."""
    from pytorch_bayesiancnn_b200 import functional as Fn
    calls = []
    role = [None]

    def rec(x, w, conv):
        calls.append((role[0], tuple(x.shape), tuple(w.shape), conv))
        return contract(x, w, conv)

    conv = conv_of(cs)
    x = torch.empty(x_shape(cs), device="meta")
    g = torch.empty(y_shape(cs), device="meta")
    w = torch.empty(w_shape(cs), device="meta")
    with contract_with(rec):
        role[0] = "wgrad"
        Fn._tc_wgrad(x, g, conv, w.shape)
        role[0] = "dgrad"
        dg = Fn._tc_dgrad(g, w, conv, x.shape)
    return calls, dg is None

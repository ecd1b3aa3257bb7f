"""Plain restatements of the per-layer Bayesian forward (bbb_conv2d_forward / bbb_linear_forward), for its tests (not a
test module itself).

- ``layer_ref``: one layer call, BBB or LRT, in float64 (oracle.bbb_forward / lrt_forward), with the magnitude ``M``,
  the element-wise sum of the absolute values of its terms, sum|x||w| + |b| + sd |eps| (BBB: w = mu + eps sigma,
  b = b_mu + eps_b sigma_b), and the float64 LRT ``sd`` = sqrt(x^2 (*) sigma^2 + sigma_b^2 + 1e-16).
- ``mean_ref``: the mean path (sample = 0) on x and W_mu rounded as the kernel rounds them (backward_ref.ROUND).
- ``var_plane_err``: the LRT variance plane on inputs whose squares are exact (``var_x``).
- ``tc_launch`` / ``simt_config``: the launch decisions of fwd_tc.cuh (launch_fwd_tc_t) and fwd_simt.cuh
  (launch_fwd_simt), restated on the host.
- ``CASES``: every per-layer geometry of the three models, the Monte-Carlo fold shapes, and the edges of both kernels,
  each with the reason it is in the table.

Error bounds.  Let u be the unit roundoff of the operands: bf16 2^-8, tf32 2^-11 (fp32 2^-24).

Tight tier, |got - ref| <= TIGHT * M with TIGHT = 1e-4.  When the reference is computed on the operands exactly as the
kernel multiplies them, all that separates the two is fp32 accumulation over K terms: about sqrt(K) 2^-24 M for
random signs, 2e-6 M at K = 16384.  Two forms:
  - the mean path (sample = 0) on x and W_mu rounded like pack_chunk (bf16 round-to-nearest-even, tf32 cvt.rna) and
    the fp32 bias;
  - the LRT variance plane on x with at most 4 significant bits, so that x^2 (8 bits) is exact in bf16 and tf32 however
    the kernel forms it (from fp32 x, or from the bf16-staged x of stage_x == 2), and W_rho constant in each output
    channel, with no bias.  Then act_std^2 - 1e-16 = c_n sum_k x_k^2 with one constant c_n per channel: the ratio must
    be the same at every (image, pixel) to TIGHT, and c_n must equal the rounding of sigma_n^2 -- or of a value within
    1e-6 of it: the kernel rounds its own fp32 sigma^2, which may land on the neighbouring grid point when sigma_n^2
    lies near a rounding boundary -- to TIGHT plus acc_bias(K), the worst bias of an fp32 sum of K positive terms
    (wgmma accumulation truncates: on an H100 the variance plane of a tf32 call at K = 16384 came out 1.5e-4 low in
    every output alike).  This is stronger than "c_n within 2u of the rounded sigma_n^2".
A dropped or doubled K block moves an element by the block's share of M (64/K, 6e-3 at K = 16384 with 64-wide
blocks), a swapped tap, a wrong im2col offset or a wrong staged image by a sizeable fraction: all far outside 1e-4.

Loose tier, |got - ref| <= C (M + |ref|), the full sampled layer against float64 on the unrounded operands.  A product
of two rounded operands is off by <= 2u relative; BBB rounds W = mu + eps sigma (formed in fp32) once and x once; LRT
rounds x and W_mu for the mean, and x^2 (u, or 3u when x^2 is formed from the bf16-staged x) and sigma^2 (u) for the
variance, so sd is off by <= 2u relative and sd |eps| by <= 2u sd |eps|.  Summed: <= 2u M, so C = 2u: 2^-7 (bf16),
2^-10 (tf32).  fp32 has no operand rounding; C_FP32 = 1e-5 covers fp32 accumulation and the fp32 softplus / sqrt.
act_std (LRT, sampling) must be within STD_C sd of the float64 sd, STD_C = 2u by the same count.
"""
import collections

import numpy as np
import torch
import torch.nn.functional as F

from oracle import bbb_oracle as O
from tests.backward_ref import ROUND, round_bf16, round_tf32  # noqa: F401  (re-exported for the tests)

TIGHT = 1e-4
U = {"bf16": 2.0 ** -8, "tf32": 2.0 ** -11, "fp32": 2.0 ** -24}
C = {"bf16": 2.0 ** -7, "tf32": 2.0 ** -10, "fp32": 1e-5}
STD_C = C
MATHS = ("fp32", "tf32", "bf16")
FOLD_STRIDE = 1 << 40           # the Philox stream stride of the MC folds of one rank (mc.MCForward / MCTrainStep)


def contract(x, w, b, conv):
    return O._contract(x, w, b, conv)


def apply_act(y, act):
    if act == "relu":
        return torch.relu(y)
    if act == "softplus":
        return F.softplus(y)                # nn.Softplus(beta=1, threshold=20)
    assert act in (None, "none")
    return y


def _d(t):
    return None if t is None else t.double()


# ---------------------------------------------------------------------------------------------------------------- #
# float64 references
# ---------------------------------------------------------------------------------------------------------------- #
def layer_ref(variant, x, W_mu, W_rho, b_mu, b_rho, eps, conv, sample=True, act="none"):
    """(ref, M, sd) of one layer call in float64.  ``eps``: BBB (W_eps, bias_eps or None), LRT the activation-shaped eps
    (NCHW, or [B, N]); ignored when not sampling.  sd: the LRT sd when sampling, else None."""
    x, W_mu, W_rho, b_mu, b_rho = (_d(t) for t in (x, W_mu, W_rho, b_mu, b_rho))
    sd = None
    if variant == "bbb":
        we, be = (eps[0].double(), _d(eps[1])) if sample else (None, None)
        ref = O.bbb_forward(x, W_mu, W_rho, b_mu, b_rho, we, be, conv, sample)
        if sample:
            W = W_mu + we * O.softplus_sigma(W_rho)
            b = None if b_mu is None else b_mu + be * O.softplus_sigma(b_rho)
        else:
            W, b = W_mu, b_mu
        M = contract(x.abs(), W.abs(), None if b is None else b.abs(), conv)
    else:
        e = eps.double() if sample else None
        ref = O.lrt_forward(x, W_mu, W_rho, b_mu, b_rho, e, conv, sample)
        M = contract(x.abs(), W_mu.abs(), None if b_mu is None else b_mu.abs(), conv)
        if sample:
            sd = torch.sqrt(O.lrt_moments(x, W_mu, W_rho, b_mu, b_rho, conv)[1])
            M = M + sd * e.abs()
    return apply_act(ref, act), M, sd


def mean_ref(x, W_mu, b_mu, conv, math, act="none"):
    """(ref, M) of the mean path (sample = 0) on x and W_mu rounded as the kernel rounds them; fp32: unrounded."""
    r = ROUND.get(math, lambda t: t.double())
    xr, wr, b = r(x), r(W_mu), _d(b_mu)
    ref = contract(xr, wr, b, conv)
    M = contract(xr.abs(), wr.abs(), None if b is None else b.abs(), conv)
    return apply_act(ref, act), M


def var_x(shape, g, device="cpu"):
    """Random values with at most 4 significant bits (m / 8 * 2^e, m in 8..15, e in -3..2, random sign): their squares
    have at most 8 and are exact in bf16 and tf32."""
    m = torch.randint(8, 16, shape, generator=g, device=device).double() / 8
    e = torch.randint(-3, 3, shape, generator=g, device=device).double()
    s = torch.randint(0, 2, shape, generator=g, device=device).double() * 2 - 1
    return (s * m * torch.exp2(e)).float()


SIGMA_REL = 1e-6       # how far the kernels' fp32 sigma^2 (log1pf of __expf or expf, squared) may lie from float64


def acc_bias(K, math):
    """Worst relative bias of an fp32 sum of K positive terms, as the kernels accumulate it: one truncation (< 2^-23
    relative) per wgmma step of 16 bf16 / 8 tf32 terms, one rounding (<= 2^-24) per fma on fp32.  Errors of that size
    are common to every output of a channel, so they shift c_n but not the spread."""
    steps, ulp = {"bf16": (16, 2.0 ** -23), "tf32": (8, 2.0 ** -23), "fp32": (1, 2.0 ** -24)}[math]
    return (K + steps - 1) // steps * ulp


def var_plane_err(act_std, x, W_rho, conv, math):
    """(spread, c_err) of the LRT variance plane of a call on ``var_x`` inputs with W_rho constant per output channel and
    no bias, both normalised so that <= 1 passes.  spread = worst |r - c_n| / (TIGHT c_n) of r = (act_std^2 - 1e-16) /
    sum_k x_k^2 over every (image, pixel) with a nonzero receptive field, c_n the median of r in channel n.  c_err: c_n
    must be, to TIGHT + acc_bias(K), what the operand rounding R makes of some value within SIGMA_REL of sigma_n^2:
    either neighbour on the bf16 / tf32 grid when sigma_n^2 lies that close to a rounding boundary (so c_n is within 2u
    of R(sigma_n^2)), sigma_n^2 itself on fp32."""
    x = x.double()
    N = W_rho.shape[0]
    ones = torch.ones(W_rho.shape, dtype=torch.float64, device=x.device)
    xsq = contract(x * x, ones, None, conv)                       # sum of x_k^2 over the receptive field
    v = act_std.double() ** 2 - 1e-16
    shape = (xsq.shape[0], N, -1)
    xsq, v = xsq.reshape(shape).transpose(0, 1).reshape(N, -1), v.reshape(shape).transpose(0, 1).reshape(N, -1)
    sig2 = O.softplus_sigma(W_rho.double().reshape(N, -1)[:, 0]) ** 2
    r_ = ROUND.get(math, lambda t: t)
    cands = (r_(sig2 * (1 - SIGMA_REL)), r_(sig2), r_(sig2 * (1 + SIGMA_REL)))
    bar_c = TIGHT + acc_bias(W_rho[0].numel(), math)
    spread, c_err = 0.0, 0.0
    for n in range(N):
        live = xsq[n] > 0
        if not bool(live.any()):
            continue
        r = v[n][live] / xsq[n][live]
        c = r.median()
        spread = max(spread, float(torch.nan_to_num((r - c).abs().max() / (TIGHT * c), nan=float("inf"))))
        c_err = max(c_err, min(float((c - cd[n]).abs() / (bar_c * cd[n])) for cd in cands))
    return spread, c_err


# ---------------------------------------------------------------------------------------------------------------- #
# normalised errors: <= 1 passes; a NaN counts as inf; where the bound is 0 the output must be exactly 0
# ---------------------------------------------------------------------------------------------------------------- #
def _norm(got, ref, bound):
    got, ref, bound = got.double(), ref.double(), bound.double()
    zero = bound == 0
    if bool(zero.any()) and not bool((got[zero] == 0).all()):
        return float("inf")
    e = (got - ref).abs() / torch.where(zero, torch.ones_like(bound), bound)
    e = torch.where(zero, torch.zeros_like(e), torch.nan_to_num(e, nan=float("inf")))
    return float(e.max()) if e.numel() else 0.0


def tight_err(got, ref, M):
    return _norm(got, ref, TIGHT * M.double())


def loose_err(got, ref, M, math):
    return _norm(got, ref, C[math] * (M.double() + ref.double().abs()))


def std_err(got, sd, math):
    return _norm(got, sd, STD_C[math] * sd.double())


# ---------------------------------------------------------------------------------------------------------------- #
# the case table
# ---------------------------------------------------------------------------------------------------------------- #
Case = collections.namedtuple("Case", "name why cin cout k s p d hw B bias variants refuse act kl sparse fold extra")


def _c(name, why, cin, cout, k=None, s=1, p=0, d=1, hw=None, B=1, bias=True, variants=("bbb", "lrt"), refuse=(),
       act="none", kl="reference", sparse=False, fold=None, extra=()):
    """k = None: a linear layer of cin -> cout.  Otherwise k, s, p, d are ints or (h, w) pairs and hw = (H, W).
    refuse: the math modes bbb_forward_supported refuses (auto then resolves to fp32 if bf16 is refused, else bf16).
    sparse: x >= 0 with half the images and the top half of every map zero (zero receptive fields), no bias.
    fold: (rows per MC sample, first image): B = rows x samples, Philox stream stride FOLD_STRIDE.
    extra: images that must be among those checked against float64 (large cases check a subset)."""
    pair = lambda v: tuple(v) if isinstance(v, (tuple, list)) else (v, v)
    if sparse:
        bias = False
    if k is None:
        return Case(name, why, cin, cout, None, None, None, None, None, B, bias, tuple(variants), tuple(refuse), act, kl,
                    sparse, fold, tuple(extra))
    return Case(name, why, cin, cout, pair(k), pair(s), pair(p), pair(d), pair(hw), B, bias, tuple(variants),
                tuple(refuse), act, kl, sparse, fold, tuple(extra))


_ALEXNET = [("conv1", 3, 64, 11, 4, 5, 32), ("conv2", 64, 192, 5, 1, 2, 4), ("conv3", 192, 384, 3, 1, 1, 2),
            ("conv4", 384, 256, 3, 1, 1, 2), ("conv5", 256, 128, 3, 1, 1, 2), ("fc", 128, 10, None, 1, 0, None)]
_LENET = [("conv1", 3, 6, 5, 1, 0, 32), ("conv2", 6, 16, 5, 1, 0, 14), ("fc1", 400, 120, None, 1, 0, None),
          ("fc2", 120, 84, None, 1, 0, None), ("fc3", 84, 10, None, 1, 0, None)]
_3CONV3FC = [("conv1", 1, 32, 5, 1, 2, 32), ("conv2", 32, 64, 5, 1, 2, 15), ("conv3", 64, 128, 5, 1, 1, 7),
             ("fc1", 512, 1000, None, 1, 0, None), ("fc2", 1000, 1000, None, 1, 0, None),
             ("fc3", 1000, 10, None, 1, 0, None)]


def _model(prefix, why, layers, B, **kw):
    return [_c(f"{prefix}_{tag}_b{B}", f"{why}: {tag}", cin, cout, k, s, p, 1, hw, B, **kw)
            for (tag, cin, cout, k, s, p, hw) in layers]


def _fold(prefix, why, layers, rows, samples, variants, first_image=0):
    return [_c(f"{prefix}_{tag}_fold{samples}x{rows}", f"{why}: {tag}", cin, cout, k, s, p, 1, hw, rows * samples,
               variants=variants, refuse=("fp32",), fold=(rows, first_image))
            for (tag, cin, cout, k, s, p, hw) in layers]


_TC = ("bf16", "tf32")
CASES = (
    _model("alexnet", "BBBAlexNet at the benchmark batch (10 classes); every map divides the 128-row tile", _ALEXNET, 512)
    + _model("alexnet100", "BBBAlexNet, 100 classes, B = 1024 (C4); fc N = 100 is a ragged 64-column tile",
             _ALEXNET[:5] + [("fc", 128, 100, None, 1, 0, None)], 1024)
    + _model("lenet", "BBBLeNet at B = 256, 3 input channels: 28x28 and 10x10 maps (OHW >= 128, and < 128 not "
             "dividing it), N = 6 and 10 with N % 4 != 0", _LENET, 256)
    + [_c("lenet1_conv1_b256", "BBBLeNet with 1 input channel (MNIST), conv1: K = 25 < one K block; its other layers "
          "are those of the 3-channel net", 1, 6, 5, 1, 0, 1, 32, 256)]
    + _model("3conv3fc", "BBB3Conv3FC at B = 256: 15x15 and 7x7 maps (OHW 225 >= 128, 25 not dividing 128), N = 1000",
             _3CONV3FC, 256)
    + _model("3conv3fc", "BBB3Conv3FC at B = 2048 (C5): many M tiles, checked on a subset of images", _3CONV3FC, 2048)
    # the MC-sample folds (desc->reserved[1..3]) of MCForward and MCTrainStep
    + _fold("lenet", "MCForward's layer fold of BBBLeNet, 10 samples x 256 images; BBB: rows x OHW % 128 == 0 at "
            "every layer", _LENET, 256, 10, ("bbb", "lrt"))
    + _fold("3conv3fc", "MCForward's layer fold of BBB3Conv3FC (LRT), 4 samples x 2048 images", _3CONV3FC, 2048, 4,
            ("lrt",))
    + _fold("alexnet", "MCTrainStep(fold=True) on BBBAlexNet (LRT), 4 samples x 512 images", _ALEXNET, 512, 4,
            ("lrt",))
    + [
        _c("lenet_conv2_fold3x128_first1000", "a fold of 3 samples whose row blocks start at image 1000 (a row block of "
           "a sharded step): the noise index of image b is b % rows + 1000", 6, 16, 5, 1, 0, 1, 14, 384,
           refuse=("fp32",), fold=(128, 1000)),
        # edges
        _c("edge_conv_b1", "a single image", 16, 24, 3, 1, 1, 1, (5, 5), 1),
        _c("edge_lin_b1", "a single row, N = 70", 100, 70, B=1),
        _c("edge_lin_m127", "M = 127: one row short of a tile; N = 6", 96, 6, B=127),
        _c("edge_lin_m128", "M = 128: exactly one tile; N = 30 (the 32-wide CUDA-core tile, N % 4 != 0)", 96, 30,
           B=128),
        _c("edge_lin_m129", "M = 129: one row into a second tile; N = 100", 96, 100, B=129),
        _c("edge_conv_m129", "M = 3 x 43 = 129 on a conv (OHW = 43 does not divide 128), K = 14", 2, 10, (1, 7), 1, 0,
           1, (1, 49), 3),
        _c("edge_cout1", "Cout = 1: one output channel", 3, 1, 3, 1, 1, 1, (7, 7), 5),
        _c("edge_lin_k100_n70", "K = 100 and N = 70: neither a multiple of the 64-wide (bf16) or 32-wide (tf32) K block "
           "nor of the 64-column tile", 100, 70, B=33),
        _c("edge_conv_k45", "K = 5*3*3 = 45 < 64 with stride 2 on a non-square map", 5, 7, 3, 2, 1, 1, (9, 8), 6),
        _c("edge_k2s3", "stride 3 > kernel 2: input pixels no output reads", 5, 7, 2, 3, 0, 1, (11, 10), 4),
        _c("edge_rect_asym", "3x2 kernel, stride (2, 1), padding (1, 2), dilation (1, 2): every axis differs",
           6, 5, (3, 2), (2, 1), (1, 2), (1, 2), (9, 8), 3),
        _c("edge_k4x2_s3_d2", "4x2 kernel, stride 3, dilation 2, padding (2, 1)", 4, 9, (4, 2), 3, (2, 1), 2, (13, 11),
           5),
        _c("edge_1x1_p1", "1x1 conv with padding 1: the border outputs read only padding", 8, 4, 1, 1, 1, 1, (6, 6), 2),
        _c("edge_sparse_conv", "zero receptive fields (x >= 0, half the images and half of every map zero, no bias): "
           "act_std must be sqrt(1e-16)", 5, 7, 3, 1, 1, 1, (10, 9), 6, sparse=True),
        _c("edge_sparse_lenet_conv1", "zero receptive fields at LeNet conv1's shape (bf16 staging of x)", 3, 6, 5, 1,
           0, 1, 32, 8, sparse=True),
        _c("edge_lin_k5000_3stages", "LRT linear K = 5000 (K % 64 = 8): the two-plane ring has 3 stages", 5000, 70,
           B=130),
        _c("edge_lin_k16384", "K = 16384: the largest K the tensor cores take (both variants size two planes); LRT "
           "runs a 2-stage ring in 231423 bytes of shared memory", 16384, 70, B=130),
        _c("edge_lin_k16385", "K = 16385: refused on the tensor cores, auto resolves to fp32", 16385, 70, B=130,
           refuse=_TC),
        _c("edge_act_relu", "epilogue_act = relu on a conv", 4, 20, 3, 1, 1, 1, (12, 12), 3, act="relu"),
        _c("edge_act_softplus", "epilogue_act = softplus on a linear layer", 150, 40, B=70, act="softplus"),
        _c("edge_kl_textbook", "the textbook KL convention, KL(q || p)", 6, 16, 5, 1, 0, 1, 14, 4, kl="textbook"),
        _c("edge_no_bias", "LeNet conv2 without a bias", 6, 16, 5, 1, 0, 1, 14, 16, bias=False),
        _c("edge_lin_no_bias", "a linear layer without a bias, N = 10", 84, 10, B=40, bias=False),
        _c("edge_y_2gb", "BBB3Conv3FC conv1 at B = 20000: y and act_std are 2.6 GB each; images 16384 on start past "
           "2^31 bytes", 1, 32, 5, 1, 2, 1, 32, 20000, extra=(16383, 16384, 16385)),
    ]
)
assert len({c.name for c in CASES}) == len(CASES)


def conv_of(cs):
    """The ((sh, sw), (ph, pw), (dh, dw)) geometry of a case, None for a linear layer."""
    return None if cs.k is None else (cs.s, cs.p, cs.d)


def x_shape(cs, B=None):
    B = cs.B if B is None else B
    return (B, cs.cin) if cs.k is None else (B, cs.cin) + cs.hw


def w_shape(cs):
    return (cs.cout, cs.cin) if cs.k is None else (cs.cout, cs.cin) + cs.k


def out_hw(cs):
    if cs.k is None:
        return 1, 1
    (sh, sw), (ph, pw), (dh, dw) = conv_of(cs)
    return ((cs.hw[0] + 2 * ph - dh * (cs.k[0] - 1) - 1) // sh + 1,
            (cs.hw[1] + 2 * pw - dw * (cs.k[1] - 1) - 1) // sw + 1)


def y_shape(cs, B=None):
    B = cs.B if B is None else B
    return (B, cs.cout) if cs.k is None else (B, cs.cout) + out_hw(cs)


def K_of(cs):
    return cs.cin * (1 if cs.k is None else cs.k[0] * cs.k[1])


def ohw_of(cs):
    oh, ow = out_hw(cs)
    return oh * ow


def resolves(cs):
    """The math mode auto runs."""
    return "fp32" if "bf16" in cs.refuse else "bf16"


def large(cs):
    """Checked against float64 on a subset of images (check_images) rather than on all of them."""
    return cs.B >= 2048 or cs.fold is not None


def check_images(cs, seed=0):
    """The images of a case compared with float64: all of them, or for a large case the first and last, the images on
    both sides of every 128-row tile boundary in the first and last three tiles, both sides of every MC-sample block,
    the row's extra images and 32 seeded random ones."""
    if not large(cs):
        return list(range(cs.B))
    ohw = ohw_of(cs)
    M = cs.B * ohw
    tiles = (M + 127) // 128
    im = {0, cs.B - 1} | set(cs.extra)
    for t in list(range(1, 4)) + list(range(max(1, tiles - 3), tiles)):
        im |= {(128 * t - 1) // ohw, min(M - 1, 128 * t) // ohw}
    if cs.fold is not None:
        rows = cs.fold[0]
        for j in range(1, cs.B // rows):
            im |= {j * rows - 1, j * rows}
    g = np.random.default_rng(seed)
    im |= set(int(v) for v in g.choice(cs.B, size=min(32, cs.B), replace=False))
    return sorted(i for i in im if 0 <= i < cs.B)


def make_inputs(cs, variant, g, device="cpu", B=None, var_plane=False):
    """fp32 layer inputs: x, W_mu, W_rho, bias_mu, bias_rho (None without a bias) and external eps (BBB: (W_eps,
    bias_eps); LRT: activation-shaped).  var_plane: x from var_x, W_rho constant per output channel, no bias."""
    B = cs.B if B is None else B
    rn = lambda shape: torch.randn(shape, generator=g, device=device)
    ws = w_shape(cs)
    fan_in = int(np.prod(ws[1:]))
    x = var_x(x_shape(cs, B), g, device) if var_plane else rn(x_shape(cs, B))
    if cs.sparse:
        x = x.abs() if var_plane else x.clamp_min(0.0)
        x[: B // 2] = 0.0
        if x.dim() == 4:
            x[:, :, : cs.hw[0] // 2] = 0.0
    W_mu = rn(ws) * fan_in ** -0.5
    if var_plane:
        W_rho = (rn(ws[0]) * 0.5 - 3.0).view((-1,) + (1,) * (len(ws) - 1)).expand(ws).contiguous()
    else:
        W_rho = rn(ws) * 0.5 - 3.0
    bias = cs.bias and not var_plane
    b_mu = rn(ws[0]) * 0.5 if bias else None
    b_rho = rn(ws[0]) * 0.5 - 3.0 if bias else None
    eps = (rn(ws), rn(ws[0]) if bias else None) if variant == "bbb" else rn(y_shape(cs, B))
    return x, W_mu, W_rho, b_mu, b_rho, eps


# ---------------------------------------------------------------------------------------------------------------- #
# launch decisions, restated from fwd_tc.cuh (launch_fwd_tc_t, tc_supported) and fwd_simt.cuh (launch_fwd_simt)
# ---------------------------------------------------------------------------------------------------------------- #
TC_BM, TC_BN, TC_BK = 128, 64, 64
TC_SMEM_LIMIT = 227 * 1024
TC_PER_SM = 228 * 1024
TC_A_BYTES, TC_B_BYTES = TC_BM * TC_BK * 2, TC_BN * TC_BK * 2


def _ceil(a, b):
    return (a + b - 1) // b


def tc_bk(tf32):
    return TC_BK // 2 if tf32 else TC_BK


def tc_kpad(K, tf32=False):
    return _ceil(K, tc_bk(tf32)) * tc_bk(tf32)


def tc_stages(K, planes):
    fixed = 2048 + 1024 + tc_kpad(K) * 8
    return min(4, (TC_SMEM_LIMIT - fixed) // (planes * (TC_A_BYTES + TC_B_BYTES)))


def tc_tile_images(ohw):
    """(images a 128-row tile can touch, mode): 'divides' (128 % OHW == 0), 'large' (OHW >= 128) or 'ragged'."""
    if TC_BM % ohw == 0:
        return TC_BM // ohw, "divides"
    if ohw >= TC_BM:
        return 2, "large"
    return _ceil(TC_BM, ohw) + 1, "ragged"


def tc_supported(cs):
    K, N = K_of(cs), cs.cout
    n_tiles = _ceil(N, TC_BN)
    return (tc_stages(K, 2) >= 2 and n_tiles * (tc_kpad(K, True) // tc_bk(True)) <= 1 << 20 and n_tiles <= 65535)


def tc_launch(cs, variant, sample, math):
    """What launch_fwd_tc_t decides for a call: planes, k_blocks, stages, shared-memory bytes, stage_x and the
    tile-image mode."""
    tf32 = math == "tf32"
    K = K_of(cs)
    planes = 2 if variant == "lrt" and sample else 1
    k_blocks = tc_kpad(K, tf32) // tc_bk(tf32)
    stages = tc_stages(K, planes)
    if k_blocks <= 8 and stages > 2:
        stages = 2
    tiles_off = _ceil(1024 + tc_kpad(K, tf32) * 8, 1024) * 1024
    smem = 1023 + tiles_off + stages * planes * (TC_A_BYTES + TC_B_BYTES)
    hw = 1 if cs.k is None else cs.hw[0] * cs.hw[1]
    timg, mode = tc_tile_images(ohw_of(cs))
    xs = timg * cs.cin * hw
    stage_x = 0
    if xs * 4 <= 32 * 1024 and smem + xs * 4 <= TC_SMEM_LIMIT:
        stage_x = 1
        if (not tf32 and 2 * (smem + xs * 4 + 1024) > TC_PER_SM
                and 2 * (_ceil(smem + xs * 2, 128) * 128 + 1024) <= TC_PER_SM):
            stage_x = 2
        smem += xs * (2 if stage_x == 2 else 4)
    return {"planes": planes, "k_blocks": k_blocks, "stages": stages, "smem": smem, "stage_x": stage_x,
            "tile_mode": mode, "tile_images": timg}


def simt_config(cs):
    """(N tile of launch_fwd_simt, linear_like) of the fp32 kernel."""
    N = cs.cout
    bn = 16 if N <= 16 else (32 if N <= 32 else 64)
    linear_like = cs.k is None or (cs.k == (1, 1) and cs.hw == (1, 1) and cs.p == (0, 0))
    return bn, linear_like

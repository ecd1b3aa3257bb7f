"""Plain restatements of the fused tensor-core chain, for its tests (not a test module itself).

- ``pack_tiled`` / ``unpack_tiled``: the "tiled packed" bf16 activation layout of include/bbb_b200.h
  (BBB_LAYOUT_PACKED_BF16), written from its comment, not from the kernels.
- ``layer_ref``: one fused layer in float64 on the operands the kernels really multiply (the bf16 roundings of the
  weight preps in fused_tc.cuh / fwd_tc.cuh / conv_s4_tc.cuh), then the activation and the 2x2 max-pool, together
  with the magnitude ``M`` the error bound scales with.
- ``norm_err``: the worst |y - ref| / (C_BF16 * (M + |ref|)); a kernel output passes when it is <= 1.
- ``CASES``: one-layer cases of the chain, and the helpers that build their steps, outputs and calls
  (``fused_call``: one bbb_layer_forward_fused_prior call in any phase, fold, first image or stream base).
"""
import collections
import contextlib
import ctypes as C

import torch
import torch.nn.functional as F

# ---------------------------------------------------------------------------------------------------------------- #
# error bound
# ---------------------------------------------------------------------------------------------------------------- #
# bf16 keeps 8 significant bits: unit roundoff u = 2^-8, one ulp <= 2^-7 * |v|.  Against a reference computed on the
# same bf16 operands, what a kernel may still differ by is:
#   - a 1-ulp different weight (softplus_sigma_fast is not log1p(exp(.)) to the last fp32 bit, and W_mu + sigma*eps is
#     formed in fp32 before its bf16 rounding): <= 2^-7 * sum |x||w|;
#   - a 1-ulp different variance weight (sigma^2 rounded to bf16), so sqrt(var) is off by <= 2^-8 relative:
#     <= 2^-8 * sqrt(var) * |eps|;
#   - the bf16 rounding of the stored output: <= 2^-8 * |y|;
#   - fp32 accumulation, the fast sqrt / exp / log of the epilogue: ~K * 2^-24, negligible.
# With M = sum|x||w| + |b| + sqrt(var)|eps| the sum is below 2^-7 * M + 2^-8 * |ref| (+ second order), so
# |y - ref| <= C_BF16 * (M + |ref|) holds for a correct kernel.  A wrong column block, a swapped tap, a wrong x^2 or a
# dropped bias moves an element by a sizeable fraction of M: the mutants of tests/test_fused_geometry_cpu.py break this
# bound by 4x or more.
C_BF16 = 2.0 ** -7

BF16_NAN_BITS = 0x7FC0          # the fill of packed outputs before a call (int16 view)


def bf16(t):
    """Round to bf16 the way the kernels do (fp32 first, then round-to-nearest-even), returned as float64."""
    return t.float().to(torch.bfloat16).double()


def norm_err(y, ref, mag):
    """Worst |y - ref| / (C_BF16 * (mag + |ref|)) over all elements (<= 1: inside the bound; a NaN counts as inf)."""
    y, ref, mag = y.double().cpu(), ref.double().cpu(), mag.double().cpu()
    e = (y - ref).abs() / (C_BF16 * (mag + ref.abs()) + 1e-300)
    return float(torch.nan_to_num(e, nan=float("inf")).max())


def sq_mag(ref, mag):
    """Magnitude for the x^2 plane against ref^2: (ref + d)^2 - ref^2 = 2 ref d + d^2 with |d| <= C (M + |ref|),
    plus the bf16 rounding of the square, stays below C_BF16 * 2 (M + |ref|)^2."""
    return 2.0 * (mag + ref.abs()) ** 2


# ---------------------------------------------------------------------------------------------------------------- #
# tiled packed layout (include/bbb_b200.h, BBB_LAYOUT_PACKED_BF16)
# ---------------------------------------------------------------------------------------------------------------- #
# The [B, F] matrix (F = H*W*C, column (h*W + w)*C + c) is stored as [ceil(B/128)][F/64][planes][128 rows x 64 bf16]:
# blocks of 128 rows x 64 columns (16 KB), and inside a block the 16-byte chunk c (8 columns) of row r sits at chunk
# c ^ (r & 7).  With the square carried, every block is [x | x^2] (32 KB), so x^2 starts 8192 elements after x.
def tiled_index(B, F, planes, plane=0, swizzle=True):
    """Element offset of (row b < B, column f < F) of `plane` inside the tiled buffer, as a [B, F] int64 tensor."""
    assert F % 64 == 0
    b = torch.arange(B, dtype=torch.int64)[:, None]
    col = torch.arange(F, dtype=torch.int64)[None, :]
    r = b & 127
    chunk = (col & 63) >> 3
    if swizzle:
        chunk = chunk ^ (r & 7)
    return (((b >> 7) * (F // 64) + (col >> 6)) * planes + plane) * 8192 + r * 64 + chunk * 8 + (col & 7)


def tiled_rows(B):
    return (B + 127) // 128 * 128


def nchw_to_cols(x):
    """[B, C, H, W] -> the [B, H*W*C] matrix of the packed layout (column (h*W + w)*C + c)."""
    return x.permute(0, 2, 3, 1).reshape(x.shape[0], -1)


def cols_to_nchw(m, C_, H, W):
    return m.reshape(m.shape[0], H, W, C_).permute(0, 3, 1, 2)


def pack_tiled(x, planes=1):
    """[B, F] values -> bf16 buffer [ceil(B/128)*128, F*planes] in the tiled packed layout.  planes == 2 adds the
    square bf16(x*x) behind every block.  Rows past B (the padding of the last 128-row block) hold bf16 NaN."""
    B, F_ = x.shape
    buf = torch.full((tiled_rows(B) * F_ * planes,), float("nan"), dtype=torch.bfloat16)
    xd = x.double()
    buf[tiled_index(B, F_, planes, 0).reshape(-1)] = xd.reshape(-1).float().to(torch.bfloat16)
    if planes == 2:
        buf[tiled_index(B, F_, planes, 1).reshape(-1)] = (xd * xd).reshape(-1).float().to(torch.bfloat16)
    return buf.view(tiled_rows(B), F_ * planes)


def unpack_tiled(buf, B, F, planes=1, plane=0, swizzle=True):
    """The [B, F] float64 matrix of `plane` of a tiled packed buffer (swizzle=False decodes without the XOR)."""
    flat = buf.reshape(-1).cpu()
    return flat[tiled_index(B, F, planes, plane, swizzle).reshape(-1)].double().view(B, F)


def padding_bits(buf, B, F, planes=1):
    """int16 bits of every element of the rows B .. ceil(B/128)*128 - 1 (all planes)."""
    Bp = tiled_rows(B)
    if Bp == B:
        return torch.empty(0, dtype=torch.int16)
    flat = buf.reshape(-1).cpu().view(torch.int16)
    idx = [tiled_index(Bp, F, planes, p)[B:].reshape(-1) for p in range(planes)]
    return flat[torch.cat(idx)]


# ---------------------------------------------------------------------------------------------------------------- #
# one fused layer in float64
# ---------------------------------------------------------------------------------------------------------------- #
def softplus_sigma(rho):
    return torch.log1p(torch.exp(rho.double()))


def _contract(x, w, b, conv):
    if conv is None:
        return F.linear(x, w, b)
    stride, padding = conv
    return F.conv2d(x, w, b, stride, padding)


def apply_act(y, act):
    if act == "relu":
        return torch.relu(y)
    if act == "softplus":
        return F.softplus(y)                 # nn.Softplus(beta=1, threshold=20)
    assert act in (None, "none")
    return y


def layer_ref(x, W_mu, W_rho, b_mu, b_rho, variant, eps_a, eps_b=None, conv=None, act="none", pool=False,
              x_sq=None):
    """One fused layer (BBB or LRT) in float64 on the operands the kernel multiplies.

    x: NCHW (conv, ``conv`` = (stride, padding)) or [B, K] in the reference feature order (linear); its values must
    be bf16-representable.  x_sq: the x^2 operand (default bf16(x*x): the plane a producing epilogue stores, and what
    the first-layer kernels compute from bf16(x)).  eps_a: BBB weight eps / LRT activation eps (shape of the pre-pool
    output); eps_b: BBB bias eps.  Returns (ref, M): the layer output after activation and pool, and the magnitude
    sum|x||w| + |b| + sqrt(var)|eps| (max over the pool window)."""
    x = x.double()
    x_sq = bf16(x * x) if x_sq is None else x_sq.double()
    W_mu, b_mu = W_mu.double(), b_mu.double()
    sig, sig_b = softplus_sigma(W_rho), softplus_sigma(b_rho)
    if variant == "bbb":
        W = bf16(W_mu + sig * eps_a.double())                 # W_mu + softplus(W_rho) * eps, one bf16 rounding
        b = b_mu + sig_b * eps_b.double()                     # the bias stays fp32
        y = _contract(x, W, b, conv)
        mag = _contract(x.abs(), W.abs(), b.abs(), conv)
    else:
        Wm, Wv = bf16(W_mu), bf16(sig * sig)                  # bf16(W_mu) and bf16(softplus(W_rho)^2)
        mean = _contract(x, Wm, b_mu, conv)
        sd = torch.sqrt(_contract(x_sq, Wv, sig_b * sig_b, conv) + 1e-16)
        e = eps_a.double()
        y = mean + sd * e
        mag = _contract(x.abs(), Wm.abs(), b_mu.abs(), conv) + sd * e.abs()
    y = apply_act(y, act)
    if pool:
        y, mag = F.max_pool2d(y, 2, 2), F.max_pool2d(mag, 2, 2)
    return y, mag


# ---------------------------------------------------------------------------------------------------------------- #
# engine queries (host-only, no GPU needed)
# ---------------------------------------------------------------------------------------------------------------- #
def nchw_path(st):
    """'s4' or 'gather': which kernel bbb_layer_forward_fused runs for a planned step with an NCHW input.
    The engine folds MC samples of an LRT layer on the stride-4 kernel only, so asking bbb_fused_supported about a
    fold of the same geometry tells the two apart without running anything."""
    from pytorch_bayesiancnn_b200 import _lib as L, fused
    d = fused._step_desc(st, 0)
    assert L.lib().bbb_fused_supported(C.byref(d), st.in_layout, fused._in_pitch(st), st.prev_hw, st.out_layout,
                                       fused._out_pitch(st)) == 0
    d.variant, d.sample, d.reserved[1] = L.VARIANT_LRT, 1, st.batch
    rc = L.lib().bbb_fused_supported(C.byref(d), st.in_layout, fused._in_pitch(st), st.prev_hw, st.out_layout,
                                     fused._out_pitch(st))
    return "s4" if rc == 0 else "gather"


# ---------------------------------------------------------------------------------------------------------------- #
# whole nets the planner accepts (or must refuse), as ModuleWrapper child lists
# ---------------------------------------------------------------------------------------------------------------- #
# item: ("conv", cin, cout, k, stride, pad[, dilation]) | ("fc", in, out) | ("relu",) | ("softplus",)
#       | ("pool", k, stride) | ("flatten", features)
NETS = {
    # stride-4 k11 conv on a grayscale 64x64 image (OW = 16: the gather kernel), a tap-GEMM on an 8x8 map with exactly
    # TAP_MAX_ITEMS = 64 schedule items, a stride-2 tap-GEMM, a linear fed by a 2x2 map (prev_hw = 4)
    "gray64": ((37, 1, 64, 64), [("conv", 1, 64, 11, 4, 5), ("relu",), ("pool", 2, 2),
                                 ("conv", 64, 128, 3, 1, 1), ("softplus",), ("pool", 2, 2),
                                 ("conv", 128, 64, 3, 2, 1), ("flatten", 256), ("fc", 256, 10)]),
    # gather first layer with pool and packed output, 1x1 taps, Cout = 192 unpooled, prev_hw = 4
    "gather_k1": ((130, 3, 8, 8), [("conv", 3, 64, 3, 1, 1), ("relu",), ("pool", 2, 2),
                                   ("conv", 64, 192, 1, 1, 0), ("softplus",),
                                   ("conv", 192, 128, 3, 1, 0), ("flatten", 512), ("fc", 512, 100)]),
    # non-square maps: 4x8 -> pooled 2x4, prev_hw = 8
    "nonsquare": ((5, 3, 4, 8), [("conv", 3, 64, 3, 1, 1), ("relu",),
                                 ("conv", 64, 64, 3, 1, 1), ("relu",), ("pool", 2, 2),
                                 ("flatten", 512), ("fc", 512, 10)]),
    # stride-4 kernel with k7 and OH != OW, Cout = 320, prev_hw = 6, fp32 logits with N = 72
    "s4_k7": ((200, 3, 48, 32), [("conv", 3, 64, 7, 4, 3), ("softplus",), ("pool", 2, 2),
                                 ("conv", 64, 320, 3, 1, 1), ("relu",), ("pool", 2, 2),
                                 ("flatten", 1920), ("fc", 1920, 72)]),
    # pooled NCHW fp32 output as the last layer, Cout = 72: the last 16-column pool group is partial
    "pool_last": ((129, 3, 32, 32), [("conv", 3, 64, 11, 4, 5), ("relu",), ("pool", 2, 2),
                                     ("conv", 64, 72, 3, 1, 1), ("relu",), ("pool", 2, 2)]),
}
# nets the planner must refuse: more than TAP_MAX_ITEMS (input pixel, 64-channel block) pairs in a tile
REFUSED_NETS = {
    "map8x8_cin128": ((6, 3, 8, 8), [("conv", 3, 128, 3, 1, 1), ("relu",),
                                     ("conv", 128, 64, 3, 1, 1), ("relu",), ("pool", 2, 2),
                                     ("flatten", 1024), ("fc", 1024, 10)]),
    "map4x4_cin320": ((6, 3, 4, 4), [("conv", 3, 320, 3, 1, 1), ("relu",),
                                     ("conv", 320, 64, 3, 1, 1), ("flatten", 1024), ("fc", 1024, 10)]),
}


def make_net(spec, variant, seed=0):
    """A ModuleWrapper whose children are the layers of `spec` (see NETS), parameters drawn from `seed`."""
    from pytorch_bayesiancnn_b200.modules import (BBBConv2d, BBBLinear, BBBLRTConv2d, BBBLRTLinear, FlattenLayer,
                                                  ModuleWrapper)
    from torch import nn

    class SpecNet(ModuleWrapper):
        def __init__(self):
            super().__init__()
            for i, it in enumerate(spec):
                kind = it[0]
                if kind == "conv":
                    cls = BBBLRTConv2d if variant == "lrt" else BBBConv2d
                    dil = it[6] if len(it) > 6 else 1
                    m = cls(it[1], it[2], it[3], stride=it[4], padding=it[5], dilation=dil)
                elif kind == "fc":
                    m = (BBBLRTLinear if variant == "lrt" else BBBLinear)(it[1], it[2])
                elif kind == "relu":
                    m = nn.ReLU()
                elif kind == "softplus":
                    m = nn.Softplus()
                elif kind == "pool":
                    m = nn.MaxPool2d(kernel_size=it[1], stride=it[2])
                else:
                    m = FlattenLayer(it[1])
                self.add_module(f"m{i}", m)

    net = SpecNet()
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in net.children():
            if hasattr(m, "W_mu"):
                fan_in = m.W_mu[0].numel()
                init_layer_params(m, fan_in, g)
    return net


def init_layer_params(m, fan_in, g, bias_sigma=None):
    """Weights of unit-scale outputs, sigma about half the spread of mu (the noise term is far above bf16 rounding).
    The bias sigma is about 0.05, or about ``bias_sigma`` when given (BBB: a bias noise term the float64 bar sees)."""
    s = fan_in ** -0.5
    rho0 = float(torch.log(torch.expm1(torch.tensor(0.5 * s))))
    m.W_mu.copy_(torch.randn(m.W_mu.shape, generator=g) * s)
    m.W_rho.copy_(rho0 + 0.1 * torch.randn(m.W_rho.shape, generator=g))
    m.bias_mu.copy_(0.5 * torch.randn(m.bias_mu.shape, generator=g))
    brho = -3.0 if bias_sigma is None else float(torch.log(torch.expm1(torch.tensor(float(bias_sigma)))))
    m.bias_rho.copy_(brho + 0.1 * torch.randn(m.bias_rho.shape, generator=g))


def net_eps(net, x_shape, variant, seed):
    """External eps for one forward of `net`, in the reference's draw order (BBB: W_eps, bias_eps per layer; LRT: one
    eps of the layer output's shape)."""
    from pytorch_bayesiancnn_b200.modules import _BayesLayer
    g = torch.Generator().manual_seed(seed)
    eps = []
    shape = x_shape
    for m in net.children():
        if isinstance(m, _BayesLayer):
            if m._conv_geometry() is None:
                out = (shape[0], m.out_features)
            else:
                (sh, sw), (ph, pw), (dh, dw) = m._conv_geometry()
                kh, kw = m.kernel_size
                out = (shape[0], m.out_channels, (shape[2] + 2 * ph - dh * (kh - 1) - 1) // sh + 1,
                       (shape[3] + 2 * pw - dw * (kw - 1) - 1) // sw + 1)
            if variant == "lrt":
                eps.append(torch.randn(out, generator=g))
            else:
                eps.append(torch.randn(m.W_mu.shape, generator=g))
                eps.append(torch.randn(m.bias_mu.shape, generator=g))
            shape = out
        elif isinstance(m, torch.nn.MaxPool2d):
            k, s = m.kernel_size, m.stride
            shape = (shape[0], shape[1], (shape[2] - k) // s + 1, (shape[3] - k) // s + 1)
        elif hasattr(m, "num_features"):
            shape = (shape[0], m.num_features)
    return eps


def net_ref(net, x, eps, variant):
    """float64 composition of the oracle's layer forwards (oracle.bbb_forward / lrt_forward), activations, pools and
    flattens of `net`'s children on the eps list `eps`; returns (output, KL)."""
    from oracle import bbb_oracle as O
    from pytorch_bayesiancnn_b200.modules import _BayesLayer
    eps = list(eps)
    x = x.double().cpu()
    kl = 0.0
    for m in net.children():
        if isinstance(m, _BayesLayer):
            p = [t.detach().double().cpu() for t in (m.W_mu, m.W_rho, m.bias_mu, m.bias_rho)]
            geo = m._conv_geometry()
            if variant == "lrt":
                x = O.lrt_forward(x, *p, eps.pop(0).double(), conv=geo)
            else:
                we, be = eps.pop(0).double(), eps.pop(0).double()
                x = O.bbb_forward(x, *p, we, be, conv=geo)
            kl = kl + float(O.kl_loss(*p, m.prior_mu, m.prior_sigma))
        elif isinstance(m, torch.nn.ReLU):
            x = torch.relu(x)
        elif isinstance(m, torch.nn.Softplus):
            x = F.softplus(x)
        elif isinstance(m, torch.nn.MaxPool2d):
            x = F.max_pool2d(x, m.kernel_size, m.stride)
        else:
            x = x.reshape(-1, m.num_features)
    assert not eps
    return x, kl


# ---------------------------------------------------------------------------------------------------------------- #
# one-layer cases of the fused chain (tests/test_gpu_fused_geometry.py, tests/test_gpu_fused_modes.py)
# ---------------------------------------------------------------------------------------------------------------- #
Case = collections.namedtuple("Case", "name why kind variant cin hw cout k s p pool act out sq wide B prev_hw")


def _c(name, why, kind, variant, cin, hw, cout, k=1, s=1, p=0, pool=False, act="none", out="packed", sq=False,
       wide=0, B=128, prev_hw=1):
    return Case(name, why, kind, variant, cin, hw, cout, k, s, p, pool, act, out, sq, wide, B, prev_hw)


CASES = [
    # ---- tap-GEMM conv layers (tap_gemm_kernel; tap_prep_conv_kernel for k > 1, tap_prep_kernel for 1x1 taps)
    _c("t8x8_c64_k3p1_pool_lrt", "8x8 map with exactly TAP_MAX_ITEMS = 64 schedule items; pooled packed + x^2; ragged "
       "second row tile", "tap", "lrt", 64, (8, 8), 128, 3, 1, 1, True, "softplus", "packed", True, 0, 129),
    _c("t8x8_k3s2p1_bbb", "stride-2 taps; unpooled bulk-copy store of one full row tile", "tap", "bbb",
       64, (8, 8), 64, 3, 2, 1, False, "relu", "packed", False, 0, 128),
    _c("t8x8_k3s2p1_wide_lrt", "stride-2 taps, BN = 128 unpooled: bulk copy of two tiles + direct store of the ragged "
       "third", "tap", "lrt", 64, (8, 8), 128, 3, 2, 1, False, "none", "packed", True, 1, 300),
    _c("t4x8_c128_items64_lrt", "non-square 4x8 map, Cin = 128 (64 items); one ragged tile: direct stores only",
       "tap", "lrt", 128, (4, 8), 64, 3, 1, 1, False, "none", "packed", False, 0, 127),
    _c("t4x8_pool_nchw72_bbb", "non-square pooled NCHW fp32 output, Cout = 72: partial 16-column pool group",
       "tap", "bbb", 64, (4, 8), 72, 3, 1, 1, True, "relu", "f32", False, 0, 129),
    _c("t4x8_pool_nchw72_lrt", "as above, LRT, one image", "tap", "lrt", 64, (4, 8), 72, 3, 1, 1, True, "softplus",
       "f32", False, 0, 1),
    _c("t4x4_c256_items64_wide_bbb", "Cin = 256 on 4x4 (64 items), BN = 128 unpooled, x^2 for an LRT consumer",
       "tap", "bbb", 256, (4, 4), 256, 3, 1, 1, False, "relu", "packed", True, 1, 129),
    _c("t4x4_c192_k1_lrt", "1x1 taps (tap_prep_kernel), Cin = Cout = 192", "tap", "lrt", 192, (4, 4), 192, 1, 1, 0,
       False, "softplus", "packed", True, 0, 129),
    _c("t4x4_k5p2_pool_bbb", "5x5 p2 taps, pooled BN = 64 (16-channel groups), Cout = 192", "tap", "bbb",
       64, (4, 4), 192, 5, 1, 2, True, "softplus", "packed", False, 0, 128),
    _c("t4x4_k5p2_pool_wide_lrt", "5x5 p2, pooled BN = 128 (32-channel groups) + x^2, three row tiles", "tap", "lrt",
       64, (4, 4), 192, 5, 1, 2, True, "relu", "packed", True, 1, 300),
    _c("t4x4_k3p0_b1_bbb", "3x3 p0 (4x4 -> 2x2), a single image", "tap", "bbb", 128, (4, 4), 128, 3, 1, 0, False,
       "relu", "packed", False, 0, 1),
    _c("t4x4_k3p0_nchw100_lrt", "unpooled NCHW fp32 map output, Cout = 100", "tap", "lrt", 64, (4, 4), 100, 3, 1, 0,
       False, "softplus", "f32", False, 0, 127),
    _c("t2x2_c256_lrt", "2x2 map, Cin = 256, 4 of 9 taps live per pixel", "tap", "lrt", 256, (2, 2), 256, 3, 1, 1,
       False, "softplus", "packed", True, 0, 128),
    _c("t2x2_pool320_bbb", "pool to 1x1, Cout = 320, pooled BN = 64", "tap", "bbb", 128, (2, 2), 320, 3, 1, 1, True,
       "none", "packed", False, 0, 129),
    _c("t2x2_pool320_wide_lrt", "Cin = 192, Cout = 320, pooled BN = 128 + x^2", "tap", "lrt", 192, (2, 2), 320, 3, 1, 1,
       True, "relu", "packed", True, 1, 300),
    _c("t2x2_k1_b300_bbb", "1x1 taps; two bulk-copied tiles and a ragged third", "tap", "bbb", 64, (2, 2), 64, 1, 1, 0,
       False, "none", "packed", False, 0, 300),
    _c("t8x8_k1_pool_b1_lrt", "1x1 taps pooled on 8x8, a single image", "tap", "lrt", 64, (8, 8), 64, 1, 1, 0, True,
       "relu", "packed", True, 0, 1),
    _c("t8x8_k5p2_pool_nchw_bbb", "5x5 p2 on 8x8, pooled NCHW fp32 4x4 output", "tap", "bbb", 64, (8, 8), 64, 5, 1, 2,
       True, "softplus", "f32", False, 0, 127),
    _c("t8x8_k3p0_c192_lrt", "3x3 p0 (8x8 -> 6x6), Cout = 192 (BN stays 64 with wide tiles on)", "tap", "lrt",
       64, (8, 8), 192, 3, 1, 0, False, "relu", "packed", True, 1, 128),
    _c("t4x4_c128_softplus_bbb", "BBB softplus unpooled, ragged tile", "tap", "bbb", 128, (4, 4), 64, 3, 1, 1, False,
       "softplus", "packed", False, 0, 127),
    _c("t2x2_nchw10_bbb", "NCHW fp32 output, Cout = 10", "tap", "bbb", 64, (2, 2), 10, 3, 1, 1, False, "none", "f32",
       False, 0, 300),
    _c("t4x4_nchw10_lrt", "Cout = 10 (N % 4 != 0: per-element Philox draws) on a 4x4 map", "tap", "lrt", 64, (4, 4), 10,
       3, 1, 1, False, "relu", "f32", False, 0, 129),
    _c("t4x4_k5p2_c192_bbb", "5x5 p2 taps, Cin = Cout = 192: tap_prep_conv R = 4, the BBB fold stages 52,800 B (opted in "
       "above 48 KB)", "tap", "bbb", 192, (4, 4), 192, 5, 1, 2, False, "relu", "packed", False, 0, 128),
    # ---- linear layers on the tap-GEMM (a 1x1 map; prev_hw = H*W of the flattened map feeding it)
    _c("l_prev1_n10_bbb", "classifier, fp32 logits, Cout = 10", "linear", "bbb", 256, (1, 1), 10, out="f32", B=129),
    _c("l_prev4_n100_lrt", "prev_hw = 4 feature permutation, Cout = 100", "linear", "lrt", 512, (1, 1), 100, out="f32",
       B=300, prev_hw=4),
    _c("l_prev8_n10_lrt", "prev_hw = 8, N % 4 != 0 Philox", "linear", "lrt", 512, (1, 1), 10, out="f32", B=127,
       prev_hw=8),
    _c("l_prev6_n72_lrt", "prev_hw = 6 (a 3x2 map), Cin = 1920 (30 K blocks), fp32 N = 72", "linear", "lrt", 1920, (1, 1),
       72, act="none", out="f32", B=128, prev_hw=6),
    _c("l_prev4_packed_bbb", "hidden linear fed by a 2x2 map, packed output + x^2", "linear", "bbb", 1024, (1, 1), 128,
       act="relu", out="packed", sq=True, B=129, prev_hw=4),
    _c("l_prev1_packed_wide_lrt", "hidden linear, BN = 128 unpooled, Cin = 192", "linear", "lrt", 192, (1, 1), 256,
       act="softplus", out="packed", sq=True, wide=1, B=300),
    _c("l_prev6_n100_b1_bbb", "prev_hw = 6, a single image", "linear", "bbb", 384, (1, 1), 100, act="softplus",
       out="f32", B=1, prev_hw=6),
    _c("l_4096_items64_lrt", "Cin = 4096: 64 K blocks, the schedule limit", "linear", "lrt", 4096, (1, 1), 10, out="f32",
       B=128),
    _c("l_prev8_n72_bbb", "BBB, prev_hw = 8: weight noise at the reference index of a permuted feature", "linear", "bbb",
       512, (1, 1), 72, act="softplus", out="f32", B=129, prev_hw=8),
    # ---- gather first layer (gemm_tc_kernel with the fused epilogue) on an NCHW fp32 image
    _c("g_c3_8x8_pool_packed_lrt", "gather, fused pool, packed output + x^2", "gather", "lrt", 3, (8, 8), 64, 3, 1, 1,
       True, "softplus", "packed", True, 0, 129),
    _c("g_c1_8x8_pool_packed_bbb", "gather, Cin = 1, Cout = 128", "gather", "bbb", 1, (8, 8), 128, 3, 1, 1, True, "relu",
       "packed", False, 0, 128),
    _c("g_c16_4x8_pool_packed_lrt", "gather, Cin = 16, non-square, three row tiles", "gather", "lrt", 16, (4, 8), 64,
       3, 1, 1, True, "relu", "packed", False, 0, 300),
    _c("g_c3_4x8_pool_nchw72_bbb", "gather, pooled NCHW fp32 output, Cout = 72", "gather", "bbb", 3, (4, 8), 72,
       3, 1, 1, True, "relu", "f32", False, 0, 127),
    _c("g_c16_8x8_pool_nchw100_lrt", "gather, pooled NCHW fp32, Cout = 100, one image", "gather", "lrt", 16, (8, 8), 100,
       3, 1, 1, True, "softplus", "f32", False, 0, 1),
    _c("g_c1_64x64_k11s4_lrt", "stride 4, k11 with OW = 16: not the stride-4 kernel, the gather one", "gather", "lrt",
       1, (64, 64), 64, 11, 4, 5, True, "relu", "packed", True, 0, 37),
    _c("g_c3_4x8_nopool_bbb", "gather, unpooled packed output", "gather", "bbb", 3, (4, 8), 64, 3, 1, 1, False, "relu",
       "packed", False, 0, 5),
    # ---- stride-4 first layer (conv_s4_kernel): 16-image row tiles, OW = 8, Cout = 64, pooled packed output
    _c("s_c3_k11_32x32_b17_lrt", "AlexNet conv1 geometry, a ragged second 16-image tile", "s4", "lrt", 3, (32, 32), 64,
       11, 4, 5, True, "relu", "packed", True, 0, 17),
    _c("s_c1_k11_64x32_b16_bbb", "Cin = 1, OH = 16, one full 16-image tile", "s4", "bbb", 1, (64, 32), 64, 11, 4, 5, True,
       "softplus", "packed", False, 0, 16),
    _c("s_c4_k7_48x32_b200_lrt", "Cin = 4, k7 p3, OH = 12 != OW", "s4", "lrt", 4, (48, 32), 64, 7, 4, 3, True,
       "softplus", "packed", True, 0, 200),
    _c("s_c3_k7_32x32_b1_bbb", "k7 p3, a single image", "s4", "bbb", 3, (32, 32), 64, 7, 4, 3, True, "relu", "packed",
       False, 0, 1),
    _c("s_c1_k7_48x32_b15_lrt", "Cin = 1, k7, 15 images (one partial tile), no x^2", "s4", "lrt", 1, (48, 32), 64,
       7, 4, 3, True, "none", "packed", False, 0, 15),
    _c("s_c4_k11_48x32_b17_bbb", "Cin = 4, k11 on 48x32, x^2 for an LRT consumer", "s4", "bbb", 4, (48, 32), 64,
       11, 4, 5, True, "relu", "packed", True, 0, 17),
    _c("s_c3_k11_32x32_b200_bbb", "AlexNet conv1, 200 images (13 tiles, the last partial)", "s4", "bbb", 3, (32, 32),
       64, 11, 4, 5, True, "softplus", "packed", False, 0, 200),
    _c("s_c4_k7_64x32_b16_lrt", "Cin = 4, k7 on 64x32 (OH = 16)", "s4", "lrt", 4, (64, 32), 64, 7, 4, 3, True, "none",
       "packed", True, 0, 16),
]
assert len({c.name for c in CASES}) == len(CASES)


def _out_hw(cs):
    h, w = cs.hw
    return (h + 2 * cs.p - cs.k) // cs.s + 1, (w + 2 * cs.p - cs.k) // cs.s + 1


def _tile_bn(cs, B=None):
    """Column tile width launch_fused picks for a tap-GEMM case (132 SMs) at batch B (default: the case's)."""
    oh, ow = _out_hw(cs)
    ng128 = 32 if cs.pool else 128
    psets = (oh // 2) * (ow // 2) if cs.pool else oh * ow
    row_tiles = ((cs.B if B is None else B) + 127) // 128
    return 128 if cs.cout % ng128 == 0 and (cs.wide or psets * (cs.cout // ng128) * row_tiles >= 132 * 6 // 10) else 64


def prep2_slab(R_):
    return R_ * 64 + 8


def _prep2_rows(cs, B=None):
    """R, the output channels per CTA of tap_prep_conv_kernel: halved from 8 until the grid covers the 132 SMs and the
    bf16 staging fits 26 KB (launch_tap_prep)."""
    planes = 2 if cs.variant == "lrt" else 1
    bn = _tile_bn(cs, B)
    ng = bn // 4 if cs.pool else bn
    npad = (cs.cout + ng - 1) // ng * ng
    n_kblk = (cs.cin + 63) // 64
    R_ = 8
    while R_ > 2 and ((npad // R_) * n_kblk < 132 or planes * cs.k * cs.k * prep2_slab(R_) * 2 > 26 * 1024):
        R_ >>= 1
    return R_


def _prep(cs, B=None):
    """The weight-prep kernel bbb_layer_forward_fused launches for a case (launch_fused / launch_conv_s4 / launch_fwd_tc):
    tap_prep_conv_kernel for a conv layer (KHW > 1, prev_hw == 1, Cin % 64 == 0) whose bf16 staging fits 48 KB, else
    tap_prep_kernel; the stride-4 and gather first layers have their own."""
    if cs.kind == "s4":
        return "conv_s4_prep_kernel"
    if cs.kind == "gather":
        return "weight_prep_kernel"
    planes = 2 if cs.variant == "lrt" else 1
    khw = cs.k * cs.k
    if khw > 1 and cs.prev_hw == 1 and cs.cin % 64 == 0 and planes * khw * prep2_slab(_prep2_rows(cs, B)) * 2 <= 48 * 1024:
        return "tap_prep_conv_kernel"
    return "tap_prep_kernel"


def fold_staging_bytes(cs, B):
    """Dynamic shared memory of tap_prep_conv_kernel's BBB fold at batch B: fp32 (mu, sigma) pairs, KHW * slab * 8."""
    return cs.k * cs.k * prep2_slab(_prep2_rows(cs, B)) * 8


def folds(cs):
    """Does the engine fold MC samples on this case's path?  Every path but the gather one."""
    return cs.kind != "gather"


def _layer(cs):
    import pytorch_bayesiancnn_b200 as bbb
    if cs.kind == "linear":
        return (bbb.BBBLRTLinear if cs.variant == "lrt" else bbb.BBBLinear)(cs.cin, cs.cout)
    cls = bbb.BBBLRTConv2d if cs.variant == "lrt" else bbb.BBBConv2d
    return cls(cs.cin, cs.cout, cs.k, stride=cs.s, padding=cs.p)


def _step(cs, m, B=None):
    """The fused._Step fused.plan builds for a case's layer `m`, at batch B (default: the case's)."""
    from pytorch_bayesiancnn_b200 import fused, _lib as L
    st = fused._Step()
    st.layer, st.batch, st.conv = m, cs.B if B is None else B, m._conv_geometry()
    st.linear = st.conv is None
    st.prev_hw = cs.prev_hw
    st.in_shape = (cs.cin,) + tuple(cs.hw)
    st.in_layout = L.LAYOUT_NCHW_F32 if cs.kind in ("gather", "s4") else L.LAYOUT_PACKED_BF16
    oh, ow = _out_hw(cs)
    st.eps_shape = (cs.cout, oh, ow)
    st.act = L.ACT_BY_NAME[cs.act]
    st.pool = cs.pool
    st.out_chw = (cs.cout, oh // 2, ow // 2) if cs.pool else (cs.cout, oh, ow)
    if cs.out == "packed":
        st.out_layout = L.LAYOUT_PACKED_BF16
    else:
        st.out_layout = L.LAYOUT_ROWMAJOR_F32 if st.out_chw[1:] == (1, 1) else L.LAYOUT_NCHW_F32
    return st


GUARD = 64
SENTINEL = -1.25e37


def _alloc_out(cs, st, dev, B=None):
    """(y, y_sq, n): a NaN-filled tiled buffer, or an fp32 buffer of n outputs + GUARD sentinel floats (B rows, default
    the case's)."""
    B = cs.B if B is None else B
    cout, oh, ow = st.out_chw
    if cs.out == "packed":
        planes = 2 if cs.sq else 1
        y = torch.full((tiled_rows(B), cout * oh * ow * planes), float("nan"), dtype=torch.bfloat16, device=dev)
        return y, (y.view(-1)[8192:] if cs.sq else None), 0
    n = B * cout * oh * ow
    y = torch.full((n + GUARD,), float("nan"), dtype=torch.float32, device=dev)
    y[n:] = SENTINEL
    return y, None, n


def step_desc(st, phase=0, fold=None, first_image=0):
    """fused._step_desc with the first image of a row block in reserved[0] bits 8..30 (out of range: a word the engine
    refuses)."""
    from pytorch_bayesiancnn_b200 import fused, functional as Fn
    d = fused._step_desc(st, phase, fold)
    if first_image:
        d.reserved[0] |= Fn.first_image_word(first_image)
    return d


def fused_call_rc(st, x, x_sq, y, y_sq, eps_a=None, eps_b=None, seed=0, stream=0, phase=0, fold=None, first_image=0,
                  stream_base=None, ws=None, kl=None):
    """One bbb_layer_forward_fused_prior call with arguments as fused.run_step passes them -- the layer's tensor prior
    and pruning mask as Fn.masked_prior_arg passes them -- plus the call's phase (FUSED_* bits), MC-sample fold
    (rows, stride), first image, device stream base (int64[1]) and workspace (default: the layer's own).
    Returns (return code, kl): kl is the fp32 scalar the call wrote (a NaN-filled one unless given)."""
    from pytorch_bayesiancnn_b200 import fused, functional as Fn, _lib as L
    m = st.layer
    dev = m.W_mu.device
    d = step_desc(st, phase, fold, first_image)
    if kl is None:
        kl = torch.full((), float("nan"), dtype=torch.float32, device=dev)
    if ws is None:
        ws = Fn.workspace(dev, d, m)
    parg, flag = Fn.masked_prior_arg(m.prior_tensors(), m.mask_tensors())
    rc = L.lib().bbb_layer_forward_fused_prior(
        C.byref(Fn.desc_with(d, flag)), Fn._ptr(x), Fn._ptr(x_sq), st.in_layout, fused._in_pitch(st), st.prev_hw,
        Fn._ptr(m.W_mu), Fn._ptr(m.W_rho), Fn._ptr(m.bias_mu), Fn._ptr(m.bias_rho),
        Fn._ptr(y), Fn._ptr(y_sq), st.out_layout, fused._out_pitch(st), Fn._ptr(kl), Fn._ptr(eps_a), Fn._ptr(eps_b),
        C.c_uint64(seed), C.c_uint64(stream), Fn._ptr(stream_base), Fn._ptr(ws), C.c_size_t(ws.numel()),
        Fn._stream(dev), parg)
    return rc, kl


def fused_call(st, x, x_sq, y, y_sq, eps_a=None, eps_b=None, seed=0, stream=0, **kw):
    """fused_call_rc that raises EngineError on a refusal; returns the KL scalar."""
    from pytorch_bayesiancnn_b200 import _lib as L
    rc, kl = fused_call_rc(st, x, x_sq, y, y_sq, eps_a, eps_b, seed, stream, **kw)
    L.check(rc, "bbb_layer_forward_fused_prior")
    return kl


def fused_supported(st, phase=0, fold=None, first_image=0, sample=True):
    """bbb_fused_supported (host-only) on a case's step, with a fold, first image or a mean-only (sample = 0) desc."""
    from pytorch_bayesiancnn_b200 import fused, _lib as L
    d = step_desc(st, phase, fold, first_image)
    d.sample = int(sample)
    return L.lib().bbb_fused_supported(C.byref(d), st.in_layout, fused._in_pitch(st), st.prev_hw, st.out_layout,
                                       fused._out_pitch(st))


@contextlib.contextmanager
def wide_tiles(on):
    """Calls inside run with bbb_set_wide_tiles(on) (a case's `wide`), restored after."""
    from pytorch_bayesiancnn_b200 import _lib as L
    prev = L.lib().bbb_set_wide_tiles(int(on))
    try:
        yield
    finally:
        L.lib().bbb_set_wide_tiles(prev)


def first_image_max(cs, rows):
    """The largest first image the engine accepts for `rows` images a call (or a folded sample): its last image's
    outputs still an int32 element count, and the index inside reserved[0] bits 8..30."""
    from pytorch_bayesiancnn_b200 import functional as Fn
    oh, ow = _out_hw(cs)
    return min(Fn.FIRST_IMAGE_MAX, (2 ** 31 - 1) // (oh * ow * cs.cout) - rows)

"""Plain restatements of the fused tensor-core chain, for its tests (not a test module itself).

- ``pack_tiled`` / ``unpack_tiled``: the "tiled packed" bf16 activation layout of include/bbb_b200.h
  (BBB_LAYOUT_PACKED_BF16), written from its comment, not from the kernels.
- ``layer_ref``: one fused layer in float64 on the operands the kernels really multiply (the bf16 roundings of the
  weight preps in fused_tc.cuh / fwd_tc.cuh / conv_s4_tc.cuh), then the activation and the 2x2 max-pool, together
  with the magnitude ``M`` the error bound scales with.
- ``norm_err``: the worst |y - ref| / (C_BF16 * (M + |ref|)); a kernel output passes when it is <= 1.
"""
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


def init_layer_params(m, fan_in, g):
    """Weights of unit-scale outputs, sigma about half the spread of mu (the noise term is far above bf16 rounding)."""
    s = fan_in ** -0.5
    rho0 = float(torch.log(torch.expm1(torch.tensor(0.5 * s))))
    m.W_mu.copy_(torch.randn(m.W_mu.shape, generator=g) * s)
    m.W_rho.copy_(rho0 + 0.1 * torch.randn(m.W_rho.shape, generator=g))
    m.bias_mu.copy_(0.5 * torch.randn(m.bias_mu.shape, generator=g))
    m.bias_rho.copy_(-3.0 + 0.1 * torch.randn(m.bias_rho.shape, generator=g))


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

"""The fused tensor-core chain layer by layer, at every geometry its planner accepts, against a float64 reference.

Each case of CASES is one bbb_layer_forward_fused call, made the way fused.run_step makes it, on external eps and a
tiled packed input built by tests/fused_ref.pack_tiled.  It checks:
  - every output element against tests/fused_ref.layer_ref within C_BF16 * (M + |ref|) (and the x^2 plane against
    ref^2 when the layer writes it);
  - every element of rows < B is written and finite, the padding rows of the last 128-row block keep their NaN fill,
    and fp32 outputs leave a guard of sentinel floats behind them untouched;
  - the KL against oracle.kl_loss to 1e-5 relative;
  - LRT: the in-kernel Philox noise is bit-identical to the same call fed philox_normal as external eps.
The `why` of a case names the branch it exists for; test_case_table_covers_every_branch checks that together they reach
every map, kernel, channel count, batch, tile width, prep and output layout listed there.  Whole nets (fused_ref.NETS)
then check the planner's wiring end to end, and the nets it must refuse run correctly unfused.
Run with -s to see the worst normalised error per case family."""
import collections
import ctypes as C
import sys

import pytest
import torch

from tests import fused_ref as R
from tests.util import scale_err

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


def _tile_bn(cs):
    """Column tile width launch_fused picks for a tap-GEMM case (132 SMs)."""
    oh, ow = _out_hw(cs)
    ng128 = 32 if cs.pool else 128
    psets = (oh // 2) * (ow // 2) if cs.pool else oh * ow
    row_tiles = (cs.B + 127) // 128
    return 128 if cs.cout % ng128 == 0 and (cs.wide or psets * (cs.cout // ng128) * row_tiles >= 132 * 6 // 10) else 64


def _prep(cs):
    return "tap_prep_conv_kernel" if cs.k > 1 and cs.prev_hw == 1 else "tap_prep_kernel"


def _layer(cs):
    import pytorch_bayesiancnn_b200 as bbb
    if cs.kind == "linear":
        return (bbb.BBBLRTLinear if cs.variant == "lrt" else bbb.BBBLinear)(cs.cin, cs.cout)
    cls = bbb.BBBLRTConv2d if cs.variant == "lrt" else bbb.BBBConv2d
    return cls(cs.cin, cs.cout, cs.k, stride=cs.s, padding=cs.p)


def _step(cs, m):
    from pytorch_bayesiancnn_b200 import fused, _lib as L
    st = fused._Step()
    st.layer, st.batch, st.conv = m, cs.B, m._conv_geometry()
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


def test_case_table_covers_every_branch():
    tap = [c for c in CASES if c.kind == "tap"]
    tg = tap + [c for c in CASES if c.kind == "linear"]
    assert {c.hw for c in tg} == {(1, 1), (2, 2), (4, 4), (8, 8), (4, 8)}
    assert {(c.k, c.s, c.p) for c in tap} == {(1, 1, 0), (3, 1, 0), (3, 1, 1), (5, 1, 2), (3, 2, 1)}
    assert {c.cin for c in tap} == {64, 128, 192, 256}
    assert {c.cout for c in tg if c.out == "packed"} >= {64, 128, 192, 320}
    assert {c.cout for c in tg if c.out == "f32"} >= {10, 72, 100}
    assert {(c.variant, c.act) for c in tg} == {(v, a) for v in ("bbb", "lrt") for a in ("none", "relu", "softplus")}
    assert {(c.variant, c.pool) for c in tap} == {(v, p) for v in ("bbb", "lrt") for p in (False, True)}
    assert {c.sq for c in tg if c.out == "packed"} == {False, True}
    assert {c.wide for c in tg} == {0, 1}
    assert {(c.pool, _tile_bn(c)) for c in tg if c.out == "packed"} == {(p, bn) for p in (False, True) for bn in (64, 128)}
    assert {c.B for c in tg} >= {1, 127, 128, 129, 300}
    # the bulk-copy store (unpooled packed, a full 128-row tile) and the direct store of a ragged last tile
    assert any(not c.pool and c.out == "packed" and c.B >= 128 and c.B % 128 for c in tg)
    assert {_prep(c) for c in tg} == {"tap_prep_conv_kernel", "tap_prep_kernel"}
    assert {c.prev_hw for c in tg if c.kind == "linear"} == {1, 4, 6, 8}
    gat = [c for c in CASES if c.kind == "gather"]
    assert {c.cin for c in gat} >= {1, 3, 16} and {c.hw for c in gat} >= {(8, 8), (4, 8)}
    assert {c.out for c in gat if c.pool} == {"packed", "f32"}
    s4 = [c for c in CASES if c.kind == "s4"]
    assert {c.cin for c in s4} == {1, 3, 4} and {(c.k, c.p) for c in s4} == {(11, 5), (7, 3)}
    assert {c.hw for c in s4} == {(32, 32), (48, 32), (64, 32)}      # 64x64 has OW = 16: the gather case above
    assert {c.B for c in s4} == {1, 15, 16, 17, 200}


# --------------------------------------------------------------------------------------------- per-layer GPU tests
_worst = collections.defaultdict(float)
GUARD = 64
SENTINEL = -1.25e37


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    yield torch.device("cuda:0")
    if _worst:
        lines = [f"  {fam:8s} worst |y - ref| / (C (M + |ref|)) = {v:.3f}" for fam, v in sorted(_worst.items())]
        sys.__stdout__.write("\n[fused geometry]\n" + "\n".join(lines) + "\n")


def _call(st, x, x_sq, y, y_sq, eps_a, eps_b, seed=0, stream=0):
    """One bbb_layer_forward_fused call, arguments as fused.run_step passes them; returns the KL scalar."""
    from pytorch_bayesiancnn_b200 import fused, functional as Fn, _lib as L
    m = st.layer
    dev = m.W_mu.device
    d = fused._step_desc(st, 0)
    kl = torch.empty((), dtype=torch.float32, device=dev)
    ws = Fn.workspace(dev, d, m)
    rc = L.lib().bbb_layer_forward_fused(
        C.byref(d), Fn._ptr(x), Fn._ptr(x_sq), st.in_layout, fused._in_pitch(st), st.prev_hw,
        Fn._ptr(m.W_mu), Fn._ptr(m.W_rho), Fn._ptr(m.bias_mu), Fn._ptr(m.bias_rho),
        Fn._ptr(y), Fn._ptr(y_sq), st.out_layout, fused._out_pitch(st), Fn._ptr(kl), Fn._ptr(eps_a), Fn._ptr(eps_b),
        C.c_uint64(seed), C.c_uint64(stream), None, Fn._ptr(ws), C.c_size_t(ws.numel()), Fn._stream(dev))
    L.check(rc, "bbb_layer_forward_fused")
    return kl


def _alloc_out(cs, st, dev):
    """(y, y_sq, n): a NaN-filled tiled buffer, or an fp32 buffer of n outputs + GUARD sentinel floats."""
    cout, oh, ow = st.out_chw
    if cs.out == "packed":
        planes = 2 if cs.sq else 1
        y = torch.full((R.tiled_rows(cs.B), cout * oh * ow * planes), float("nan"), dtype=torch.bfloat16, device=dev)
        return y, (y.view(-1)[8192:] if cs.sq else None), 0
    n = cs.B * cout * oh * ow
    y = torch.full((n + GUARD,), float("nan"), dtype=torch.float32, device=dev)
    y[n:] = SENTINEL
    return y, None, n


@pytest.mark.gpu
@pytest.mark.parametrize("cs", CASES, ids=[c.name for c in CASES])
def test_fused_layer_matches_float64_reference(dev, cs):
    from oracle import bbb_oracle as O
    from pytorch_bayesiancnn_b200 import _lib as L, philox_normal
    idx = CASES.index(cs)
    g = torch.Generator().manual_seed(1000 + idx)
    m = _layer(cs)
    with torch.no_grad():
        R.init_layer_params(m, m.W_mu[0].numel(), g)
    m = m.to(dev)
    st = _step(cs, m)
    if cs.kind in ("gather", "s4"):
        assert R.nchw_path(st) == cs.kind
    B, cout, (oh, ow) = cs.B, cs.cout, _out_hw(cs)

    # input: bf16-representable values; a packed input carries x^2 for an LRT layer, its padding rows are NaN
    if cs.kind == "linear":
        x = R.bf16(torch.randn(B, cs.cin, generator=g))                       # reference feature order c*HW + pix
        cols = x.view(B, cs.cin // cs.prev_hw, cs.prev_hw).transpose(1, 2).reshape(B, -1)
    else:
        x = R.bf16(torch.randn((B, cs.cin) + tuple(cs.hw), generator=g))
        cols = R.nchw_to_cols(x)
    if st.in_layout == L.LAYOUT_PACKED_BF16:
        xin = R.pack_tiled(cols, 2 if cs.variant == "lrt" else 1).to(dev)
        xin_sq = xin.view(-1)[8192:] if cs.variant == "lrt" else None
    else:
        xin, xin_sq = x.float().to(dev), None

    pre_shape = (B, cout) if cs.kind == "linear" else (B, cout, oh, ow)
    if cs.variant == "lrt":
        ea, eb = torch.randn(pre_shape, generator=g), None
    else:
        ea, eb = torch.randn(m.W_mu.shape, generator=g), torch.randn(cout, generator=g)
    conv = None if cs.kind == "linear" else ((cs.s, cs.s), (cs.p, cs.p))
    p = [t.detach().cpu() for t in (m.W_mu, m.W_rho, m.bias_mu, m.bias_rho)]
    ref, mag = R.layer_ref(x, *p, cs.variant, ea, eb, conv=conv, act=cs.act, pool=cs.pool)

    prev = L.lib().bbb_set_wide_tiles(cs.wide)
    try:
        y, y_sq, n = _alloc_out(cs, st, dev)
        kl = _call(st, xin, xin_sq, y, y_sq, ea.to(dev), None if eb is None else eb.to(dev))
        torch.cuda.synchronize()
        if cs.variant == "lrt":
            # in-kernel Philox vs the same stream drawn by philox_normal (NHWC-flat element index of the pre-pool output)
            seed, stream = 77, 500 + idx
            z = philox_normal(int(torch.Size(pre_shape).numel()), seed, stream, 0, device=dev)
            if cs.kind != "linear":
                z = z.view(B, oh, ow, cout).permute(0, 3, 1, 2)
            z = z.reshape(pre_shape).contiguous()
            y1, y1_sq, _ = _alloc_out(cs, st, dev)
            _call(st, xin, xin_sq, y1, y1_sq, None, None, seed, stream)
            y2, y2_sq, _ = _alloc_out(cs, st, dev)
            _call(st, xin, xin_sq, y2, y2_sq, z, None, seed, stream)
            torch.cuda.synchronize()
    finally:
        L.lib().bbb_set_wide_tiles(prev)

    fam = cs.kind
    if cs.out == "packed":
        F_ = st.out_chw[0] * st.out_chw[1] * st.out_chw[2]
        planes = 2 if cs.sq else 1
        refc = ref if cs.kind == "linear" else R.nchw_to_cols(ref)
        magc = mag if cs.kind == "linear" else R.nchw_to_cols(mag)
        yc = R.unpack_tiled(y, B, F_, planes)
        assert bool(torch.isfinite(yc).all()), "rows < B not all written / not finite"
        err = R.norm_err(yc, refc, magc)
        if cs.sq:
            ys = R.unpack_tiled(y, B, F_, planes, plane=1)
            assert bool(torch.isfinite(ys).all())
            err_sq = R.norm_err(ys, refc * refc, R.sq_mag(refc, magc))
            assert err_sq <= 1.0, f"x^2 plane: {err_sq:.3f}"
            _worst[fam + "^2"] = max(_worst[fam + "^2"], err_sq)
        pad = R.padding_bits(y, B, F_, planes)
        assert bool((pad == R.BF16_NAN_BITS).all()), "padding rows of the last row tile were written"
    else:
        out = y[:n].cpu().double().view(ref.shape)
        assert bool(torch.isfinite(out).all()), "outputs not all written / not finite"
        err = R.norm_err(out, ref, mag)
        assert bool((y[n:].cpu() == SENTINEL).all()), "the guard behind the fp32 output was written"
    _worst[fam] = max(_worst[fam], err)
    assert err <= 1.0, f"{cs.name}: normalised error {err:.3f}"

    kl_ref = float(O.kl_loss(*[t.double() for t in p], m.prior_mu, m.prior_sigma))
    assert abs(float(kl) - kl_ref) <= 1e-5 * abs(kl_ref), (float(kl), kl_ref)

    if cs.variant == "lrt":
        bits = torch.int16 if cs.out == "packed" else torch.int32
        assert torch.equal(y1.view(bits), y2.view(bits)), "in-kernel Philox noise differs from philox_normal"
        if cs.out == "packed":
            assert bool(torch.isfinite(R.unpack_tiled(y1, B, F_, planes)).all())


# --------------------------------------------------------------------------------------------- whole nets
@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["lrt", "bbb"])
@pytest.mark.parametrize("name", sorted(R.NETS) + sorted(R.REFUSED_NETS))
def test_whole_net_matches_float64_oracle(dev, name, variant):
    """The planner's wiring (layouts, pitches, prev_hw, y_sq selection) end to end: the fused chain (math='auto',
    no_grad) and the same net with fuse=False against an fp64 composition of the oracle's layers on identical eps.
    The nets the planner refuses must run unfused and still match."""
    import pytorch_bayesiancnn_b200 as bbb
    fusable = name in R.NETS
    shape, spec = R.NETS[name] if fusable else R.REFUSED_NETS[name]
    seed = sorted(list(R.NETS) + list(R.REFUSED_NETS)).index(name)
    net = R.make_net(spec, variant, seed=seed).to(dev)
    net.set_flag("math", "auto")
    x = R.bf16(torch.randn(shape, generator=torch.Generator().manual_seed(50 + seed))).float()
    eps = R.net_eps(net, shape, variant, seed=90 + seed)
    ref, kl_ref = R.net_ref(net, x, eps, variant)
    with torch.no_grad(), bbb.external_eps(eps):
        out, kl = net(x.to(dev))
    torch.cuda.synchronize()
    assert (net._fused_plans.get(tuple(shape)) is not None) == fusable
    assert tuple(out.shape) == tuple(ref.shape)
    assert bool(torch.isfinite(out).all())
    assert scale_err(out, ref) < 1e-2, scale_err(out, ref)
    assert abs(float(kl) - kl_ref) <= 1e-5 * abs(kl_ref)
    net.set_flag("fuse", False)
    with torch.no_grad(), bbb.external_eps(eps):
        out2, kl2 = net(x.to(dev))
    torch.cuda.synchronize()
    assert scale_err(out2, ref) < 1e-2, scale_err(out2, ref)
    assert abs(float(kl2) - kl_ref) <= 1e-5 * abs(kl_ref)

"""Host-side checks of the fused chain's geometry coverage (no GPU needed): the restated tiled packed layout, what
fused.plan builds for nets beyond BBBAlexNet and what it must refuse, and that the per-layer error bound of
tests/fused_ref.py is tight enough to catch plausible kernel bugs (each mutant of the reference breaks it 4x)."""
import pytest
import torch
import torch.nn.functional as F
from torch import nn

from tests import fused_ref as R


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()


# ------------------------------------------------------------------------------------------------------ layout
def test_tiled_index_hand_computed_offsets():
    idx = R.tiled_index(130, 128, 1)
    assert int(idx[0, 0]) == 0
    assert int(idx[0, 9]) == 9                                  # row 0: no swizzle
    assert int(idx[1, 0]) == 64 + 8                             # row 1, chunk 0 -> chunk 1
    assert int(idx[1, 8]) == 64                                 # row 1, chunk 1 -> chunk 0
    assert int(idx[3, 70]) == 8192 + 3 * 64 + (0 ^ 3) * 8 + 6   # second 64-column block
    assert int(idx[129, 5]) == 2 * 8192 + 64 + 8 + 5           # second 128-row block, after both column blocks
    idx2 = R.tiled_index(130, 128, 2, 0)
    sq = R.tiled_index(130, 128, 2, 1)
    assert int(idx2[0, 64]) == 2 * 8192                         # [x | x^2] blocks: 32 KB each
    assert torch.equal(sq - idx2, torch.full_like(sq, 8192))   # y_sq = y + 8192 elements


@pytest.mark.parametrize("B, F_, planes", [(1, 64, 1), (129, 192, 2), (256, 128, 1), (300, 320, 2)])
def test_pack_unpack_round_trip(B, F_, planes):
    g = torch.Generator().manual_seed(B)
    x = R.bf16(torch.randn(B, F_, generator=g))
    buf = R.pack_tiled(x, planes)
    assert buf.dtype == torch.bfloat16 and tuple(buf.shape) == (R.tiled_rows(B), F_ * planes)
    assert torch.equal(R.unpack_tiled(buf, B, F_, planes), x)
    if planes == 2:
        assert torch.equal(R.unpack_tiled(buf, B, F_, planes, plane=1), R.bf16(x * x))
    # a bijection: every element of the buffer is one (row, column, plane), the rows past B are padding
    all_idx = torch.cat([R.tiled_index(R.tiled_rows(B), F_, planes, p).reshape(-1) for p in range(planes)])
    assert torch.equal(all_idx.sort().values, torch.arange(buf.numel()))
    pad = R.padding_bits(buf, B, F_, planes)
    assert pad.numel() == (R.tiled_rows(B) - B) * F_ * planes
    assert bool((pad == R.BF16_NAN_BITS).all())


# ------------------------------------------------------------------------------------------------------ planner
_P, _N, _R = 1, 0, 2     # LAYOUT_PACKED_BF16, LAYOUT_NCHW_F32, LAYOUT_ROWMAJOR_F32
# per step: (in_layout, prev_hw, pool, out_layout, out_chw); the first step's NCHW kernel
EXPECTED = {
    "gray64": ("gather", [(_N, 1, True, _P, (64, 8, 8)), (_P, 1, True, _P, (128, 4, 4)),
                          (_P, 1, False, _P, (64, 2, 2)), (_P, 4, False, _R, (10, 1, 1))]),
    "gather_k1": ("gather", [(_N, 1, True, _P, (64, 4, 4)), (_P, 1, False, _P, (192, 4, 4)),
                             (_P, 1, False, _P, (128, 2, 2)), (_P, 4, False, _R, (100, 1, 1))]),
    "nonsquare": ("gather", [(_N, 1, False, _P, (64, 4, 8)), (_P, 1, True, _P, (64, 2, 4)),
                             (_P, 8, False, _R, (10, 1, 1))]),
    "s4_k7": ("s4", [(_N, 1, True, _P, (64, 6, 4)), (_P, 1, True, _P, (320, 3, 2)),
                     (_P, 6, False, _R, (72, 1, 1))]),
    "pool_last": ("s4", [(_N, 1, True, _P, (64, 4, 4)), (_P, 1, True, _N, (72, 2, 2))]),
}


@pytest.mark.parametrize("variant", ["lrt", "bbb"])
@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_planner_builds_the_expected_steps(built, name, variant):
    from pytorch_bayesiancnn_b200 import fused
    shape, spec = R.NETS[name]
    net = R.make_net(spec, variant)
    steps = fused.plan(list(net.children()), shape)
    path, want = EXPECTED[name]
    assert steps is not None, name
    got = [(st.in_layout, st.prev_hw, st.pool, st.out_layout, st.out_chw) for st in steps]
    assert got == want
    assert R.nchw_path(steps[0]) == path


def _refused_children(kind):
    from pytorch_bayesiancnn_b200.modules import BBBConv2d, BBBLinear, FlattenLayer
    if kind in R.REFUSED_NETS:
        return R.REFUSED_NETS[kind][0], list(R.make_net(R.REFUSED_NETS[kind][1], "bbb").children())
    if kind == "cin_not_multiple_of_64":         # a 96-channel map cannot be tiled into whole 64-column blocks
        return (4, 3, 8, 8), [BBBConv2d(3, 96, 3, padding=1), nn.ReLU(), BBBConv2d(96, 64, 3, padding=1),
                              nn.MaxPool2d(2, 2), FlattenLayer(1024), BBBLinear(1024, 10)]
    if kind == "dilation":
        return (4, 3, 8, 8), [BBBConv2d(3, 64, 3, padding=1), nn.ReLU(), BBBConv2d(64, 64, 3, padding=2, dilation=2),
                              FlattenLayer(4096), BBBLinear(4096, 10)]
    assert kind == "pool_3x3_stride2"
    return (4, 3, 8, 8), [BBBConv2d(3, 64, 3, padding=1), nn.ReLU(), nn.MaxPool2d(3, 2),
                          FlattenLayer(576), BBBLinear(576, 10)]


@pytest.mark.parametrize("kind", sorted(R.REFUSED_NETS) + ["cin_not_multiple_of_64", "dilation", "pool_3x3_stride2"])
def test_planner_refuses_what_the_engine_cannot_fuse(built, kind):
    from pytorch_bayesiancnn_b200 import fused
    shape, kids = _refused_children(kind)
    assert fused.plan(kids, shape) is None


# ------------------------------------------------------------------------------------------------------ bar sensitivity
def _conv_case(variant, seed=0, B=4, cin=64, cout=64, hw=4, bias_scale=0.5):
    g = torch.Generator().manual_seed(seed)
    x = R.bf16(torch.randn(B, cin, hw, hw, generator=g))
    K = cin * 9
    W_mu = torch.randn(cout, cin, 3, 3, generator=g) * K ** -0.5
    W_rho = torch.full((cout, cin, 3, 3), float(torch.log(torch.expm1(torch.tensor(0.5 * K ** -0.5)))))
    b_mu = bias_scale * torch.randn(cout, generator=g)
    b_rho = torch.full((cout,), -3.0)
    if variant == "lrt":
        eps_a, eps_b = torch.randn(B, cout, hw, hw, generator=g), None
    else:
        eps_a, eps_b = torch.randn(W_mu.shape, generator=g), torch.randn(cout, generator=g)
    return x, W_mu, W_rho, b_mu, b_rho, eps_a, eps_b


CONV = ((1, 1), (1, 1))


@pytest.mark.parametrize("variant", ["lrt", "bbb"])
def test_bar_catches_an_unswizzled_decode(variant):
    x, W_mu, W_rho, b_mu, b_rho, ea, eb = _conv_case(variant)
    ref, mag = R.layer_ref(x, W_mu, W_rho, b_mu, b_rho, variant, ea, eb, conv=CONV, act="relu", pool=True)
    cols = R.nchw_to_cols(ref)
    buf = R.pack_tiled(cols, 1)
    B, F_ = cols.shape
    assert R.norm_err(R.unpack_tiled(buf, B, F_), cols, R.nchw_to_cols(mag)) <= 1.0
    assert R.norm_err(R.unpack_tiled(buf, B, F_, swizzle=False), cols, R.nchw_to_cols(mag)) >= 4.0


def test_bar_catches_swapped_x_and_x_squared():
    x, W_mu, W_rho, b_mu, b_rho, ea, eb = _conv_case("lrt")
    x = x.abs()                                                    # a ReLU output: the swapped variance stays >= 0
    ref, mag = R.layer_ref(x, W_mu, W_rho, b_mu, b_rho, "lrt", ea, conv=CONV, act="softplus")
    mut, _ = R.layer_ref(R.bf16(x * x), W_mu, W_rho, b_mu, b_rho, "lrt", ea, conv=CONV, act="softplus", x_sq=x)
    assert R.norm_err(mut, ref, mag) >= 4.0


@pytest.mark.parametrize("variant", ["lrt", "bbb"])
@pytest.mark.parametrize("hw", [4, 6, 8])
def test_bar_catches_a_transposed_prev_hw_order(variant, hw):
    g = torch.Generator().manual_seed(hw)
    B, C_, N = 4, 64, 10
    xr = R.bf16(torch.randn(B, C_ * hw, generator=g))             # reference order: c * HW + pix
    W_mu = torch.randn(N, C_ * hw, generator=g) * (C_ * hw) ** -0.5
    W_rho = torch.full(W_mu.shape, -4.0)
    b_mu, b_rho = 0.5 * torch.randn(N, generator=g), torch.full((N,), -3.0)
    ea = torch.randn(B, N, generator=g) if variant == "lrt" else torch.randn(W_mu.shape, generator=g)
    eb = None if variant == "lrt" else torch.randn(N, generator=g)
    ref, mag = R.layer_ref(xr, W_mu, W_rho, b_mu, b_rho, variant, ea, eb)
    xt = xr.view(B, C_, hw).transpose(1, 2).reshape(B, -1)        # the packed order read as if it were the reference's
    mut, _ = R.layer_ref(xt, W_mu, W_rho, b_mu, b_rho, variant, ea, eb)
    assert R.norm_err(mut, ref, mag) >= 4.0


@pytest.mark.parametrize("variant", ["lrt", "bbb"])
@pytest.mark.parametrize("tap", [0, 4, 8])
def test_bar_catches_one_dropped_kernel_tap(variant, tap):
    # a non-negative input (a ReLU output) and weights of one sign make every tap a coherent part of the sum
    x, W_mu, W_rho, b_mu, b_rho, ea, eb = _conv_case(variant, seed=tap)
    x = x.abs()
    W_mu = W_mu.abs()
    ref, mag = R.layer_ref(x, W_mu, W_rho, b_mu, b_rho, variant, ea, eb, conv=CONV)
    W_cut, rho_cut = W_mu.clone(), W_rho.clone()
    W_cut[:, :, tap // 3, tap % 3] = 0.0
    rho_cut[:, :, tap // 3, tap % 3] = -200.0                      # sigma = 0: the tap contributes nothing
    mut, _ = R.layer_ref(x, W_cut, rho_cut, b_mu, b_rho, variant, ea, eb, conv=CONV)
    assert R.norm_err(mut, ref, mag) >= 4.0


@pytest.mark.parametrize("variant", ["lrt", "bbb"])
@pytest.mark.parametrize("act", ["none", "relu", "softplus"])
def test_bar_catches_a_pool_window_offset_by_one_pixel(variant, act):
    x, W_mu, W_rho, b_mu, b_rho, ea, eb = _conv_case(variant, hw=8)
    ref, mag = R.layer_ref(x, W_mu, W_rho, b_mu, b_rho, variant, ea, eb, conv=CONV, act=act, pool=True)
    pre, _ = R.layer_ref(x, W_mu, W_rho, b_mu, b_rho, variant, ea, eb, conv=CONV, act=act)
    shifted = F.pad(pre, (0, 1, 0, 1), value=float("-inf"))[..., 1:, 1:]
    mut = F.max_pool2d(shifted, 2, 2)
    assert R.norm_err(mut, ref, mag) >= 4.0


@pytest.mark.parametrize("variant", ["lrt", "bbb"])
def test_bar_catches_a_dropped_bias(variant):
    # bias of the same size as the weighted sum, as a trained layer's may be
    x, W_mu, W_rho, b_mu, b_rho, ea, eb = _conv_case(variant, bias_scale=2.0)
    ref, mag = R.layer_ref(x, W_mu, W_rho, b_mu, b_rho, variant, ea, eb, conv=CONV, act="relu")
    mut, _ = R.layer_ref(x, W_mu, W_rho, torch.zeros_like(b_mu), torch.full_like(b_rho, -200.0), variant,
                         ea, eb, conv=CONV, act="relu")
    assert R.norm_err(mut, ref, mag) >= 4.0

"""Host-side checks of the tensor-core backward (no GPU needed; the support queries need the built library).

functional._tc_wgrad and _tc_dgrad turn the weight and input gradients of a Bayesian layer into plain contractions
(functional._tc_contract) with the operands' roles swapped.  Here, for every case of tests/backward_ref.CASES:
  - with the contraction replaced by a float64 F.conv2d / F.linear, the decomposition equals torch.nn.grad exactly
    (to float64 summation order), so a wrong gradient on the GPU can only come from the kernel or the element-wise glue;
  - every contraction it issues is accepted by bbb_forward_supported in bf16 and tf32, except in the cases marked as
    falling back, where one is refused (or _tc_dgrad gives up) -- the layer then runs on the CUDA-core kernels.
test_case_table_reaches_every_branch checks that the table covers the branches of the decomposition and of the
CUDA-core kernels, and the last tests check the float64 reference of tests/backward_ref.py itself."""
import ctypes as C

import pytest
import torch

from tests import backward_ref as R


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()


def _features(cs):
    """What the decomposition of a case exercises."""
    calls, dgrad_none = R.contractions(cs)
    wg = [c for c in calls if c[0] == "wgrad"]
    f = {"chunks": len(wg), "ragged": len({c[1] for c in wg}) > 1, "dgrad_none": dgrad_none}
    if cs.k is not None:
        (sh, sw), (ph, pw), (dh, dw) = R.conv_of(cs)
        _, _, oh, ow = R.y_shape(cs)
        qh, qw = dh * (cs.k[0] - 1) - ph, dw * (cs.k[1] - 1) - pw
        hup, wup = cs.hw[0] - (dh * (cs.k[0] - 1) - 2 * ph), cs.hw[1] - (dw * (cs.k[1] - 1) - 2 * pw)
        f["q_negative"] = qh < 0 or qw < 0
        f["zero_insert"] = (sh, sw) != (1, 1) and (hup != (oh - 1) * sh + 1 or wup != (ow - 1) * sw + 1)
        f["stride_gt_kernel"] = sh > cs.k[0] or sw > cs.k[1]
    return f


def _supported(x_shape, w_shape, conv, math):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    d = Fn.make_desc(x_shape, w_shape, conv, L.VARIANT_BBB, False, False, 0.0, 1.0, math)
    return int(L.lib().bbb_forward_supported(C.byref(d))) == 0


@pytest.mark.parametrize("cs", R.CASES, ids=[c.name for c in R.CASES])
def test_every_contraction_is_accepted_unless_the_case_falls_back(built, cs):
    from pytorch_bayesiancnn_b200 import _lib as L
    calls, dgrad_none = R.contractions(cs)
    assert dgrad_none == (cs.fallback == "dgrad")
    for math in (L.MATH_BF16_TC, L.MATH_TF32_TC):
        ok = [_supported(x, w, conv, math) for _, x, w, conv in calls]
        refused = [c for c, o in zip(calls, ok) if not o]
        if cs.fallback == "wgrad":
            assert refused and all(c[0] == "wgrad" for c in refused), refused
        else:
            assert not refused, refused


def test_linear_wgrad_refusal_boundary(built):
    """K of the linear wgrad is the batch: 16384 is accepted, 16385 refused -- both bf16 and tf32."""
    from pytorch_bayesiancnn_b200 import _lib as L
    for math in (L.MATH_BF16_TC, L.MATH_TF32_TC):
        assert _supported((24, 16384), (5, 16384), None, math)
        assert not _supported((24, 16385), (5, 16385), None, math)


@pytest.mark.parametrize("cs", R.CASES, ids=[c.name for c in R.CASES])
def test_decomposition_equals_torch_nn_grad(cs):
    from pytorch_bayesiancnn_b200 import functional as Fn
    g = torch.Generator().manual_seed(R.CASES.index(cs))
    conv = R.conv_of(cs)
    x = torch.randn(R.x_shape(cs), generator=g, dtype=torch.float64)
    w = torch.randn(R.w_shape(cs), generator=g, dtype=torch.float64)
    gy = torch.randn(R.y_shape(cs), generator=g, dtype=torch.float64)
    with R.contract_with(R.contract):
        gw = Fn._tc_wgrad(x, gy, conv, w.shape)
        gx = Fn._tc_dgrad(gy, w, conv, x.shape)
    if conv is None:
        ref_w, ref_x = gy.t() @ x, gy @ w
        mag_w, mag_x = gy.abs().t() @ x.abs(), gy.abs() @ w.abs()
    else:
        s, p, d = conv
        ref_w = torch.nn.grad.conv2d_weight(x, w.shape, gy, s, p, d)
        ref_x = torch.nn.grad.conv2d_input(x.shape, w, gy, s, p, d)
        mag_w = torch.nn.grad.conv2d_weight(x.abs(), w.shape, gy.abs(), s, p, d)
        mag_x = torch.nn.grad.conv2d_input(x.shape, w.abs(), gy.abs(), s, p, d)
    assert gw.shape == ref_w.shape
    assert bool(((gw - ref_w).abs() <= 1e-13 * mag_w).all())
    if cs.fallback == "dgrad":
        assert gx is None
    else:
        assert gx.shape == ref_x.shape
        assert bool(((gx - ref_x).abs() <= 1e-13 * mag_x).all())


def test_case_table_reaches_every_branch():
    f = {cs.name: _features(cs) for cs in R.CASES}
    conv = [cs for cs in R.CASES if cs.k is not None]
    chunks = {f[cs.name]["chunks"] for cs in conv}
    assert 1 in chunks and max(chunks) >= 26                                  # one wgrad chunk, and many
    assert any(f[cs.name]["chunks"] == 4 and not f[cs.name]["ragged"] for cs in conv)   # AlexNet conv1 at B=512
    assert any(f[cs.name]["ragged"] for cs in conv)                           # a ragged last chunk
    assert any(f[cs.name]["zero_insert"] for cs in conv)                      # zero insertion padded to hup != OH
    assert any(f[cs.name]["q_negative"] for cs in conv)                       # _tc_dgrad gives up
    assert any(f[cs.name]["stride_gt_kernel"] for cs in conv)
    assert {cs.fallback for cs in R.CASES} == {None, "wgrad", "dgrad"}
    assert any(cs.fallback == "wgrad" and cs.k is None for cs in R.CASES)     # both wgrad refusals: linear and conv
    assert any(cs.fallback == "wgrad" and cs.k is not None for cs in R.CASES)
    K = lambda cs: cs.cin * (1 if cs.k is None else cs.k[0] * cs.k[1])
    assert any(cs.cout > 64 for cs in conv) and any(cs.cout > 64 for cs in R.CASES if cs.k is None)   # N > 64
    assert any(cs.cin > 64 for cs in conv)                                    # dgrad with Cin > 64
    assert any(K(cs) > 64 and cs.cout > 64 for cs in conv)                    # K > 64 with N > 64 on a conv
    assert any(K(cs) % 32 for cs in R.CASES) and any(K(cs) % 64 for cs in R.CASES)
    assert any(cs.B == 1 and cs.k is None for cs in R.CASES) and any(cs.B == 1 and cs.k is not None for cs in R.CASES)
    assert any(cs.cout == 1 for cs in R.CASES)
    assert any(cs.k is not None and (cs.k[0] != cs.k[1] or cs.s[0] != cs.s[1] or cs.p[0] != cs.p[1]
                                      or cs.d[0] != cs.d[1]) for cs in R.CASES)


# ------------------------------------------------------------------------------------------------ the reference itself
def _layer_inputs(variant, conv, bias, g, positive=False):
    f = (lambda t: t.abs()) if positive else (lambda t: t)
    x = f(torch.randn((3, 4, 7, 6) if conv else (5, 9), generator=g, dtype=torch.float64))
    ws = (5, 4, 3, 3) if conv else (6, 9)
    W_mu = f(torch.randn(ws, generator=g, dtype=torch.float64) * 0.3)
    W_rho = torch.randn(ws, generator=g, dtype=torch.float64) - 2.0
    b_mu = f(torch.randn(ws[0], generator=g, dtype=torch.float64)) if bias else None
    b_rho = torch.randn(ws[0], generator=g, dtype=torch.float64) - 2.0 if bias else None
    geom = ((2, 1), (1, 1), (1, 1)) if conv else None
    ys = R.contract(x, W_mu, geom).shape
    if variant == "bbb":
        eps = (f(torch.randn(ws, generator=g, dtype=torch.float64)),
               f(torch.randn(ws[0], generator=g, dtype=torch.float64)) if bias else None)
    else:
        eps = f(torch.randn(ys, generator=g, dtype=torch.float64))
    gout = f(torch.randn(ys, generator=g, dtype=torch.float64))
    return x, W_mu, W_rho, b_mu, b_rho, eps, gout, geom


@pytest.mark.parametrize("variant", ["bbb", "lrt"])
@pytest.mark.parametrize("conv", [True, False])
@pytest.mark.parametrize("bias", [True, False])
def test_bounds_dominate_and_are_tight(variant, conv, bias):
    """M >= |ref| everywhere, and M == ref when every input is positive (then no term cancels)."""
    g = torch.Generator().manual_seed(4 * (variant == "lrt") + 2 * conv + bias)
    args = _layer_inputs(variant, conv, bias, g)
    ref = R.grads(variant, *args[:-1], conv=args[-1])
    mag = R.bounds(variant, *args[:-1], conv=args[-1])
    for r, m in zip(ref, mag):
        if r is not None:
            assert bool((m >= r.abs() * (1 - 1e-12)).all())
    pos = _layer_inputs(variant, conv, bias, g, positive=True)
    ref = R.grads(variant, *pos[:-1], conv=pos[-1])
    mag = R.bounds(variant, *pos[:-1], conv=pos[-1])
    for r, m in zip(ref, mag):
        if r is not None:
            assert torch.allclose(r, m, rtol=1e-12, atol=0)


def test_operand_rounding_restatements():
    t = torch.tensor([1.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11,
                      -(1.0 + 2.0 ** -11), 1.0 + 2.0 ** -11 - 2.0 ** -23])
    # bf16: ties to even (1 + 2^-8 -> 1, 1 + 3*2^-8 -> 1 + 2^-6)
    assert R.round_bf16(t)[:3].tolist() == [1.0, 1.0, 1.0 + 2.0 ** -6]
    # tf32: ties away from zero (1 + 2^-11 -> 1 + 2^-10, 1 + 3*2^-11 -> 1 + 2^-9), below a tie rounds down
    assert R.round_tf32(t)[3:].tolist() == [1.0 + 2.0 ** -10, 1.0 + 2.0 ** -9, -(1.0 + 2.0 ** -10), 1.0]

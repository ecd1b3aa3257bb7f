"""Host-side checks of the per-layer forward's case table and reference (no GPU needed; the support queries need the
built library).

- Every case of tests/forward_ref.CASES is accepted or refused by bbb_forward_supported exactly as its row says, in
  every math mode, and the host restatement of tc_supported agrees with the engine.
- test_case_table_covers_every_branch: the table reaches every launch decision of the tensor-core forward (stage_x,
  ring depth, tile-image mode, ragged N and K for both operand types) and every CUDA-core tile configuration.
- The mutants: a reference with one plausible kernel bug built in breaks its tier by 4x or more at the table's shapes
  (batch cut down for the CPU), so each bar is tight enough to catch that bug.
- The reference itself: M bounds |ref| and equals it when every term is positive; var_x squares are exact."""
import ctypes as C

import pytest
import torch

from tests import forward_ref as R


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()


def _rc(cs, variant, math, sample=True):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    fold = None if cs.fold is None else (cs.fold[0], R.FOLD_STRIDE)
    d = Fn.make_desc(R.x_shape(cs), R.w_shape(cs), R.conv_of(cs), L.VARIANT_LRT if variant == "lrt" else L.VARIANT_BBB,
                     sample, cs.bias, 0.0, 0.1, L.MATH_BY_NAME[math], L.KL_BY_NAME[cs.kl], L.ACT_BY_NAME[cs.act],
                     fold=fold, first_image=0 if cs.fold is None else cs.fold[1])
    return int(L.lib().bbb_forward_supported(C.byref(d)))


@pytest.mark.parametrize("cs", R.CASES, ids=[c.name for c in R.CASES])
def test_support_is_as_the_row_says(built, cs):
    for variant in cs.variants:
        for math in R.MATHS + ("auto",):
            want_ok = math not in cs.refuse
            assert (_rc(cs, variant, math) == 0) == want_ok, (variant, math)
            if cs.fold is None and want_ok:
                assert _rc(cs, variant, math, sample=False) == 0, (variant, math, "sample=False")
    if cs.fold is None:
        assert R.tc_supported(cs) == ("bf16" not in cs.refuse)
    assert R.resolves(cs) in R.MATHS and R.resolves(cs) not in cs.refuse


def test_largest_tensor_core_k(built):
    """K = 16384 is the largest K the tensor cores take, for both variants (tc_supported sizes two planes): the LRT call
    runs a 2-stage ring in 231423 bytes of shared memory (of 227 KB), BBB a 4-stage one; K = 16385 is refused in bf16
    and tf32 and resolves to fp32 under auto."""
    big = next(c for c in R.CASES if c.name == "edge_lin_k16384")
    past = next(c for c in R.CASES if c.name == "edge_lin_k16385")
    for math in ("bf16", "tf32"):
        lrt = R.tc_launch(big, "lrt", True, math)
        assert lrt["stages"] == 2 and lrt["smem"] == 231423 and lrt["smem"] <= R.TC_SMEM_LIMIT, lrt
        assert R.tc_launch(big, "bbb", True, math)["stages"] == 4
    assert R.tc_supported(big) and not R.tc_supported(past)
    for variant in ("bbb", "lrt"):
        assert _rc(big, variant, "bf16") == 0 and _rc(big, variant, "tf32") == 0
        assert _rc(past, variant, "bf16") != 0 and _rc(past, variant, "tf32") != 0 and _rc(past, variant, "fp32") == 0
    assert R.resolves(past) == "fp32"


def _runs(cs):
    """(variant, sample, bias) of the calls the GPU test makes for a case (the mean path unfolded, then the sampled
    layer)."""
    return {(v, s, cs.bias) for v in cs.variants for s in (False, True)}


def test_case_table_covers_every_branch():
    tc = [(cs, v, s, m, R.tc_launch(cs, v, s, m)) for cs in R.CASES for v in cs.variants for s in (False, True)
          for m in ("bf16", "tf32") if m not in cs.refuse]
    assert {t["stage_x"] for *_, m, t in tc if m == "bf16"} == {0, 1, 2}
    assert {t["stage_x"] for *_, m, t in tc if m == "tf32"} == {0, 1}      # tf32 never stages x as bf16
    # LeNet conv1 LRT in bf16 stages x as bf16: x^2 is formed from the bf16 value there
    assert R.tc_launch(next(c for c in R.CASES if c.name == "lenet_conv1_b256"), "lrt", True, "bf16")["stage_x"] == 2
    assert {t["stages"] for *_, t in tc} == {2, 3, 4}
    assert {t["tile_mode"] for *_, t in tc} == {"divides", "large", "ragged"}
    assert {R.ohw_of(cs) for cs, *_ in tc} >= {784, 225, 100, 25}
    acc_tc = [cs for cs in R.CASES if "bf16" not in cs.refuse]
    assert any(cs.cout % 64 for cs in acc_tc)                                  # ragged N tile
    assert any(R.K_of(cs) % 64 for cs in acc_tc) and any(R.K_of(cs) % 32 for cs in acc_tc)   # ragged K, bf16 / tf32
    assert any(cs.cout % 4 and "lrt" in cs.variants for cs in acc_tc)         # Philox per element, N % 4 != 0
    assert {6, 10, 70, 100, 1000} <= {cs.cout for cs in R.CASES}
    simt = {R.simt_config(cs) for cs in R.CASES if "fp32" not in cs.refuse}
    assert simt == {(bn, lin) for bn in (16, 32, 64) for lin in (True, False)}
    runs = set().union(*(_runs(cs) for cs in R.CASES))
    assert runs == {(v, s, b) for v in ("bbb", "lrt") for s in (False, True) for b in (False, True)}
    folds = [cs for cs in R.CASES if cs.fold]
    assert any("bbb" in cs.variants for cs in folds) and any("lrt" in cs.variants for cs in folds)
    assert any(cs.fold[1] for cs in folds)                                     # a fold with a first image
    assert any(cs.B == 1 and cs.k is None for cs in R.CASES) and any(cs.B == 1 and cs.k for cs in R.CASES)
    assert {127, 128, 129} <= {cs.B * R.ohw_of(cs) for cs in R.CASES}
    assert any(cs.cout == 1 for cs in R.CASES)
    assert {cs.act for cs in R.CASES} == {"none", "relu", "softplus"} and {cs.kl for cs in R.CASES} == {"reference",
                                                                                                        "textbook"}
    assert any(cs.sparse for cs in R.CASES)
    assert any(cs.k and (cs.s[0] > cs.k[0] or cs.s[1] > cs.k[1]) for cs in R.CASES)
    assert any(cs.k and (cs.d != (1, 1)) for cs in R.CASES)
    assert any(cs.k and (cs.k[0] != cs.k[1] or cs.p[0] != cs.p[1]) for cs in R.CASES)
    Ks = {R.K_of(cs): cs for cs in R.CASES}
    assert "bf16" not in Ks[16384].refuse and set(Ks[16385].refuse) == {"bf16", "tf32"}
    assert any(cs.B * R.ohw_of(cs) * cs.cout * 4 > 2 ** 31 for cs in R.CASES)   # y past 2^31 bytes
    big = next(cs for cs in R.CASES if cs.B * R.ohw_of(cs) * cs.cout * 4 > 2 ** 31)
    per = R.ohw_of(big) * big.cout * 4
    assert any(i * per >= 2 ** 31 for i in R.check_images(big))


def test_check_images_cover_tile_and_sample_boundaries():
    cs = next(c for c in R.CASES if c.name == "3conv3fc_conv3_fold4x2048")
    im = set(R.check_images(cs))
    assert {0, cs.B - 1, 2047, 2048, 4095, 4096, 6143, 6144} <= im
    ohw = R.ohw_of(cs)
    assert {127 // ohw, 128 // ohw, (cs.B * ohw - 129) // ohw} <= im
    assert R.check_images(cs) == R.check_images(cs)
    small = next(c for c in R.CASES if c.name == "edge_lin_m129")
    assert R.check_images(small) == list(range(129))


# ------------------------------------------------------------------------------------------------ mutants
CPU_B = 2


def _inp(cs, variant, var_plane=False):
    g = torch.Generator().manual_seed(R.CASES.index(cs) * 2 + (variant == "lrt"))
    return R.make_inputs(cs, variant, g, B=min(cs.B, CPU_B), var_plane=var_plane)


def _drop_k_block(w, k0, k1):
    wf = w.reshape(w.shape[0], -1).clone()
    wf[:, k0:k1] = 0
    return wf.view(w.shape)


def _nhwc_roll(t):
    """The activation-shaped tensor read one NHWC pixel over (the eps of the neighbouring pixel, or image for OHW = 1)."""
    if t.dim() == 2:
        return t.roll(1, 0)
    B, N, H, W = t.shape
    return t.permute(0, 2, 3, 1).reshape(B * H * W, N).roll(1, 0).view(B, H, W, N).permute(0, 3, 1, 2)


@pytest.mark.parametrize("cs", R.CASES, ids=[c.name for c in R.CASES])
def test_mutants_break_their_tier(monkeypatch, cs):
    conv = R.conv_of(cs)
    x, W_mu, W_rho, b_mu, b_rho, eps = _inp(cs, "lrt")
    ref, M = R.mean_ref(x, W_mu, b_mu, conv, "fp32", cs.act)
    found = {}
    # one K block dropped (the last full one, or all of K < the block), in both block widths
    K = R.K_of(cs)
    for bk in (64, 32):
        k0 = max(0, (K // bk - 1) * bk)
        got, _ = R.mean_ref(x, _drop_k_block(W_mu, k0, min(K, k0 + bk)), b_mu, conv, "fp32", cs.act)
        found[f"dropped K block of {bk}"] = R.tight_err(got, ref, M)
    # one kernel tap swapped
    if cs.k is not None and cs.k != (1, 1):
        w = W_mu.clone()
        w[:, :, 0, 0], w[:, :, -1, -1] = W_mu[:, :, -1, -1], W_mu[:, :, 0, 0]
        found["swapped tap"] = R.tight_err(R.mean_ref(x, w, b_mu, conv, "fp32", cs.act)[0], ref, M)
    # the bias of the next column
    if cs.bias and cs.cout > 1:
        found["next column's bias"] = R.tight_err(R.mean_ref(x, W_mu, b_mu.roll(-1), conv, "fp32", cs.act)[0], ref, M)
    # LRT: eps of the neighbouring pixel
    ref, M, sd = R.layer_ref("lrt", x, W_mu, W_rho, b_mu, b_rho, eps, conv, True, cs.act)
    if eps.numel() // cs.cout >= 2:
        got = R.layer_ref("lrt", x, W_mu, W_rho, b_mu, b_rho, _nhwc_roll(eps), conv, True, cs.act)[0]
        found["eps of the neighbouring pixel"] = R.loose_err(got, ref, M, "bf16")
    # sigma without the softplus, both variants
    with monkeypatch.context() as mp:
        mp.setattr(R.O, "softplus_sigma", lambda rho: rho)
        got = R.layer_ref("lrt", x, W_mu, W_rho, b_mu, b_rho, eps, conv, True, cs.act)[0]
    found["sigma without softplus (lrt)"] = R.loose_err(got, ref, M, "bf16")
    xb, Wb, Rb, bb, brb, eb = _inp(cs, "bbb")
    refb, Mb, _ = R.layer_ref("bbb", xb, Wb, Rb, bb, brb, eb, conv, True, cs.act)
    with monkeypatch.context() as mp:
        mp.setattr(R.O, "softplus_sigma", lambda rho: rho)
        got = R.layer_ref("bbb", xb, Wb, Rb, bb, brb, eb, conv, True, cs.act)[0]
    found["sigma without softplus (bbb)"] = R.loose_err(got, refb, Mb, "bf16")
    # the 1e-16 dropped where the receptive field is zero
    if cs.sparse:
        var0 = sd.double() ** 2 - 1e-16
        sd0 = var0.clamp_min(0).sqrt()
        mean = R.layer_ref("lrt", x, W_mu, W_rho, b_mu, b_rho, eps, conv, False, "none")[0]
        found["1e-16 dropped (act_std)"] = R.std_err(sd0, sd, "bf16")
        found["1e-16 dropped (y)"] = R.loose_err(R.apply_act(mean + sd0 * eps.double(), cs.act), ref, M, "bf16")
    # x^2 of the neighbouring image, on the variance plane
    if min(cs.B, CPU_B) >= 2:
        xv, Wm, Wr, _, _, ev = _inp(cs, "lrt", var_plane=True)
        sd_ok = R.layer_ref("lrt", xv, Wm, Wr, None, None, ev, conv, True)[2]
        ok = R.var_plane_err(sd_ok, xv, Wr, conv, "fp32")
        assert max(ok) < 1e-6, ok                                           # the plain reference passes, with room
        sig2 = R.O.softplus_sigma(Wr.double()) ** 2
        bad = torch.sqrt(R.contract(xv.double().roll(1, 0) ** 2, sig2, None, conv) + 1e-16)
        found["x^2 of the neighbouring image"] = R.var_plane_err(bad, xv, Wr, conv, "fp32")[0]
    for what, e in found.items():
        assert e >= 4, (cs.name, what, e)


# ------------------------------------------------------------------------------------------------ the reference itself
@pytest.mark.parametrize("variant", ["bbb", "lrt"])
@pytest.mark.parametrize("name", ["edge_rect_asym", "edge_lin_k100_n70", "lenet_conv1_b256"])
def test_magnitude_bounds_and_is_tight(variant, name):
    """M >= |ref| everywhere, and M == ref when every input (and eps) is positive."""
    cs = next(c for c in R.CASES if c.name == name)
    x, W_mu, W_rho, b_mu, b_rho, eps = _inp(cs, variant)
    ref, M, sd = R.layer_ref(variant, x, W_mu, W_rho, b_mu, b_rho, eps, R.conv_of(cs))
    assert bool((M >= ref.abs() * (1 - 1e-12)).all())
    pos = lambda t: None if t is None else (tuple(pos(u) for u in t) if isinstance(t, tuple) else t.abs())
    ref, M, sd = R.layer_ref(variant, pos(x), pos(W_mu), W_rho, pos(b_mu), b_rho, pos(eps), R.conv_of(cs))
    assert torch.allclose(ref, M, rtol=1e-12, atol=0)
    assert (sd is None) == (variant == "bbb")


def test_var_x_squares_are_exact_in_bf16_and_tf32():
    x = R.var_x((4096,), torch.Generator().manual_seed(0)).double()
    for r in (R.round_bf16, R.round_tf32):
        assert torch.equal(r(x), x) and torch.equal(r(x * x), x * x)
    assert len(set(x.abs().tolist())) > 30 and bool((x < 0).any())

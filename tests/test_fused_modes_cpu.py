"""Host-side checks of the fused chain's mode coverage (no GPU needed): that tests/test_gpu_fused_modes.py reaches every
weight-prep kernel in every variant and prior mode, what bbb_fused_supported must refuse, and that the float64 bars it
uses are tight enough to catch a plausible mode bug (each mutant of the reference breaks its bar 4x, at the parameters
of tests/fused_ref.init_layer_params)."""
import pytest
import torch

from tests import fused_ref as R
from tests import mask_ref as MR
from tests.fused_ref import CASES

PREPS = ("tap_prep_conv_kernel", "tap_prep_kernel", "conv_s4_prep_kernel", "weight_prep_kernel")
PRIORS = ("scalar", "TP", "MK", "TP+MK")


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()


def _fold_batch(cs):
    """The folded batch test_gpu_fused_modes runs (_Layer.fold_rows)."""
    if cs.variant == "lrt":
        return cs.B * 3
    return (256 if cs.B > 128 else 128) * 2


# ------------------------------------------------------------------------------------------------------ coverage
def test_modes_reach_every_prep_variant_and_prior():
    """{prep} x {LRT, BBB, BBB fold} x {scalar, TP, MK, TP+MK}: the mask and prior tests run every case, and every BBB
    case the engine folds folded as well; the gather weight_prep has no fold (the engine refuses one)."""
    reached = set()
    for cs in CASES:
        reached |= {(R._prep(cs), cs.variant, p) for p in PRIORS}
        if cs.variant == "bbb" and R.folds(cs):
            reached |= {(R._prep(cs, _fold_batch(cs)), "bbb fold", p) for p in PRIORS}
    want = {(k, v, p) for k in PREPS for v in ("lrt", "bbb", "bbb fold") for p in PRIORS}
    want -= {("weight_prep_kernel", "bbb fold", p) for p in PRIORS}
    assert reached == want, sorted(want - reached)


def test_modes_reach_the_branches_alexnet_does_not_have():
    bbb = [c for c in CASES if c.variant == "bbb"]
    conv_fold = [c for c in bbb if R.folds(c) and R._prep(c, _fold_batch(c)) == "tap_prep_conv_kernel"]
    # tap_prep_conv_kernel's fold: phase 2 with n >= N (Cout 72, 10), four K blocks, staging opted in above 48 KB
    assert {c.cout for c in conv_fold} >= {10, 72}
    assert 256 in {c.cin for c in conv_fold}
    assert any(c.k == 5 and R.fold_staging_bytes(c, _fold_batch(c)) > 48 * 1024 for c in conv_fold)
    # tap_prep_kernel's fold and in-kernel noise with the prev_hw reorder
    assert {c.prev_hw for c in bbb if c.kind == "linear"} >= {4, 6, 8}
    assert {c.cout for c in bbb if c.out == "f32"} >= {10, 72, 100}
    # LRT folds whose ragged 128-row tiles straddle two samples
    assert any(c.variant == "lrt" and c.kind in ("tap", "linear") and c.B % 128 for c in CASES)
    # the largest first image of one s4, one tap and one linear LRT case
    from tests.test_gpu_fused_modes import LAST_IMAGE_CASES
    assert {c.kind for c in LAST_IMAGE_CASES} == {"s4", "tap", "linear"}


# ------------------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize("cs", CASES, ids=[c.name for c in CASES])
def test_bbb_fused_supported_refusals(built, cs):
    m = R._layer(cs)
    st = R._step(cs, m)
    assert R.fused_supported(st) == 0
    rows = cs.B
    if not R.folds(cs):
        assert R.fused_supported(R._step(cs, m, rows * 2), fold=(rows, 1 << 40)) == -2       # no fold on the gather path
    else:
        B = _fold_batch(cs)
        S = 3 if cs.variant == "lrt" else 2
        frows = B // S
        assert R.fused_supported(R._step(cs, m, B), fold=(frows, 1 << 40)) == 0
        assert R.fused_supported(R._step(cs, m, B), fold=(frows, 1 << 40), sample=False) == -2   # a mean-only call
        nrows = max(frows, 2)
        assert R.fused_supported(R._step(cs, m, nrows * S + 1), fold=(nrows, 1 << 40)) == -1     # batch % rows
        if cs.variant == "bbb":
            assert R.fused_supported(R._step(cs, m, 128), fold=(64, 1 << 40)) == -2             # rows % 128
            assert R.fused_supported(R._step(cs, m, 384), fold=(192, 1 << 40)) == -2
    fi = R.first_image_max(cs, cs.B)
    assert R.fused_supported(st, first_image=fi) == 0
    assert R.fused_supported(st, first_image=fi + 1) == -1


# ------------------------------------------------------------------------------------------------------ bar sensitivity
def _case(name):
    return next(c for c in CASES if c.name == name)


def _setup(cs, seed=0, bias_sigma=None):
    """(x, params, conv, generator) of a case at the parameters the GPU tests use (float64, CPU)."""
    g = torch.Generator().manual_seed(seed)
    m = R._layer(cs)
    with torch.no_grad():
        R.init_layer_params(m, m.W_mu[0].numel(), g, bias_sigma)
    p = [t.detach().cpu().double() for t in (m.W_mu, m.W_rho, m.bias_mu, m.bias_rho)]
    shape = (cs.B, cs.cin) if cs.kind == "linear" else (cs.B, cs.cin) + tuple(cs.hw)
    x = R.bf16(torch.randn(shape, generator=g))
    conv = None if cs.kind == "linear" else ((cs.s, cs.s), (cs.p, cs.p))
    return x, p, conv, g


def _act_shape(cs):
    oh, ow = R._out_hw(cs)
    return (cs.cout,) if cs.kind == "linear" else (cs.cout, oh, ow)


def _ref(cs, x, p, conv, ea, eb):
    return R.layer_ref(x, *p, cs.variant, ea, eb, conv=conv, act=cs.act, pool=cs.pool)


MUTANT_CASES = ["t4x4_nchw10_lrt", "t2x2_nchw10_bbb", "l_prev8_n10_lrt", "l_prev4_packed_bbb", "s_c3_k11_32x32_b17_lrt",
                "s_c4_k11_48x32_b17_bbb"]


@pytest.mark.parametrize("name", MUTANT_CASES)
def test_bar_catches_a_sample_drawn_on_the_previous_stream(name):
    cs = _case(name)
    x, p, conv, g = _setup(cs)
    if cs.variant == "lrt":
        e = [torch.randn((cs.B,) + _act_shape(cs), generator=g) for _ in range(2)]        # samples j - 1 and j
        ref, mag = _ref(cs, x, p, conv, e[1], None)
        mut, _ = _ref(cs, x, p, conv, e[0], None)
    else:
        e = [(torch.randn(p[0].shape, generator=g), torch.randn(cs.cout, generator=g)) for _ in range(2)]
        ref, mag = _ref(cs, x, p, conv, *e[1])
        mut, _ = _ref(cs, x, p, conv, *e[0])
    assert R.norm_err(mut, ref, mag) >= 4.0


@pytest.mark.parametrize("name", MUTANT_CASES)
@pytest.mark.parametrize("frac", [0.5, 0.95])
def test_bar_catches_a_mask_shifted_by_one_element(name, frac):
    cs = _case(name)
    x, p, conv, g = _setup(cs)
    wm = torch.rand(p[0].shape, generator=g) >= frac
    ea = torch.randn((cs.B,) + _act_shape(cs) if cs.variant == "lrt" else p[0].shape, generator=g)
    eb = None if cs.variant == "lrt" else torch.randn(cs.cout, generator=g)
    ref, mag = _ref(cs, x, MR.masked_params(*p, wm), conv, ea, eb)
    shifted = wm.reshape(-1).roll(1).view(wm.shape)
    mut, _ = _ref(cs, x, MR.masked_params(*p, shifted), conv, ea, eb)
    assert R.norm_err(mut, ref, mag) >= 4.0


@pytest.mark.parametrize("name", [c.name for c in CASES if c.kind == "linear" and c.prev_hw > 1])
def test_bar_catches_a_mask_in_packed_order(name):
    cs = _case(name)
    x, p, conv, g = _setup(cs)
    wm = torch.rand(p[0].shape, generator=g) >= 0.5
    ea = torch.randn((cs.B, cs.cout) if cs.variant == "lrt" else p[0].shape, generator=g)
    eb = None if cs.variant == "lrt" else torch.randn(cs.cout, generator=g)
    ref, mag = _ref(cs, x, MR.masked_params(*p, wm), conv, ea, eb)
    # the mask's feature k' = pix * C + c of the packed input read as the reference's k = c * HW + pix
    hw = cs.prev_hw
    packed = wm.view(cs.cout, hw, cs.cin // hw).transpose(1, 2).reshape(wm.shape)
    mut, _ = _ref(cs, x, MR.masked_params(*p, packed), conv, ea, eb)
    assert R.norm_err(mut, ref, mag) >= 4.0


@pytest.mark.parametrize("name", MUTANT_CASES)
@pytest.mark.parametrize("convention", ["reference", "textbook"])
@pytest.mark.parametrize("masked", [False, True])
def test_kl_bar_catches_a_prior_read_one_element_off(name, convention, masked):
    cs = _case(name)
    _, p, _, g = _setup(cs)
    sp = torch.nn.functional.softplus
    pri = (p[0] + 0.05 * torch.randn(p[0].shape, generator=g).double(),
           sp(p[1] + 0.5 * torch.randn(p[1].shape, generator=g).double()),
           p[2] + 0.05 * torch.randn(p[2].shape, generator=g).double(),
           sp(p[3] + 0.5 * torch.randn(p[3].shape, generator=g).double()))
    wm = (torch.rand(p[0].shape, generator=g) >= 0.5) if masked else torch.ones(p[0].shape, dtype=torch.bool)
    ref = float(MR.kl_ref(*p, wm, None, 0.0, 0.1, convention, prior=pri))
    off = tuple(t.reshape(-1).roll(1).view(t.shape) for t in pri)
    mut = float(MR.kl_ref(*p, wm, None, 0.0, 0.1, convention, prior=off))
    assert abs(mut - ref) >= 4 * 1e-5 * abs(ref)


@pytest.mark.parametrize("name", [c.name for c in CASES if c.variant == "bbb"])
def test_bar_catches_the_bias_eps_one_element_early(name):
    """eps_b[n] from Philox element N*K + n - 1 (the last weight's for n = 0) instead of N*K + n, at the bias sigma of
    the GPU BBB noise test."""
    from tests.test_gpu_fused_modes import BIAS_SIGMA
    cs = _case(name)
    if cs.kind == "s4" and cs.B > 17:
        pytest.skip("covered by the smaller stride-4 cases")
    x, p, conv, g = _setup(cs, bias_sigma=BIAS_SIGMA)
    nk = p[0].numel()
    z = torch.randn(nk + cs.cout, generator=g)
    ref, mag = _ref(cs, x, p, conv, z[:nk].view(p[0].shape), z[nk:])
    mut, _ = _ref(cs, x, p, conv, z[:nk].view(p[0].shape), z[nk - 1:nk - 1 + cs.cout])
    assert R.norm_err(mut, ref, mag) >= 4.0


@pytest.mark.parametrize("name", [n for n in MUTANT_CASES if n.endswith("_lrt")])
def test_bar_catches_lrt_noise_one_image_off(name):
    cs = _case(name)
    x, p, conv, g = _setup(cs)
    z = torch.randn((cs.B + 1,) + _act_shape(cs), generator=g)           # images first_image - 1 ... first_image + B - 1
    ref, mag = _ref(cs, x, p, conv, z[1:], None)
    mut, _ = _ref(cs, x, p, conv, z[:-1], None)
    assert R.norm_err(mut, ref, mag) >= 4.0

"""Host-side answers for the folded training step (MCTrainStep(fold=True)): how mc.train_fold_groups groups a rank's
samples, which layer calls layer_fold(grad=True) refuses, the per-group KL weights, and the refusals of
bbb_lrt_noise_grad that need no GPU.  Only host-only queries of the built library; no GPU needed."""
import ctypes as C
import math

import pytest

from tests import backward_ref as R
from tests.util import CFG_PRIORS

STRIDE = 1 << 40
NETS = (("alexnet", 3), ("lenet", 3), ("3conv3fc", 1))


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()


def _net(key, inputs, variant, math_name):
    from pytorch_bayesiancnn_b200.models import get_model
    net = get_model(key, inputs, 10, CFG_PRIORS, variant, "softplus")
    net.set_flag("math", math_name)
    return net


@pytest.mark.parametrize("key,inputs", NETS)
@pytest.mark.parametrize("variant", ["lrt", "bbb"])
@pytest.mark.parametrize("math_name", ["bf16", "tf32", "fp32"])
@pytest.mark.parametrize("B", [256, 300])
def test_planner_folds_lrt_on_tensor_cores_only(built, key, inputs, variant, math_name, B):
    """10 local samples: every LRT net on a tensor-core math mode takes them in one group of 10 (the budget, the int32
    cap and the backward's row limits all allow it); BBB nets and fp32 keep the sample loop."""
    from pytorch_bayesiancnn_b200 import mc
    net = _net(key, inputs, variant, math_name)
    groups = mc.train_fold_groups(net, (B, inputs, 32, 32), 10, STRIDE)
    if variant == "lrt" and math_name != "fp32":
        assert groups == [(0, 10)], groups
    else:
        assert groups is None


def test_planner_respects_fold_group_and_first_image(built):
    from pytorch_bayesiancnn_b200 import mc
    net = _net("lenet", 3, "lrt", "bf16")
    assert mc.train_fold_groups(net, (256, 3, 32, 32), 5, STRIDE, fold_group=2) == [(0, 2), (2, 2), (4, 1)]
    assert mc.train_fold_groups(net, (128, 3, 32, 32), 4, 2 * STRIDE, first_image=128) == [(0, 4)]
    assert mc.train_fold_groups(net, (256, 3, 32, 32), 1, STRIDE) is None          # one sample: nothing to fold
    assert mc.train_fold_groups(net, (256, 3, 32, 32), 5, STRIDE, fold_group=1) is None


def test_planner_limits_the_rows_of_a_linear_weight_gradient(built):
    """BBBLeNet at B = 2000 rows: one group of 10 samples would give the linear layers' weight gradients K = 20000 rows,
    above the 16384 the contraction takes, so the planner splits into groups whose G x B fits (2 x 5)."""
    from pytorch_bayesiancnn_b200 import mc
    net = _net("lenet", 3, "lrt", "bf16")
    groups = mc.train_fold_groups(net, (2000, 3, 32, 32), 10, STRIDE)
    assert groups == [(0, 5), (5, 5)], groups
    G = max(n for _, n in groups)
    assert G * 2000 <= 16384 < 10 * 2000
    # the same refusal, asked directly of the layer: fc1 (400 -> 120) at 10 x 2000 rows
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    cfg = net.fc1._cfg(True)
    assert Fn._fold_grad_refusal(cfg, (20000, 400), (120, 400), True) is not None
    assert Fn._fold_grad_refusal(cfg, (10000, 400), (120, 400), True) is None


def test_planner_caps_before_the_int32_limit(built):
    """BBB3Conv3FC on 1x32x32 at 2048 rows with a budget that allows everything: the int32 element cap of conv1's output
    (2048 x 32 x 32 x 32 = 2^26 elements) would allow 31 samples, but the linear layers' weight gradients take at most
    16384 rows, so groups hold 8."""
    from pytorch_bayesiancnn_b200 import mc
    net = _net("3conv3fc", 1, "lrt", "bf16")
    assert ((1 << 31) - 1) // (2048 * 32 * 32 * 32) == 31
    groups = mc.train_fold_groups(net, (2048, 1, 32, 32), 40, STRIDE, budget=1 << 40)
    assert groups == [(8 * i, 8) for i in range(5)], groups


def test_kl_weights_sum_to_the_sample_loop(built):
    from pytorch_bayesiancnn_b200 import mc
    for n_local in range(2, 30):
        for g in range(2, 9):
            groups = mc.layer_fold_groups(n_local, 1, 1, fold_group=g)
            for beta, S in ((0.1, 30), (1.0, n_local), (2.5e-4, 100)):
                w = mc.train_fold_kl_weights(groups, beta, S)
                assert [x / (beta / S) for x in w] == pytest.approx([n for _, n in groups], rel=1e-12)
                assert math.isclose(sum(w), n_local * beta / S, rel_tol=1e-12)


@pytest.mark.parametrize("cs", R.CASES, ids=[c.name for c in R.CASES])
def test_fold_grad_refuses_exactly_the_fallback_cases(built, cs):
    """layer_fold(grad=True) refuses a call whose tensor-core backward would fall back to the CUDA-core kernels (they
    do not know the fold) -- the fallback column of the backward case table -- and accepts the rest, in bf16 and tf32."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    for m in (L.MATH_BF16_TC, L.MATH_TF32_TC):
        cfg = {"variant": L.VARIANT_LRT, "math": m, "conv": R.conv_of(cs)}
        why = Fn._fold_grad_refusal(cfg, R.x_shape(cs), R.w_shape(cs), True)
        assert (why is not None) == (cs.fallback is not None), (cs.name, why)
        assert (Fn.tc_backward_refusal(R.x_shape(cs), R.w_shape(cs), R.conv_of(cs), m) is None) == (why is None)


def test_fold_grad_refuses_bbb_and_fp32(built):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    conv = ((1, 1), (0, 0), (1, 1))
    shapes = ((256, 3, 32, 32), (6, 3, 5, 5))
    assert "BBB" in Fn._fold_grad_refusal({"variant": L.VARIANT_BBB, "math": L.MATH_BF16_TC, "conv": conv}, *shapes, True)
    assert "fp32" in Fn._fold_grad_refusal({"variant": L.VARIANT_LRT, "math": L.MATH_FP32, "conv": conv}, *shapes, True)
    assert Fn._fold_grad_refusal({"variant": L.VARIANT_LRT, "math": L.MATH_AUTO, "conv": conv}, *shapes, True) is None


def test_contraction_list_matches_the_backward(built):
    """The host-only list of contractions is what _tc_wgrad and _tc_dgrad issue (tests/backward_ref.contractions)."""
    from pytorch_bayesiancnn_b200 import functional as Fn
    for cs in R.CASES:
        calls, dgrad_none = R.contractions(cs)
        got = Fn._tc_backward_contractions(R.x_shape(cs), R.w_shape(cs), R.conv_of(cs))
        if dgrad_none:
            assert got is None
        else:
            assert got == list(dict.fromkeys((x, w, cv) for _, x, w, cv in calls)), cs.name
        wg = Fn._tc_backward_contractions(R.x_shape(cs), R.w_shape(cs), R.conv_of(cs), need_x=False)
        assert wg == list(dict.fromkeys((x, w, cv) for role, x, w, cv in calls if role == "wgrad")), cs.name


def _noise_grad_rc(desc):
    from pytorch_bayesiancnn_b200 import _lib as L
    lib = L.lib()
    rc = int(lib.bbb_lrt_noise_grad(C.byref(desc), None, None, C.c_uint64(1), C.c_uint64(2), None, None, None))
    return rc, lib.bbb_last_error().decode()


def test_lrt_noise_grad_refusals(built):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    conv = ((1, 1), (0, 0), (1, 1))
    mk = lambda variant=L.VARIANT_LRT, sample=True, B=512, fold=None, first=0, xs=(3, 32, 32): Fn.make_desc(
        (B,) + xs, (6, xs[0], 5, 5), conv, variant, sample, True, 0.0, 0.1, L.MATH_BF16_TC, fold=fold, first_image=first)
    rc, msg = _noise_grad_rc(mk(variant=L.VARIANT_BBB))
    assert rc == -1 and "LRT" in msg
    rc, msg = _noise_grad_rc(mk(sample=False))
    assert rc == -2 and "sample" in msg
    rc, msg = _noise_grad_rc(mk(fold=(200, STRIDE)))                  # 512 rows are not whole samples of 200
    assert rc == -1 and "multiple" in msg
    # first image: (first + rows) x OH x OW x Cout must stay an int32 count (28 x 28 x 6 = 4704 per image)
    last_ok = ((1 << 31) - 1) // 4704 - 256
    rc, msg = _noise_grad_rc(mk(B=256, first=last_ok + 1))
    assert rc == -1 and "first image" in msg
    rc, msg = _noise_grad_rc(mk(B=256, first=last_ok))
    assert rc == -1 and "NULL" in msg                                # accepted up to the pointers
    # a fold counts the rows of one sample: the same first image passes with 256-row samples of a larger batch
    assert "NULL" in _noise_grad_rc(mk(B=512, first=last_ok, fold=(256, STRIDE)))[1]
    assert "first image" in _noise_grad_rc(mk(B=512, first=last_ok + 1, fold=(256, STRIDE)))[1]
    # a fold whose whole batch passes int32 counts is an invalid geometry
    rc, msg = _noise_grad_rc(mk(B=256 * -(-((1 << 31) // 4704 + 1) // 256), fold=(256, STRIDE)))
    assert rc == -1 and "geometry" in msg
    rc, msg = _noise_grad_rc(mk())
    assert rc == -1 and "NULL" in msg

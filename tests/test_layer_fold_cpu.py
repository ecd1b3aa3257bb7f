"""Host-side answers for folding the Monte-Carlo samples of BBBLeNet / BBB3Conv3FC into passes of the per-layer
tensor-core kernel: what bbb_forward_supported accepts, how bbb_workspace_bytes grows, and how MCForward groups a
rank's samples.  No GPU needed."""
import ctypes as C
import math

import pytest

from tests.util import CFG_PRIORS

STRIDE = 1 << 40
NETS = (("lenet", 1), ("3conv3fc", 1))             # MNIST-shaped inputs, as uncertainty_estimation.py uses them


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()


def _layers(key, variant, inputs, batch):
    """(layer, input shape) of every Bayesian layer of the net on a batch of `batch` 32x32 images."""
    from pytorch_bayesiancnn_b200 import mc, models as M
    cls = {"lenet": M.BBBLeNet, "3conv3fc": M.BBB3Conv3FC}[key]
    net = cls(10, inputs, CFG_PRIORS, variant, "softplus")
    chain = mc._per_image_chain(list(net.children()), (batch, inputs, 32, 32))
    assert chain is not None
    return chain


def _desc(m, xs, fold, math=None, sample=True):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    cfg = m._cfg(True)
    return Fn.make_desc(tuple(xs), tuple(m.W_mu.shape), cfg["conv"], cfg["variant"], sample, m.bias_mu is not None,
                        cfg["prior_mu"], cfg["prior_sigma"], cfg["math"] if math is None else math,
                        cfg["kl_convention"], cfg["act"], fold=fold)


def _rc(d):
    from pytorch_bayesiancnn_b200 import _lib as L
    return int(L.lib().bbb_forward_supported(C.byref(d)))


@pytest.mark.parametrize("key,inputs", NETS)
def test_forward_supported_answers_for_folded_layers(built, key, inputs):
    from pytorch_bayesiancnn_b200 import _lib as L
    S = 3
    for variant in ("lrt", "bbb"):
        for rows in (200, 256, 2048):
            layers, _, _ = _layers(key, variant, inputs, S * rows)
            assert len(layers) == 5 if key == "lenet" else len(layers) == 6
            # LRT folds any rows that divide the batch; BBB needs every 128-row tile inside one sample (B = 200: no)
            want = -2 if (variant == "bbb" and rows == 200) else 0
            rcs = [_rc(_desc(m, xs, (rows, STRIDE))) for m, xs in layers]
            if want == 0:
                assert rcs == [0] * len(layers), (variant, rows, rcs, L.lib().bbb_last_error())
            else:
                assert -2 in rcs and set(rcs) <= {0, -2}, (variant, rows, rcs)
                assert rcs[-1] == -2                          # a linear layer at 200 rows per sample
            for m, xs in layers:
                assert _rc(_desc(m, xs, None)) == 0           # unfolded: as before
        layers, _, _ = _layers(key, variant, inputs, S * 256 + 128)
        for m, xs in layers:                                  # not a whole number of samples
            assert _rc(_desc(m, xs, (256, STRIDE))) == -1
        layers, _, _ = _layers(key, variant, inputs, S * 256)
        for m, xs in layers:
            assert _rc(_desc(m, xs, (256, STRIDE), math=L.MATH_FP32)) == -2      # the CUDA-core path does not fold
            assert _rc(_desc(m, xs, (256, STRIDE), math=L.MATH_TF32_TC)) == 0    # tf32 uses the same kernel
            assert _rc(_desc(m, xs, (256, STRIDE), sample=False)) == -2          # a mean-only call has no samples


@pytest.mark.parametrize("key,inputs", NETS)
def test_workspace_grows_by_the_sample_count_for_bbb_only(built, key, inputs):
    from pytorch_bayesiancnn_b200 import _lib as L
    lib = L.lib()
    fp32 = L.LayerDesc()
    fp32.math = L.MATH_FP32
    off = (int(lib.bbb_workspace_bytes(C.byref(fp32))) + 1023) // 1024 * 1024    # where the operand sets start
    S = 4
    for variant in ("lrt", "bbb"):
        layers, _, _ = _layers(key, variant, inputs, S * 256)
        for m, xs in layers:
            one = int(lib.bbb_workspace_bytes(C.byref(_desc(m, xs, None))))
            folded = int(lib.bbb_workspace_bytes(C.byref(_desc(m, xs, (256, STRIDE)))))
            if variant == "bbb":
                assert folded == off + S * ((one - off + 1023) // 1024 * 1024), (xs, one, folded)
            else:
                assert folded == one


def test_unfolded_descs_keep_reserved_zero(built):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    for variant in (L.VARIANT_LRT, L.VARIANT_BBB):
        d = Fn.make_desc((8, 3, 32, 32), (6, 3, 5, 5), ((1, 1), (0, 0), (1, 1)), variant, True, True, 0.0, 0.1,
                         L.MATH_AUTO)
        assert list(d.reserved) == [0, 0, 0, 0]
        d = Fn.make_desc((8, 400), (120, 400), None, variant, True, True, 0.0, 0.1, L.MATH_AUTO)
        assert list(d.reserved) == [0, 0, 0, 0]
    d = Fn.make_desc((8, 400), (120, 400), None, L.VARIANT_BBB, True, True, 0.0, 0.1, L.MATH_AUTO, fold=(4, 3 << 40))
    assert d.reserved[1] == 4 and (d.reserved[2] & 0xFFFFFFFF) | ((d.reserved[3] & 0xFFFFFFFF) << 32) == 3 << 40
    assert not Fn.layer_fold_active()
    with Fn.layer_fold(256, STRIDE):
        assert Fn.layer_fold_active()
    assert not Fn.layer_fold_active()


def _check_groups(groups, n_local):
    assert groups[0][0] == 0
    ids = [s + k for s, n in groups for k in range(n)]
    assert ids == list(range(n_local))                       # every local id exactly once, in order
    sizes = [n for _, n in groups]
    assert max(sizes) - min(sizes) <= 1                      # as equal as possible


@pytest.mark.parametrize("world", [1, 8])
def test_group_size_of_c5_respects_budget_and_int32(built, world):
    """C5: BBB3Conv3FC-10, 1x32x32, B = 2048, 100 samples (13 local samples on rank 0 of 8)."""
    from pytorch_bayesiancnn_b200 import mc
    B = 2048
    n_local = len(mc.local_samples(100, world, 0))
    layers, pass_bytes, big = _layers("3conv3fc", "lrt", 1, B)
    assert big == B * 32 * 32 * 32                           # conv1's output
    assert pass_bytes == 4 * 2 * big                         # conv1's output in and out of the softplus
    for budget in (mc.LAYER_FOLD_BUDGET, 1 << 30, 4 << 30, 64 << 30):
        groups = mc.layer_fold_groups(n_local, pass_bytes, big, budget)
        assert groups is not None
        G = max(n for _, n in groups)
        assert G * pass_bytes <= budget or budget < 2 * pass_bytes
        assert G * big <= (1 << 31) - 1                      # every layer call's counts fit int32
        for m, xs in layers:
            assert G * math.prod(xs) <= (1 << 31) - 1
        _check_groups(groups, n_local)
        if budget == 64 << 30:
            cap = ((1 << 31) - 1) // big                     # the int32 limit binds: 31 samples of conv1's output
            assert cap == 31 and G <= cap and len(groups) == -(-n_local // cap)
    groups = mc.layer_fold_groups(n_local, pass_bytes, big, fold_group=5)
    assert max(n for _, n in groups) <= 5
    _check_groups(groups, n_local)
    assert mc.layer_fold_groups(n_local, pass_bytes, big, budget=pass_bytes) is None     # one sample per pass: no fold
    assert mc.layer_fold_groups(1, pass_bytes, big) is None


def test_groups_cover_every_local_id():
    from pytorch_bayesiancnn_b200 import mc
    for n_local in range(2, 40):
        for g in range(2, 12):
            groups = mc.layer_fold_groups(n_local, 1, 1, fold_group=g)
            _check_groups(groups, n_local)
            assert max(n for _, n in groups) <= g
            assert len(groups) == -(-n_local // g)


def test_refuses_children_that_mix_images():
    from torch import nn
    from pytorch_bayesiancnn_b200 import mc
    from pytorch_bayesiancnn_b200.modules import FlattenLayer
    assert mc._per_image_chain([nn.BatchNorm2d(3)], (4, 3, 8, 8)) is None
    assert mc._per_image_chain([FlattenLayer(96)], (4, 3, 8, 8)) is None      # view(-1, 96) would mix images
    assert mc._per_image_chain([nn.MaxPool2d(3, 2), FlattenLayer(27)], (4, 3, 8, 8)) is not None

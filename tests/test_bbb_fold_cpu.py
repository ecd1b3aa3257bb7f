"""Host-side answers for folding the Monte-Carlo samples of a BBB net into one pass of the fused chain: what
bbb_fused_supported accepts, how bbb_workspace_bytes grows, and what fused.plan returns.  No GPU needed."""
import ctypes as C

import pytest

from tests.util import CFG_PRIORS

S = 5
STRIDE = 1 << 40


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()


def _steps(variant, batch):
    from pytorch_bayesiancnn_b200 import fused
    from pytorch_bayesiancnn_b200.models import BBBAlexNet
    net = BBBAlexNet(10, 3, CFG_PRIORS, variant, "softplus")
    steps = fused.plan(list(net.children()), (batch, 3, 32, 32))
    assert steps is not None and len(steps) == 6
    return net, steps


def _supported(st, fold):
    from pytorch_bayesiancnn_b200 import fused, _lib as L
    d = fused._step_desc(st, 0, fold)
    return L.lib().bbb_fused_supported(C.byref(d), st.in_layout, fused._in_pitch(st), st.prev_hw, st.out_layout,
                                       fused._out_pitch(st))


def test_fused_supported_answers_for_a_bbb_fold(built):
    from pytorch_bayesiancnn_b200 import _lib as L
    for rows, bbb_rc in ((256, 0), (200, -2), (384, 0), (64, -2)):
        for variant, want in (("bbb", bbb_rc), ("lrt", 0)):                # LRT folds any rows, as before
            _, steps = _steps(variant, S * rows)
            for i, st in enumerate(steps):
                rc = _supported(st, (rows, STRIDE))
                assert rc == want, (variant, rows, i, rc, L.lib().bbb_last_error())
    # a batch that is not a whole number of samples is invalid for either variant
    for variant in ("bbb", "lrt"):
        _, steps = _steps(variant, 5 * 256 + 128)
        assert _supported(steps[0], (256, STRIDE)) == -1


def test_workspace_grows_by_the_sample_count_for_a_bbb_fold_only(built):
    from pytorch_bayesiancnn_b200 import fused, _lib as L
    lib = L.lib()
    fp32 = L.LayerDesc()
    fp32.math = L.MATH_FP32
    off = (int(lib.bbb_workspace_bytes(C.byref(fp32))) + 1023) // 1024 * 1024    # where the operand sets start
    for variant in ("bbb", "lrt"):
        _, steps = _steps(variant, S * 256)
        for st in steps:
            one = int(lib.bbb_workspace_bytes(C.byref(fused._step_desc(st, 0))))
            folded = int(lib.bbb_workspace_bytes(C.byref(fused._step_desc(st, 0, (256, STRIDE)))))
            if variant == "bbb":
                assert folded == off + S * ((one - off + 1023) // 1024 * 1024), (st.out_chw, one, folded)
            else:
                assert folded == one
            # the prep-only and GEMM-only halves of a call size the same workspace
            assert folded == int(lib.bbb_workspace_bytes(C.byref(fused._step_desc(st, L.FUSED_SKIP_PREP, (256, STRIDE)))))


def test_planner_folds_bbb_alexnet_only_for_whole_row_tiles(built):
    from pytorch_bayesiancnn_b200 import fused
    from pytorch_bayesiancnn_b200.models import BBBAlexNet
    net = BBBAlexNet(10, 3, CFG_PRIORS, "bbb", "softplus")
    kids = list(net.children())
    steps = fused.plan(kids, (S * 256, 3, 32, 32), fold=(256, STRIDE))
    assert steps is not None and len(steps) == 6 and all(st.batch == S * 256 for st in steps)
    assert fused.plan(kids, (S * 200, 3, 32, 32), fold=(200, STRIDE)) is None
    assert fused.plan(kids, (S * 200, 3, 32, 32)) is not None                # unfolded, the same net still fuses

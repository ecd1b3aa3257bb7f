"""Host-side checks of bf16 activations (act_dtype = BBB_DTYPE_BF16) on the per-layer forward (no GPU needed; the support
queries need the built library).

- bbb_forward_supported accepts the bf16 desc of every case of tests/forward_ref.CASES on bf16 and on auto wherever auto
  resolves to bf16 (folds and first image included), exactly where it accepts the fp32 desc; it refuses bf16 on fp32 and
  tf32 (and auto resolving to fp32) with BBB_E_UNSUPPORTED.
- functional.layer_io, the host logic of BayesLayerFn: which desc a call sends and which dtype y has, per math mode and
  input dtype."""
import ctypes as C

import pytest
import torch

from tests import forward_ref as R

E_UNSUPPORTED = -2


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()


def _desc(cs, variant, math, act_dtype, sample=True):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    fold = None if cs.fold is None else (cs.fold[0], R.FOLD_STRIDE)
    return Fn.make_desc(R.x_shape(cs), R.w_shape(cs), R.conv_of(cs), L.VARIANT_LRT if variant == "lrt" else L.VARIANT_BBB,
                        sample, cs.bias, 0.0, 0.1, L.MATH_BY_NAME[math], L.KL_BY_NAME[cs.kl], L.ACT_BY_NAME[cs.act],
                        act_dtype=act_dtype, fold=fold, first_image=0 if cs.fold is None else cs.fold[1])


def _rc(cs, variant, math, act_dtype, sample=True):
    from pytorch_bayesiancnn_b200 import _lib as L
    return int(L.lib().bbb_forward_supported(C.byref(_desc(cs, variant, math, act_dtype, sample))))


@pytest.mark.parametrize("cs", R.CASES, ids=[c.name for c in R.CASES])
def test_bf16_support_follows_the_fp32_desc_on_bf16_operands(built, cs):
    from pytorch_bayesiancnn_b200 import _lib as L
    bf16 = L.DTYPE_BF16
    for variant in cs.variants:
        samples = (True, False) if cs.fold is None else (True,)
        for sample in samples:
            for math in ("bf16", "auto"):
                want_ok = R.resolves(cs) == "bf16" if math == "auto" else "bf16" not in cs.refuse
                rc = _rc(cs, variant, math, bf16, sample)
                assert (rc == 0) == want_ok, (variant, math, sample, rc)
                if want_ok:
                    assert _rc(cs, variant, math, L.DTYPE_F32, sample) == 0
                else:
                    assert rc == E_UNSUPPORTED, (variant, math, sample, rc)
            for math in ("fp32", "tf32"):
                assert _rc(cs, variant, math, bf16, sample) == E_UNSUPPORTED, (variant, math, sample)


def test_unknown_act_dtype_is_refused(built):
    cs = next(c for c in R.CASES if c.name == "lenet_conv2_b256")
    for math in R.MATHS + ("auto",):
        assert _rc(cs, "lrt", math, 2) == E_UNSUPPORTED, math


@pytest.mark.parametrize("name", ["lenet_conv1_b256", "3conv3fc_fc2_b2048", "lenet_fc1_fold10x256",
                                  "lenet_conv2_fold3x128_first1000", "edge_lin_k16384", "edge_lin_k16385"])
def test_layer_io_chooses_the_path_and_output_dtype(built, name):
    """bf16 input on bf16 / auto: bf16 I/O where the engine takes the bf16 desc, else the fp32 call with y rounded to
    bf16 -- bf16 y either way.  fp32 / tf32, and every non-bf16 input: the fp32 desc and an fp32 y, as before."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    cs = next(c for c in R.CASES if c.name == name)
    for variant in cs.variants:
        for math in R.MATHS + ("auto",):
            accepted = R.resolves(cs) == "bf16" if math == "auto" else (math == "bf16" and "bf16" not in cs.refuse)
            d = _desc(cs, variant, math, L.DTYPE_F32)
            io, y_dtype = Fn.layer_io(d, torch.bfloat16)
            if math in ("bf16", "auto"):
                assert (io, y_dtype) == (accepted, torch.bfloat16), (variant, math)
                assert d.act_dtype == (L.DTYPE_BF16 if accepted else L.DTYPE_F32)
            else:
                assert (io, y_dtype, d.act_dtype) == (False, torch.float32, L.DTYPE_F32), (variant, math)
            for dt in (torch.float32, torch.float16, torch.float64):
                d = _desc(cs, variant, math, L.DTYPE_BF16)
                assert Fn.layer_io(d, dt) == (False, torch.float32) and d.act_dtype == L.DTYPE_F32, (variant, math, dt)

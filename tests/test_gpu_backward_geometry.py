"""The Bayesian layer backward at every geometry the three models train with, on all three math paths, against the
float64 reference of tests/backward_ref.py.

- The contraction kernel on its own: every distinct contraction functional._tc_wgrad / _tc_dgrad issue for a case of
  backward_ref.CASES (each ragged last wgrad chunk included) runs through functional._tc_contract in bf16 and in tf32 and
  is compared with float64 on the operands rounded as the kernel rounds them: |got - ref| <= 1e-4 M, M the contraction
  of the absolute values.  What remains is fp32 accumulation only, so a dropped or doubled 64-wide K block (about
  1e-3 M at K = 8192) fails.
- The layer backward end to end, both variants, with and without a bias, math fp32 / tf32 / bf16: every gradient
  within C M of the float64 gradient (M: backward_ref.bounds), exactly 0 where M is 0, and the tensor-core backward
  pinned -- it must run in tf32 and bf16 unless the case is marked as falling back, and must not be called in fp32.
  C comes from the operand unit roundoff u (bf16 2^-8, tf32 2^-11): a product of two rounded operands is off by 2u,
  and the LRT variance path adds the error of act_std.  C_FP32 allows for fp32 summation over the reduction.
  Measured on an H100 80GB HBM3, worst |got - ref| / M over all cases, variants and gradients: fp32 5.2e-7,
  tf32 9.0e-4 (2u = 9.8e-4), bf16 7.4e-3 (2u = 7.8e-3); the contraction on its own 1.1e-6 (bf16) and 2.4e-6 (tf32);
  the KL backward 7.4e-7.
- The branches of the backward on a few cases: Philox noise, a first image, sample=False, no input gradient, an LRT
  layer fed zero receptive fields (act_std = 1e-8), a bf16 forward with the CUDA-core backward; two runs of the
  tensor-core backward are bit-identical; bbb_kl_backward in both KL conventions against its closed form.
- The benchmark's training step (mc.MCTrainStep, BBBAlexNet, B = 512) against float64 oracle autograd.
Run with -s to see the worst normalised error per family."""
import collections
import ctypes as C
import sys

import numpy as np
import pytest
import torch

from tests import backward_ref as R
from tests.util import scale_err

pytestmark = pytest.mark.gpu
C_BAR = {"fp32": 1e-5, "tf32": 2.5e-3, "bf16": 1e-2}
CONTRACT_BAR = 1e-4
NAMES = ("x", "W_mu", "W_rho", "bias_mu", "bias_rho")
_worst = collections.defaultdict(float)


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    yield torch.device("cuda:0")
    if _worst:
        lines = [f"  {fam:28s} worst |got - ref| / M = {v:.3e}" for fam, v in sorted(_worst.items())]
        sys.__stdout__.write("\n[backward geometry]\n" + "\n".join(lines) + "\n")


def _normalised(got, ref, mag):
    """max |got - ref| / mag over the elements with mag > 0 (a NaN counts as inf); got must be exactly 0 where mag is 0."""
    got, ref, mag = got.double(), ref.double(), mag.double()
    zero = mag == 0
    assert bool((got[zero] == 0).all()), "a nonzero value where every term is zero (an unwritten or stray output)"
    e = (got - ref).abs() / torch.where(zero, torch.ones_like(mag), mag)
    e = torch.where(zero, torch.zeros_like(e), torch.nan_to_num(e, nan=float("inf")))
    return float(e.max()) if e.numel() else 0.0


# --------------------------------------------------------------------------------------------- the contraction kernel
@pytest.mark.parametrize("cs", R.CASES, ids=[c.name for c in R.CASES])
def test_contraction_matches_float64_on_rounded_operands(dev, cs):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    calls, _ = R.contractions(cs)
    # distinct shapes, in order; a refused wgrad (the case falls back) is not run
    shapes = list(dict.fromkeys((x, w, conv) for role, x, w, conv in calls
                                if not (role == "wgrad" and cs.fallback == "wgrad")))
    g = torch.Generator(device=dev).manual_seed(R.CASES.index(cs))
    prev = Fn._tc_math
    try:
        for (xs, ws, conv) in shapes:
            x = torch.randn(xs, generator=g, device=dev)
            w = torch.randn(ws, generator=g, device=dev)
            for math, code in (("bf16", L.MATH_BF16_TC), ("tf32", L.MATH_TF32_TC)):
                Fn._tc_math = code
                got = Fn._tc_contract(x, w, conv)
                xr, wr = R.ROUND[math](x), R.ROUND[math](w)
                ref = R.contract(xr, wr, conv)
                mag = R.contract(xr.abs(), wr.abs(), conv)
                assert got.shape == ref.shape
                e = _normalised(got, ref, mag)
                _worst["contract " + math] = max(_worst["contract " + math], e)
                assert e <= CONTRACT_BAR, (math, xs, ws, conv, e)
    finally:
        Fn._tc_math = prev


# --------------------------------------------------------------------------------------------- the layer end to end
MATHS = ("fp32", "tf32", "bf16")


def _inputs(cs, variant, bias, dev, seed, sparse=False):
    """fp32 layer inputs on the device: x, W_mu, W_rho, bias_mu, bias_rho, (external) eps, gout.  ``sparse``: x >= 0
    with whole images and the top half of every map zero, so that whole receptive fields are zero."""
    g = torch.Generator(device=dev).manual_seed(seed)
    rn = lambda shape: torch.randn(shape, generator=g, device=dev)
    ws = R.w_shape(cs)
    fan_in = int(np.prod(ws[1:]))
    x = rn(R.x_shape(cs))
    if sparse:
        x = x.clamp_min(0.0)
        x[: cs.B // 2] = 0.0
        if x.dim() == 4:
            x[:, :, : cs.hw[0] // 2] = 0.0
    W_mu = rn(ws) * fan_in ** -0.5
    W_rho = rn(ws) * 0.5 - 3.0
    b_mu = rn(ws[0]) * 0.5 if bias else None
    b_rho = rn(ws[0]) * 0.5 - 3.0 if bias else None
    eps = (rn(ws), rn(ws[0]) if bias else None) if variant == "bbb" else rn(R.y_shape(cs))
    gout = rn(R.y_shape(cs))
    return x, W_mu, W_rho, b_mu, b_rho, eps, gout


def _cfg(cs, variant, math, sample=True):
    from pytorch_bayesiancnn_b200 import _lib as L
    return {"conv": R.conv_of(cs), "variant": L.VARIANT_LRT if variant == "lrt" else L.VARIANT_BBB,
            "sample": bool(sample), "prior_mu": 0.0, "prior_sigma": 0.1, "math": L.MATH_BY_NAME[math],
            "kl_convention": L.KL_REFERENCE, "act": L.ACT_NONE, "owner": None}


class _PathRecorder:
    """Wraps BayesLayerFn._backward_tc: records None (gave up), "refused" (a contraction the kernel does not take) or
    "ran" for each call."""

    def __init__(self, monkeypatch):
        from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
        self.calls = []
        orig = Fn.BayesLayerFn._backward_tc

        def rec(ctx, gy):
            try:
                out = orig(ctx, gy)
            except L.EngineError:
                self.calls.append("refused")
                raise
            self.calls.append("ran" if out is not None else None)
            return out

        monkeypatch.setattr(Fn.BayesLayerFn, "_backward_tc", staticmethod(rec))


def _engine_grads(cs, variant, math, inp, x_grad=True, sample=True, eps_mode="external", seed=0, stream=0,
                  first_image=0):
    """Forward + backward of one layer call on the engine; returns ([gx, gW_mu, gW_rho, gb_mu, gb_rho], the eps the
    forward used, for the reference)."""
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import functional as Fn
    x, W_mu, W_rho, b_mu, b_rho, eps, gout = inp
    leaves = [x.clone().requires_grad_(x_grad)] + [None if t is None else t.clone().requires_grad_(True)
                                                    for t in (W_mu, W_rho, b_mu, b_rho)]
    cfg = _cfg(cs, variant, math, sample)
    with Fn.first_image(first_image):
        if eps_mode == "external" and sample:
            ext = [eps[0]] + ([eps[1]] if eps[1] is not None else []) if variant == "bbb" else [eps]
            with bbb.external_eps(ext):
                y, _ = Fn.BayesLayerFn.apply(*leaves, cfg)
        else:
            bbb.manual_seed(seed, stream)
            y, _ = Fn.BayesLayerFn.apply(*leaves, cfg)
    torch.autograd.backward([y], [gout])
    if eps_mode == "philox" and sample:        # the noise the kernels drew, regenerated on the host side
        if variant == "bbb":
            nw = W_mu.numel()
            eps = (bbb.philox_normal(nw, seed, stream, 0, device=x.device).view_as(W_mu),
                   bbb.philox_normal(b_mu.numel(), seed, stream, nw, device=x.device) if b_mu is not None else None)
        else:
            shp = R.y_shape(cs)
            per = int(np.prod(shp[1:]))
            z = bbb.philox_normal(int(np.prod(shp)), seed, stream, first_image * per, device=x.device)
            eps = z.view(shp) if len(shp) == 2 else z.view(shp[0], shp[2], shp[3], shp[1]).permute(0, 3, 1, 2)
    return [t.grad if t is not None and t.requires_grad else None for t in leaves], eps


def _compare(got, inp, eps, cs, variant, C_, fam, sample=True, x_grad=True):
    x, W_mu, W_rho, b_mu, b_rho, _, gout = inp
    args = (variant, x, W_mu, W_rho, b_mu, b_rho, eps, gout, R.conv_of(cs), sample)
    ref, mag = R.grads(*args), R.bounds(*args)
    for name, a, r, m in zip(NAMES, got, ref, mag):
        if name == "x" and not x_grad:
            assert a is None
            continue
        if r is None:
            assert a is None, name
            continue
        assert a is not None and a.shape == r.shape, name
        e = _normalised(a, r, m)
        _worst[f"{fam} {name}"] = max(_worst[f"{fam} {name}"], e)
        assert e <= C_, (cs.name, fam, name, e)


def _expect_path(rec, cs, math, x_grad=True):
    if math == "fp32":
        assert rec.calls == [], "the tensor-core backward ran on the fp32 path"
        return
    want = "ran"
    if cs.fallback == "wgrad":
        want = "refused"
    elif cs.fallback == "dgrad" and x_grad:
        want = None
    assert rec.calls == [want], (cs.name, math, rec.calls)


@pytest.mark.parametrize("variant", ["bbb", "lrt"])
@pytest.mark.parametrize("cs", R.CASES, ids=[c.name for c in R.CASES])
def test_layer_backward_matches_float64(dev, monkeypatch, cs, variant):
    for bias in (True, False):
        inp = _inputs(cs, variant, bias, dev, seed=10 * R.CASES.index(cs) + 2 * (variant == "lrt") + bias)
        for math in MATHS:
            rec = _PathRecorder(monkeypatch)
            got, eps = _engine_grads(cs, variant, math, inp)
            _expect_path(rec, cs, math)
            _compare(got, inp, eps, cs, variant, C_BAR[math], f"{math} {variant}")
            monkeypatch.undo()


BRANCH_CASES = ["lenet_conv1_b256", "edge_k2s3", "edge_lin_k100_n70", "edge_1x1_p1", "alexnet_conv2_b1000"]
BRANCHES = ["philox", "first_image", "no_sample", "no_x_grad", "sparse_lrt", "simt_after_bf16"]


@pytest.mark.parametrize("branch", BRANCHES)
@pytest.mark.parametrize("name", BRANCH_CASES)
def test_backward_branches(dev, monkeypatch, name, branch):
    cs = next(c for c in R.CASES if c.name == name)
    idx = R.CASES.index(cs)
    variants = ("lrt",) if branch in ("first_image", "sparse_lrt") else ("bbb", "lrt")
    maths = ("bf16",) if branch == "simt_after_bf16" else MATHS
    for variant in variants:
        bias = branch != "sparse_lrt"
        inp = _inputs(cs, variant, bias, dev, seed=1000 + 10 * idx + BRANCHES.index(branch),
                      sparse=branch == "sparse_lrt")
        for math in maths:
            if branch == "simt_after_bf16":
                monkeypatch.setenv("BBB_B200_BWD", "simt")
            rec = _PathRecorder(monkeypatch)
            kw = dict(x_grad=branch != "no_x_grad", sample=branch != "no_sample")
            mode = "philox" if branch in ("philox", "first_image", "sparse_lrt") else "external"
            got, eps = _engine_grads(cs, variant, math, inp, eps_mode=mode, seed=77 + idx, stream=3 + idx,
                                     first_image=1000 if branch == "first_image" else 0, **kw)
            if branch == "simt_after_bf16":
                assert rec.calls == []
            else:
                _expect_path(rec, cs, math, kw["x_grad"])
            # the CUDA-core backward after a bf16 forward reads the bf16 forward's act_std: the bf16 bar
            C_ = C_BAR["bf16"] if branch == "simt_after_bf16" else C_BAR[math]
            _compare(got, inp, eps, cs, variant, C_, f"{math} {variant}", **kw)
            monkeypatch.undo()


@pytest.mark.parametrize("math", ["bf16", "tf32"])
@pytest.mark.parametrize("name", ["alexnet_conv1_b512", "3conv3fc_conv1_b300", "3conv3fc_fc2_b300"])
def test_tensor_core_backward_is_deterministic(dev, monkeypatch, name, math):
    """No atomics in the tensor-core backward: two runs on the same inputs give the same bits."""
    cs = next(c for c in R.CASES if c.name == name)
    for variant in ("bbb", "lrt"):
        inp = _inputs(cs, variant, True, dev, seed=5)
        rec = _PathRecorder(monkeypatch)
        a, _ = _engine_grads(cs, variant, math, inp, eps_mode="philox", seed=9, stream=1)
        b, _ = _engine_grads(cs, variant, math, inp, eps_mode="philox", seed=9, stream=1)
        assert rec.calls == ["ran", "ran"]
        for name_, u, v in zip(NAMES, a, b):
            assert torch.equal(u, v), (variant, name_)
        monkeypatch.undo()


# --------------------------------------------------------------------------------------------- KL backward
@pytest.mark.parametrize("convention", ["reference", "textbook"])
@pytest.mark.parametrize("n", [884736, 1000003])
def test_kl_backward_matches_closed_form(dev, convention, n):
    """bbb_kl_backward against the float64 closed form (oracle.kl_loss / kl_textbook differentiated by hand), element by
    element within 1e-5 of the sum of the absolute values of its terms; n = 1000003 leaves a grid-stride tail.  The
    kernel adds into g_mu / g_rho: a second call doubles them exactly."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    g = torch.Generator(device=dev).manual_seed(n)
    mu = torch.randn(n, generator=g, device=dev) * 0.2
    rho = torch.linspace(-10.0, 5.0, n, device=dev)[torch.randperm(n, generator=g, device=dev)]
    pm, ps, go = (float(np.float32(v)) for v in (0.05, 0.1, 0.37))      # the fp32 values the kernel receives
    gkl = torch.tensor(go, device=dev)
    g_mu, g_rho = torch.zeros_like(mu), torch.zeros_like(mu)
    conv = L.KL_BY_NAME[convention]
    call = lambda: L.check(L.lib().bbb_kl_backward(Fn._ptr(mu), Fn._ptr(rho), C.c_uint64(n), C.c_float(pm), C.c_float(ps),
                                                   C.c_int32(conv), Fn._ptr(gkl), Fn._ptr(g_mu), Fn._ptr(g_rho),
                                                   Fn._stream(dev)), "bbb_kl_backward")
    call()
    torch.cuda.synchronize()
    m, r = mu.double(), rho.double()
    s = torch.log1p(torch.exp(r))
    sg = torch.sigmoid(r)
    d, ad = m - pm, m.abs() + abs(pm)      # mu - prior_mu is itself a sum of two terms
    if convention == "reference":         # KL(prior || posterior), metrics.py:27-29 with the call-site binding
        dm, mag_m = d / s ** 2, ad / s ** 2
        ds = 1 / s - ps ** 2 / s ** 3 - d ** 2 / s ** 3
        mag_s = 1 / s + ps ** 2 / s ** 3 + ad ** 2 / s ** 3
    else:                                 # KL(posterior || prior)
        dm, mag_m = d / ps ** 2, ad / ps ** 2
        ds, mag_s = -1 / s + s / ps ** 2, 1 / s + s / ps ** 2
    e_mu = _normalised(g_mu, go * dm, go * mag_m)
    e_rho = _normalised(g_rho, go * ds * sg, go * mag_s * sg)
    _worst[f"kl {convention} mu"] = max(_worst[f"kl {convention} mu"], e_mu)
    _worst[f"kl {convention} rho"] = max(_worst[f"kl {convention} rho"], e_rho)
    assert e_mu <= 1e-5 and e_rho <= 1e-5, (e_mu, e_rho)
    first = (g_mu.clone(), g_rho.clone())
    call()
    torch.cuda.synchronize()
    assert torch.equal(g_mu, 2 * first[0]) and torch.equal(g_rho, 2 * first[1])


# --------------------------------------------------------------------------------------------- the training step
# (relative error of the loss, scale-relative error of every parameter gradient): about 3x the worst measured on an
# H100 80GB HBM3 over both variants -- auto (bf16) 3.2e-4 and 1.7e-2, tf32 7.4e-6 and 9.1e-3
TRAIN_BAR = {"auto": (9e-4, 5e-2), "tf32": (2e-5, 2.5e-2)}


@pytest.mark.parametrize("math", ["auto", "tf32"])
@pytest.mark.parametrize("variant", ["lrt", "bbb"])
def test_alexnet_b512_training_step_matches_float64_oracle(dev, variant, math):
    """The benchmark's training step: mc.MCTrainStep on BBBAlexNet at B = 512 with 2 MC samples, against float64
    oracle autograd (main_bayesian.py:46-58) on the same Philox noise: the loss and every parameter gradient.  With
    these parameters the label's log-probability is far below -100, where softmax and p_bar both underflow fp32: the
    gradient of the loss must still be finite (it was NaN when MCTrainStep formed their ratio from the two)."""
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import mc
    from tests.test_gpu_mc import MC_NS, _engine_eps, _net, _oracle_train_grads
    B, S = 512, 2
    net, params = _net("alexnet", 10, 3, variant, dev, math)
    x = torch.rand(B, 3, 32, 32, generator=torch.Generator().manual_seed(4))
    labels = torch.randint(0, 10, (B,), generator=torch.Generator().manual_seed(5))
    step = mc.MCTrainStep(net, x.to(dev), S, train_size=50000.0, seed=21)
    out = step(x.to(dev), labels.to(dev), beta=0.1)
    torch.cuda.synchronize()
    eps = [[e.to(dev) for e in _engine_eps(bbb, "alexnet", 10, 3, variant, B, 21, MC_NS | (j << 40), dev)]
           for j in range(S)]
    P = [{k: v.to(dev) for k, v in p.items()} for p in params]
    ref_loss, ref_grads = _oracle_train_grads("alexnet", P, x.to(dev), labels.to(dev), eps, variant, 10, 50000.0, 0.1,
                                              dtype=torch.float64)
    e_loss = abs(float(out["head"][0]) - float(ref_loss)) / abs(float(ref_loss))
    got = [g for m in net.children() if hasattr(m, "W_mu") for g in (m.W_mu.grad, m.W_rho.grad, m.bias_mu.grad, m.bias_rho.grad)]
    assert len(got) == len(ref_grads)
    errs = [scale_err(a, b) for a, b in zip(got, ref_grads)]
    fam = f"train {math} {variant}"
    _worst[fam + " loss"] = max(_worst[fam + " loss"], e_loss)
    for i, e in enumerate(errs):
        key = f"{fam} {('W_mu', 'W_rho', 'bias_mu', 'bias_rho')[i % 4]}"
        _worst[key] = max(_worst[key], e)
    print(fam, "loss", e_loss, "grads", ["%.2e" % e for e in errs])
    assert all(bool(torch.isfinite(a).all()) for a in got), "non-finite parameter gradients"
    assert e_loss <= TRAIN_BAR[math][0], e_loss
    assert max(errs) <= TRAIN_BAR[math][1], errs

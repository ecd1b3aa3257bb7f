"""bf16 activations (act_dtype = BBB_DTYPE_BF16) on the GPU: the tensor-core layer kernel reading bf16 x and writing
bf16 y, autograd through it, the nets and the Monte-Carlo steps.

- Forward, at every tensor-core case of tests/forward_ref.CASES, both variants, folded and unfolded: on bf16 inputs the
  operands are those of the fp32-I/O call, so y must be that call's y rounded to bf16 (RNE) bit for bit, and act_std
  and the KL bitwise equal -- a mismatch means the tile schedule or the accumulation order moved.  The bf16 y is within
  the loose bf16 tier of the float64 reference (forward_ref.loose_err).
- Backward, at every layer geometry the three models train with (tests/backward_ref.py), both variants, unfolded and
  under layer_fold(grad=True): the gradients of a bf16-I/O layer equal those of the fp32-I/O layer fed the upcast x and
  gy, bit for bit (gx after rounding to bf16).
- BBBLeNet, BBB3Conv3FC and BBBAlexNet (fused chain) return bf16 logits within the bf16 bar of the oracle; MCForward
  (uncertainty and information outputs; eager, captured and overlapped) and MCTrainStep(fold=True) with bf16 inputs
  likewise.
Run with -s to see the errors."""
import ctypes as C

import pytest
import torch

from oracle import bbb_oracle as O
from tests import backward_ref as BR
from tests import forward_ref as R
from tests.util import CFG_PRIORS, scale_err

pytestmark = pytest.mark.gpu
BF16_TOL = 1e-2                 # the scale-relative bar of a bf16 net against the oracle (tests/test_gpu_parity.py)
MC_NS = 1 << 63
SEED = 41


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _call(cs, variant, math, x, W, sample, bf16, seed=0, stream=0, want_std=False, fold=None, first_image=0):
    """One layer call through the C ABI with fp32 (bf16=False) or bf16 activations: (y, act_std, kl)."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    dev = x.device
    W_mu, W_rho, b_mu, b_rho = W
    conv = R.conv_of(cs)
    d = Fn.make_desc(tuple(x.shape), tuple(W_mu.shape), conv, L.VARIANT_LRT if variant == "lrt" else L.VARIANT_BBB,
                     sample, b_mu is not None, 0.0, 0.1, L.MATH_BY_NAME[math], L.KL_BY_NAME[cs.kl],
                     L.ACT_BY_NAME[cs.act], act_dtype=L.DTYPE_BF16 if bf16 else L.DTYPE_F32,
                     fold=None if fold is None else (fold, R.FOLD_STRIDE), first_image=first_image)
    yshape = R.y_shape(cs, x.shape[0])
    y = torch.full(yshape, float("nan"), dtype=torch.bfloat16 if bf16 else torch.float32, device=dev)
    std = torch.full(yshape, float("nan"), dtype=torch.float32, device=dev) if want_std else None
    kl = torch.full((), float("nan"), dtype=torch.float32, device=dev)
    ws = Fn.workspace(dev, d)
    fn = L.lib().bbb_linear_forward if conv is None else L.lib().bbb_conv2d_forward
    L.check(fn(C.byref(d), Fn._ptr(x), Fn._ptr(W_mu), Fn._ptr(W_rho), Fn._ptr(b_mu), Fn._ptr(b_rho), Fn._ptr(y),
               Fn._ptr(kl), Fn._ptr(std), None, None, C.c_uint64(seed), C.c_uint64(stream), None, Fn._ptr(ws),
               C.c_size_t(ws.numel()), Fn._stream(dev)), f"{cs.name} {variant} {math} bf16={bf16}")
    torch.cuda.synchronize()
    return y, std, kl


TC_PARAMS = [(cs, v) for cs in R.CASES if "bf16" not in cs.refuse for v in cs.variants]


@pytest.mark.parametrize("cs,variant", TC_PARAMS, ids=[f"{cs.name}-{v}" for cs, v in TC_PARAMS])
def test_bf16_io_forward_is_the_rounded_fp32_io_forward(dev, cs, variant):
    from tests.test_gpu_layer_forward_geometry import _philox_eps
    idx = R.CASES.index(cs)
    g = torch.Generator(device=dev).manual_seed(2000 + 2 * idx + (variant == "lrt"))
    x, W_mu, W_rho, b_mu, b_rho, _ = R.make_inputs(cs, variant, g, dev)
    xh = x.bfloat16()
    xf = xh.float()                                      # bf16-representable: the fp32-I/O call sees the same operands
    del x
    W = (W_mu, W_rho, b_mu, b_rho)
    lrt = variant == "lrt"
    fold = cs.fold[0] if cs.fold else None
    first = cs.fold[1] if cs.fold else 0
    seed, stream = 23 + idx, 9 + 5 * idx
    for sample in ((False, True) if fold is None else (True,)):
        for want_std in ((True, False) if lrt and sample else (False,)):
            kw = dict(seed=seed, stream=stream, want_std=want_std, fold=fold, first_image=first)
            yf, sf, klf = _call(cs, variant, "bf16", xf, W, sample, False, **kw)
            yh, sh, klh = _call(cs, variant, "bf16", xh, W, sample, True, **kw)
            assert yh.dtype == torch.bfloat16 and bool(torch.isfinite(yh).all()), (sample, want_std)
            assert torch.equal(yh, yf.bfloat16()), (sample, want_std, "y is not the rounded fp32-I/O y")
            assert torch.equal(klh, klf), (sample, want_std, "kl")
            if want_std:
                assert torch.equal(sh, sf), (sample, "act_std")
            del yf, sf
            ya, _, _ = _call(cs, variant, "auto", xh, W, sample, True, **kw)
            assert torch.equal(ya, yh), "auto did not run the bf16 path"
            del ya
            if sample and (want_std or not lrt):
                imgs = R.check_images(cs, idx)
                rows = cs.B if fold is None else fold
                for j in range(cs.B // rows):
                    sub = [i - j * rows for i in imgs if j * rows <= i < (j + 1) * rows]
                    if not sub:
                        continue
                    blk = slice(j * rows, (j + 1) * rows)
                    eps = _philox_eps(cs, variant, seed, stream + j * R.FOLD_STRIDE, rows, first, cs.bias, dev)
                    ref, M, _ = R.layer_ref(variant, xf[blk][sub], W_mu, W_rho, b_mu, b_rho,
                                            eps if variant == "bbb" else eps[sub], R.conv_of(cs), True, cs.act)
                    e = R.loose_err(yh[blk][sub], ref, M, "bf16")
                    assert e <= 1, (cs.name, variant, j, e)
                    del eps, ref, M
            del yh, sh
            torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------------- backward
TRAIN_CASES = [cs for cs in BR.CASES if cs.name.split("_")[0] in ("alexnet", "lenet", "3conv3fc")]


def _layer(cs, variant, dev):
    from pytorch_bayesiancnn_b200 import modules as M
    lrt = variant == "lrt"
    torch.manual_seed(BR.CASES.index(cs))
    if cs.k is None:
        layer = (M.BBBLRTLinear if lrt else M.BBBLinear)(cs.cin, cs.cout, priors=CFG_PRIORS)
    else:
        layer = (M.BBBLRTConv2d if lrt else M.BBBConv2d)(cs.cin, cs.cout, cs.k, stride=cs.s, padding=cs.p,
                                                          dilation=cs.d, priors=CFG_PRIORS)
    layer = layer.to(dev).train()
    layer.set_flag("math", "bf16")
    return layer


def _grads(layer, x, gy, fold=None):
    """(y, gx, parameter gradients) of one sampled layer call on sample 3 of seed SEED."""
    from pytorch_bayesiancnn_b200 import functional as Fn
    params = [layer.W_mu, layer.W_rho, layer.bias_mu, layer.bias_rho]
    for p in params:
        p.grad = None
    x = x.clone().requires_grad_(True)
    with Fn.mc_sample(3, SEED):
        if fold is None:
            y = layer(x)
        else:
            with Fn.layer_fold(fold, 1 << 40, grad=True):
                y = layer(x)
    y.backward(gy)
    torch.cuda.synchronize()
    return y.detach(), x.grad, [p.grad.clone() for p in params]


@pytest.mark.parametrize("variant", ["lrt", "bbb"])
@pytest.mark.parametrize("cs", TRAIN_CASES, ids=[c.name for c in TRAIN_CASES])
def test_bf16_io_backward_equals_fp32_io_backward(dev, cs, variant):
    layer = _layer(cs, variant, dev)
    g = torch.Generator(device=dev).manual_seed(5)
    runs = [(BR.x_shape(cs), BR.y_shape(cs), None)]
    if variant == "lrt":                                 # folded: 3 samples of 8 images
        runs.append(((24,) + BR.x_shape(cs)[1:], (24,) + BR.y_shape(cs)[1:], 8))
    for xs, ys, fold in runs:
        x = torch.randn(xs, device=dev, generator=g).bfloat16()
        gy = torch.randn(ys, device=dev, generator=g).bfloat16()
        yh, gxh, gph = _grads(layer, x, gy, fold)
        yf, gxf, gpf = _grads(layer, x.float(), gy.float(), fold)
        assert yh.dtype == torch.bfloat16 and gxh.dtype == torch.bfloat16 and yf.dtype == torch.float32
        assert torch.equal(yh, yf.bfloat16()), (fold, "y")
        assert torch.equal(gxh, gxf.bfloat16()), (fold, "gx")
        for name, a, b in zip(("W_mu", "W_rho", "bias_mu", "bias_rho"), gph, gpf):
            assert a.dtype == torch.float32 and torch.equal(a, b), (fold, name)


# -------------------------------------------------------------------------------------------------------------- nets
NETS = (("lenet", 3), ("3conv3fc", 1), ("alexnet", 3))


@pytest.mark.parametrize("variant", ["lrt", "bbb"])
@pytest.mark.parametrize("key,inputs", NETS)
def test_nets_return_bf16_logits_within_the_bf16_bar(dev, key, inputs, variant):
    import pytorch_bayesiancnn_b200 as bbb
    from tests.test_gpu_mc import _net
    B = 130
    net, params = _net(key, 10, inputs, variant, dev, "auto")
    xh = torch.rand(B, inputs, 32, 32, generator=torch.Generator().manual_seed(6)).bfloat16()
    eps = O.draw_eps_like_reference(O.eps_shapes(key, 10, inputs, variant, B), seed=8)
    ref, refkl = O.net_forward(key, params, xh.float(), eps, variant, "softplus", 0.0, 0.1, 10)
    with torch.no_grad(), bbb.external_eps(eps):
        logits, kl = net(xh.to(dev))
    torch.cuda.synchronize()
    assert logits.dtype == torch.bfloat16 and tuple(logits.shape) == (B, 10)
    if key == "alexnet":
        assert net._fused_plans[(B, 3, 32, 32)] is not None        # the fused chain ran
    e = scale_err(logits.float(), ref)
    print(key, variant, "bf16 activations: logits scale err", e)
    assert e < BF16_TOL, (key, variant, e)
    assert abs(float(kl) - float(refkl)) <= 1e-5 * abs(float(refkl))


# ------------------------------------------------------------------------------------------------------- MC steps
def _mc_oracle_logits(key, params, xh, inputs, variant, S, dev):
    import pytorch_bayesiancnn_b200 as bbb
    from tests.test_gpu_mc import _engine_eps
    out = []
    for j in range(S):
        eps = _engine_eps(bbb, key, 10, inputs, variant, xh.shape[0], SEED, MC_NS | (j << 40), dev)
        out.append(O.net_forward(key, params, xh.float().cpu(), eps, variant, "softplus", 0.0, 0.1, 10)[0])
    return out


@pytest.mark.parametrize("variant", ["lrt", "bbb"])
@pytest.mark.parametrize("key,inputs", NETS)
def test_mc_forward_with_bf16_inputs(dev, key, inputs, variant):
    """Per-sample logits within the bf16 bar of the oracle on the same noise; log_outputs, the uncertainty and the
    information outputs equal their float64 restatements on those logits; the captured step (serial, and overlapped
    with two steps in flight) replays the eager step bit for bit."""
    from pytorch_bayesiancnn_b200 import mc
    from tests.info_ref import information
    from tests.test_gpu_mc import _net
    B, S = 128, 4
    net, params = _net(key, 10, inputs, variant, dev, "auto")
    xh = torch.rand(B, inputs, 32, 32, generator=torch.Generator().manual_seed(7)).bfloat16().to(dev)
    kw = dict(want_uncertainty=True, want_information=True, seed=SEED)
    eng = mc.MCForward(net, xh, S, graph=False, **kw)
    if key == "alexnet":
        assert eng.fold_steps is not None
    elif variant == "lrt" or key == "lenet":
        assert eng.layer_fold is not None
    out = {k: v.clone() for k, v in eng(xh).items()}
    torch.cuda.synchronize()
    refs = _mc_oracle_logits(key, params, xh, inputs, variant, S, dev)
    errs = [scale_err(eng.logits[j], refs[j]) for j in range(S)]
    print(key, variant, "MCForward bf16 inputs: per-sample logits scale err", max(errs))
    assert max(errs) < BF16_TOL, errs
    L_ = [t.double().cpu() for t in eng.logits]
    lo = O.mc_combine(L_)
    assert float((out["log_outputs"].double().cpu() - lo).abs().max()) <= 1e-4 * max(1.0, float(lo.abs().max()))
    pred, epi, ale, ent = O.uncertainty(L_)
    assert scale_err(out["pred"], pred) < 1e-6
    for k, r in (("epistemic", epi), ("aleatoric", ale), ("entropy", ent)):
        assert float((out[k].double().cpu() - r).abs().max()) < 5e-5, k
    ree, rmi = information(L_)
    assert float((out["expected_entropy"].double().cpu() - ree).abs().max()) < 5e-5
    assert float((out["mutual_info"].double().cpu() - rmi).abs().max()) < 5e-5
    for extra in ({}, {"overlap": True, "inflight": 2}):
        cap = mc.MCForward(net, xh, S, **extra, **kw)
        res = cap(xh)
        cap.wait()
        torch.cuda.synchronize()
        assert torch.equal(cap.logits_all[0], eng.logits), extra
        for k in out:
            assert torch.equal(res[k], out[k]), (extra, k)
        assert cap.timeouts() == 0


TRAIN_BAR = (5e-3, 5e-2)        # loss relative error, parameter-gradient scale error against float64 oracle autograd


@pytest.mark.parametrize("key,inputs", [("lenet", 3), ("3conv3fc", 1)])
def test_folded_training_step_with_bf16_inputs(dev, key, inputs):
    from pytorch_bayesiancnn_b200 import mc
    from tests.test_gpu_mc import _engine_eps, _net, _oracle_train_grads
    import pytorch_bayesiancnn_b200 as bbb
    B, S, beta, train_size = 96, 4, 0.1, 5000.0
    net, params = _net(key, 10, inputs, "lrt", dev, "auto")
    xh = torch.rand(B, inputs, 32, 32, generator=torch.Generator().manual_seed(4)).bfloat16().to(dev)
    labels = torch.randint(0, 10, (B,), generator=torch.Generator().manual_seed(5)).to(dev)
    step = mc.MCTrainStep(net, xh, S, train_size=train_size, seed=SEED, fold=True)
    assert step.layer_fold == (S, 1)
    out = step(xh, labels, beta=beta)
    torch.cuda.synchronize()
    grads = [p.grad.clone() for p in step.params]
    assert all(g_.dtype == torch.float32 and bool(torch.isfinite(g_).all()) for g_ in grads)
    eps = [[e.to(dev) for e in _engine_eps(bbb, key, 10, inputs, "lrt", B, SEED, MC_NS | (j << 40), dev)]
           for j in range(S)]
    P = [{k: v.to(dev) for k, v in p.items()} for p in params]
    ref_loss, ref_grads = _oracle_train_grads(key, P, xh.float(), labels, eps, "lrt", 10, train_size, beta,
                                              dtype=torch.float64)
    e_loss = abs(float(out["head"][0]) - float(ref_loss)) / abs(float(ref_loss))
    errs = [scale_err(a, b) for a, b in zip(grads, ref_grads)]
    print(key, "MCTrainStep(fold=True) bf16 inputs: loss rel err", e_loss, "worst grad scale err", max(errs))
    assert e_loss <= TRAIN_BAR[0], e_loss
    assert max(errs) <= TRAIN_BAR[1], errs

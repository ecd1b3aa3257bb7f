"""Pruning masks on the GPU: every path of the engine honours a layer's W_mask / bias_mask (set_weight_mask).

1. All-ones masks, bitwise: y, act_std and KL of every per-layer case (tests/forward_ref.CASES; fp32, tf32, bf16 and bf16
   activations; BBB and LRT; folded), and the gradients of the layer autograd on every math mode (tensor-core and
   CUDA-core backward), the fused BBBAlexNet chain, MCForward (captured, cached preps, steps in flight) and a folded
   MCTrainStep, all equal the unmasked calls.
2. Random masks at 50 % and 95 %: every per-layer case against the float64 restatement (tests/mask_ref.py) on the same
   external eps at the loose bar of tests/forward_ref.py, and its KL within 1e-5 relative; the masked call equals,
   bit for bit, the unmasked call on parameters zeroed where pruned (mu = 0, rho = -inf: sigma = 0) in y, act_std,
   the input gradient and the kept elements' gradients.  Nets pruned by prune_by_snr likewise, through MCForward.
3. Pruned d mu and d rho are exactly 0 on every backward, the KL's included; a fully pruned layer without a bias has KL
   exactly 0.
4. NaN / inf in pruned mu / rho change no output.
5. A folded MCTrainStep and the sample loop agree with masks as they do without them.
6. A captured engine refuses to replay once a mask was first set, cleared or re-allocated; an in-place update is read by
   the next replay, with and without cached preps."""
import ctypes as C

import pytest
import torch

from oracle import bbb_oracle as O
from tests import forward_ref as R
from tests import mask_ref as MR
from tests.util import CFG_PRIORS, load_params_into

pytestmark = pytest.mark.gpu
PM, PS, SEED = 0.05, 0.1, 41


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _rand_mask(shape, keep, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.rand(shape, generator=g, device=dev) < keep


# ------------------------------------------------------------------------------------------- (1-4) the per-layer call
def _layer(cs, variant, math, inp, mask, first_image, bf16_act=False, eps=None, seed=7, stream=3):
    """One sampling layer call (external eps when given, else in-kernel noise); None when the desc is refused."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    x, W_mu, W_rho, b_mu, b_rho = inp
    dev = x.device
    fold = None if cs.fold is None or eps is not None else (cs.fold[0], R.FOLD_STRIDE)
    d = Fn.make_desc(tuple(x.shape), tuple(W_mu.shape), R.conv_of(cs), L.VARIANT_LRT if variant == "lrt" else L.VARIANT_BBB,
                     True, b_mu is not None, PM, PS, L.MATH_BY_NAME[math], L.KL_BY_NAME[cs.kl], L.ACT_BY_NAME[cs.act],
                     fold=fold, first_image=first_image)
    if bf16_act:
        ok, _ = Fn.layer_io(d, torch.bfloat16)
        if not ok:
            return None
        x = x.to(torch.bfloat16)
    if L.lib().bbb_forward_supported(C.byref(d)) != 0:
        return None
    ea = eb = None
    if eps is not None:
        ea, eb = (eps if variant == "bbb" else (eps, None))
    y = torch.empty(R.y_shape(cs, x.shape[0]), dtype=x.dtype, device=dev)
    std = torch.empty(R.y_shape(cs, x.shape[0]), dtype=torch.float32, device=dev) if variant == "lrt" else None
    kl = torch.full((), float("nan"), dtype=torch.float32, device=dev)
    ws = Fn.workspace(dev, d)
    fn = L.lib().bbb_linear_forward_prior if R.conv_of(cs) is None else L.lib().bbb_conv2d_forward_prior
    parg, flag = Fn.masked_prior_arg(None, mask)
    rc = fn(C.byref(Fn.desc_with(d, flag)), Fn._ptr(x), Fn._ptr(W_mu), Fn._ptr(W_rho), Fn._ptr(b_mu), Fn._ptr(b_rho), Fn._ptr(y),
            Fn._ptr(kl), Fn._ptr(std), Fn._ptr(ea), Fn._ptr(eb), C.c_uint64(seed), C.c_uint64(stream), None,
            Fn._ptr(ws), C.c_size_t(ws.numel()), Fn._stream(dev), parg)
    L.check(rc, "layer forward (mask)")
    torch.cuda.synchronize()
    return y, std, kl


def _zeroed(inp, mask):
    """The parameters an unmasked call must see to compute what the masked one does: mu = 0, rho = -inf where pruned."""
    x, W_mu, W_rho, b_mu, b_rho = inp
    wm, bm = mask
    W_mu, W_rho = W_mu.where(wm, 0.0), W_rho.where(wm, float("-inf"))
    if bm is not None:
        b_mu, b_rho = b_mu.where(bm, 0.0), b_rho.where(bm, float("-inf"))
    return x, W_mu.contiguous(), W_rho.contiguous(), b_mu, b_rho


def _poisoned(inp, mask):
    """NaN mu and inf rho (softplus overflows) at every pruned element."""
    x, W_mu, W_rho, b_mu, b_rho = inp
    wm, bm = mask
    W_mu, W_rho = W_mu.where(wm, float("nan")), W_rho.where(wm, 100.0)
    if bm is not None:
        b_mu, b_rho = b_mu.where(bm, float("nan")), b_rho.where(bm, float("inf"))
    return x, W_mu.contiguous(), W_rho.contiguous(), b_mu, b_rho


def _eq(a, b):
    return all((p is None and q is None) or torch.equal(p, q) for p, q in zip(a, b))


@pytest.mark.parametrize("cs", R.CASES, ids=[c.name for c in R.CASES])
def test_layer_forward_with_a_mask(dev, cs):
    ran = 0
    for variant in cs.variants:
        g = torch.Generator(device=dev).manual_seed(11)
        x, W_mu, W_rho, b_mu, b_rho, eps = R.make_inputs(cs, variant, g, device=dev)
        inp = (x, W_mu, W_rho, b_mu, b_rho)
        ones = (torch.ones_like(W_mu, dtype=torch.bool), None if b_mu is None else torch.ones_like(b_mu, dtype=torch.bool))
        fi = cs.fold[1] if cs.fold is not None and cs.fold[1] else 5
        for math in R.MATHS:
            for bf16_act in ((False, True) if math == "bf16" else (False,)):
                a = _layer(cs, variant, math, inp, None, fi, bf16_act)
                if a is None:
                    continue
                assert _eq(a, _layer(cs, variant, math, inp, ones, fi, bf16_act)), (cs.name, variant, math, bf16_act)
                ran += 1
                for k, keep in enumerate((0.5, 0.05)):
                    wm = _rand_mask(W_mu.shape, keep, 30 + k, dev)
                    bm = None if b_mu is None else _rand_mask(b_mu.shape, 0.5, 40 + k, dev)
                    mask = (wm, bm)
                    got = _layer(cs, variant, math, inp, mask, fi, bf16_act)
                    # bit for bit the unmasked call on zeroed parameters, and pruned mu / rho never reach an output
                    zero = _layer(cs, variant, math, _zeroed(inp, mask), None, fi, bf16_act)
                    assert _eq(got[:2], zero[:2]), (cs.name, variant, math, bf16_act, keep)
                    assert _eq(got, _layer(cs, variant, math, _poisoned(inp, mask), mask, fi, bf16_act)), (cs.name, variant, math, keep)
                    ref_kl = float(MR.kl_ref(W_mu, W_rho, b_mu, b_rho, wm, bm, PM, PS, cs.kl))
                    assert abs(float(got[2]) - ref_kl) <= 1e-5 * abs(ref_kl), (cs.name, variant, math, float(got[2]), ref_kl)
                    if bf16_act or cs.fold is not None:
                        continue
                    # against float64 on the same external eps
                    ext = _layer(cs, variant, math, inp, mask, 0, eps=eps)
                    if ext is None:
                        continue
                    ref, M, sd = MR.layer_ref(variant, x, W_mu, W_rho, b_mu, b_rho, wm, bm, eps, R.conv_of(cs), True, cs.act)
                    assert R.loose_err(ext[0], ref, M, math) <= 1.0, (cs.name, variant, math, keep)
                    if sd is not None and cs.act in (None, "none"):
                        assert R.std_err(ext[1], sd, math) <= 1.0, (cs.name, variant, math, keep)
    if not cs.refuse or len(cs.refuse) < len(R.MATHS):
        assert ran > 0, cs.name


def test_fully_pruned_layer_has_kl_zero(dev):
    import pytorch_bayesiancnn_b200 as bbb
    for cls in (bbb.BBBConv2d, bbb.BBBLRTConv2d):
        m = cls(3, 8, 3, bias=False).to(dev)
        m.set_weight_mask(torch.zeros_like(m.W_mu, dtype=torch.bool))
        for math in ("fp32", "bf16"):
            m.set_flag("math", math)
            x = torch.randn(4, 3, 8, 8, device=dev)
            with torch.no_grad():
                y = m(x)
            assert float(m.kl_loss().detach()) == 0.0
            m._kl_cache = None
            assert float(m.kl_loss().detach()) == 0.0           # the stand-alone KL kernel
            assert bool((y == 0).all()) if cls is bbb.BBBConv2d else bool(y.isfinite().all())


# ------------------------------------------------------------------------------------------ (1-4) the layer autograd
def _layer_grads(m, x, seed=5):
    import pytorch_bayesiancnn_b200 as bbb
    m.zero_grad()
    x = x.clone().requires_grad_(True)
    bbb.manual_seed(seed)
    y = m(x)
    g = torch.Generator(device=x.device).manual_seed(1)
    w = torch.randn(y.shape, generator=g, device=x.device)
    ((y * w).sum() + 0.3 * m.kl_loss()).backward()
    return y.detach(), x.grad, [p.grad.clone() for p in (m.W_mu, m.W_rho, m.bias_mu, m.bias_rho)]


def _same_grad(a, b, math):
    """Parameter gradients of two runs: bitwise on the tensor-core backward (no atomics); the CUDA-core wgrad (math
    'fp32') adds its M splits with atomics, in no fixed order, so there within fp32 rounding of the sum."""
    if math != "fp32":
        return torch.equal(a, b)
    return bool(((a - b).abs() <= 1e-5 * b.abs().max().clamp_min(1e-30)).all())


@pytest.mark.parametrize("math", ["fp32", "tf32", "bf16", "auto"])
@pytest.mark.parametrize("kind", ["conv", "linear"])
@pytest.mark.parametrize("variant", ["lrt", "bbb"])
def test_layer_backward_with_a_mask(dev, math, kind, variant):
    import pytorch_bayesiancnn_b200 as bbb
    torch.manual_seed(3)
    if kind == "conv":
        m = (bbb.BBBLRTConv2d if variant == "lrt" else bbb.BBBConv2d)(16, 64, 3, padding=1).to(dev)
        x = torch.randn(32, 16, 16, 16, device=dev)
    else:
        m = (bbb.BBBLRTLinear if variant == "lrt" else bbb.BBBLinear)(256, 128).to(dev)
        x = torch.randn(128, 256, device=dev)
    m.set_flag("math", math)
    m.train()
    base = _layer_grads(m, x)
    m.set_weight_mask(torch.ones_like(m.W_mu, dtype=torch.bool), torch.ones_like(m.bias_mu, dtype=torch.bool))
    ones = _layer_grads(m, x)
    assert torch.equal(base[0], ones[0]) and torch.equal(base[1], ones[1])
    for a, b in zip(base[2], ones[2]):
        assert _same_grad(a, b, math), (math, kind, variant)
    for keep in (0.5, 0.05):
        wm, bm = _rand_mask(m.W_mu.shape, keep, 7, dev), _rand_mask(m.bias_mu.shape, 0.5, 8, dev)
        m.set_weight_mask(wm, bm)
        y, gx, (gwm, gwr, gbm, gbr) = _layer_grads(m, x)
        for gr, mk in ((gwm, wm), (gwr, wm), (gbm, bm), (gbr, bm)):
            assert bool((gr[~mk] == 0).all()), (math, kind, variant, keep)
        # NaN / inf at pruned elements change nothing
        with torch.no_grad():
            saved = [p.clone() for p in (m.W_mu, m.W_rho, m.bias_mu, m.bias_rho)]
            m.W_mu.masked_fill_(~wm, float("nan")); m.W_rho.masked_fill_(~wm, 100.0)
            m.bias_mu.masked_fill_(~bm, float("inf")); m.bias_rho.masked_fill_(~bm, float("nan"))
        p = _layer_grads(m, x)
        assert torch.equal(p[0], y) and torch.equal(p[1], gx)
        for a, b in zip(p[2], (gwm, gwr, gbm, gbr)):
            assert _same_grad(a, b, math), (math, kind, variant, keep)
        with torch.no_grad():
            for t, s in zip((m.W_mu, m.W_rho, m.bias_mu, m.bias_rho), saved):
                t.copy_(s)
        # the data term equals the unmasked layer's on zeroed parameters (its KL is another matter: log 0)
        z = (bbb.BBBLRTConv2d if variant == "lrt" else bbb.BBBConv2d)(16, 64, 3, padding=1) if kind == "conv" else \
            (bbb.BBBLRTLinear if variant == "lrt" else bbb.BBBLinear)(256, 128)
        z = z.to(dev)
        z.set_flag("math", math)
        with torch.no_grad():
            z.W_mu.copy_(m.W_mu.where(wm, 0.0)); z.W_rho.copy_(m.W_rho.where(wm, -float("inf")))
            z.bias_mu.copy_(m.bias_mu.where(bm, 0.0)); z.bias_rho.copy_(m.bias_rho.where(bm, -float("inf")))
        bbb.manual_seed(5)
        xz = x.clone().requires_grad_(True)
        yz = z(xz)
        g = torch.Generator(device=dev).manual_seed(1)
        (yz * torch.randn(yz.shape, generator=g, device=dev)).sum().backward()
        assert torch.equal(yz.detach(), y), (math, kind, variant, keep)
        assert torch.equal(xz.grad, gx), (math, kind, variant, keep)
        # the KL part: the kept elements' terms (pruned ones contribute no value and no gradient)
        ref = float(MR.kl_ref(m.W_mu, m.W_rho, m.bias_mu, m.bias_rho, wm, bm, m.prior_mu, m.prior_sigma))
        assert abs(float(m.kl_loss().detach()) - ref) <= 1e-5 * abs(ref)


# ------------------------------------------------------------------------------------------------- (1, 2, 5, 6) nets
def _net(model, variant, dev, math="auto"):
    from pytorch_bayesiancnn_b200 import models as M
    cls = {"alexnet": M.BBBAlexNet, "lenet": M.BBBLeNet, "3conv3fc": M.BBB3Conv3FC}[model]
    params = O.init_params(model, 10, 3, CFG_PRIORS, seed=123)
    net = load_params_into(cls(10, 3, CFG_PRIORS, variant, "softplus"), params).to(dev).train()
    net.set_flag("math", math)
    return net


def _layers(net):
    return [m for m in net.modules() if hasattr(m, "W_mu")]


def _kl_net(net):
    return sum(float(MR.kl_ref(m.W_mu, m.W_rho, m.bias_mu, m.bias_rho, *(m.mask_tensors() or
               (torch.ones_like(m.W_mu, dtype=torch.bool), None)), m.prior_mu, m.prior_sigma)) for m in _layers(net))


@pytest.mark.parametrize("model", ["alexnet", "lenet", "3conv3fc"])
@pytest.mark.parametrize("variant", ["lrt", "bbb"])
def test_mc_forward_with_masks(dev, model, variant):
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import mc
    B = 128
    x = torch.randn(B, 3, 32, 32, generator=torch.Generator().manual_seed(2)).to(dev)
    labels = torch.randint(0, 10, (B,), generator=torch.Generator().manual_seed(3)).to(dev)
    net = _net(model, variant, dev)
    kw = dict(want_uncertainty=True, with_labels=True, train_size=100.0, beta=0.5, seed=SEED)
    configs = [dict(fold=True), dict(fold=False), dict(overlap=True, inflight=2), dict(cache_prep=False)]

    def run_all():
        outs = []
        for c in configs:
            eng = mc.MCForward(net, x, 4, **kw, **c)
            o = eng(x, labels)
            if c.get("inflight"):
                eng.wait()
            torch.cuda.synchronize()
            outs.append({k: v.clone() for k, v in o.items()})
        with torch.no_grad():
            y, kl = net(x)
        return outs, (y.clone(), float(kl))

    plain, py = run_all()
    for m in _layers(net):
        m.set_weight_mask(torch.ones_like(m.W_mu, dtype=torch.bool), torch.ones_like(m.bias_mu, dtype=torch.bool))
    ones, oy = run_all()
    for a, b in zip(plain, ones):
        for k in a:
            assert torch.equal(a[k], b[k]), (model, variant, k)
    assert py[1] == oy[1]
    for frac in (0.5, 0.95):
        for m in _layers(net):
            m.clear_weight_mask()
        bbb.prune_by_snr(net, frac)
        outs, (y, kl) = run_all()
        ref = _kl_net(net)
        assert abs(kl - ref) <= 1e-5 * abs(ref), (model, variant, frac, kl, ref)
        for o in outs:
            assert abs(float(o["kl"]) - ref) <= 1e-5 * abs(ref), (model, variant, frac)
            assert torch.isfinite(o["log_outputs"]).all()
        for k in outs[0]:                                       # captured, in flight and uncached: the same step
            assert torch.equal(outs[0][k], outs[2][k]) and torch.equal(outs[0][k], outs[3][k]), (model, variant, frac, k)


@pytest.mark.parametrize("math", ["tf32", "bf16"])
def test_train_step_with_masks(dev, math):
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import mc
    B, S = 64, 4
    net = _net("lenet", "lrt", dev, math)
    x = torch.rand(B, 3, 32, 32, generator=torch.Generator().manual_seed(4)).to(dev)
    labels = torch.randint(0, 10, (B,), generator=torch.Generator().manual_seed(5)).to(dev)
    params = [p for m in _layers(net) for p in (m.W_mu, m.W_rho, m.bias_mu, m.bias_rho)]

    def step(fold):
        net.zero_grad()
        out = mc.MCTrainStep(net, x, S, train_size=1000.0, seed=SEED, fold=fold)(x, labels, beta=0.1)
        torch.cuda.synchronize()
        return {k: v.clone() for k, v in out.items()}, [p.grad.clone() for p in params]

    base = {f: step(f) for f in (True, False)}
    for m in _layers(net):
        m.set_weight_mask(torch.ones_like(m.W_mu, dtype=torch.bool), torch.ones_like(m.bias_mu, dtype=torch.bool))
    for f in (True, False):
        o, g = step(f)
        for k in o:
            assert torch.equal(o[k], base[f][0][k]), (math, f, k)
        for a, b in zip(g, base[f][1]):
            assert torch.equal(a, b), (math, f)
    bbb.prune_by_snr(net, 0.9, biases=True)
    of, gf = step(True)
    ol, gl = step(False)
    for k in of:
        assert torch.equal(of[k], ol[k]), (math, k)            # as without masks (tests/test_gpu_train_fold.py)
    masks = [t for m in _layers(net) for t in (m.W_mask, m.W_mask, m.bias_mask, m.bias_mask)]
    for a, b, mk in zip(gf, gl, masks):
        assert bool((a[~mk] == 0).all()) and bool((b[~mk] == 0).all())
        assert float((a - b).abs().max()) <= 1e-4 * max(float(b.abs().max()), 1e-30), math
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    before = [p.detach().clone() for p in params]
    opt.step()
    for p, b0, mk in zip(params, before, masks):
        assert torch.equal(p.detach()[~mk], b0[~mk])           # Adam leaves zero-gradient elements where they are


def test_captured_engines_follow_the_mask(dev):
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import _lib as L, mc
    net = _net("alexnet", "lrt", dev)
    B, S = 128, 2
    x = torch.randn(B, 3, 32, 32, generator=torch.Generator().manual_seed(6)).to(dev)
    g = torch.Generator().manual_seed(8)
    loader = [(torch.randn(B, 3, 32, 32, generator=g), torch.randint(0, 10, (B,), generator=g)) for _ in range(2)]
    held = mc.MCForward(net, x, S, seed=SEED)
    graphed = bbb.GraphedForward(net, x)
    bbb.prune_by_snr(net, 0.5)                              # masks set for the first time: the captured graphs hold none
    with pytest.raises(L.EngineError, match="mask"):
        held(x)
    with pytest.raises(L.EngineError, match="mask"):
        graphed(x)
    for cache_prep in (True, False):
        eng = mc.MCForward(net, x, S, seed=SEED, cache_prep=cache_prep)
        k0 = float(eng(x)["kl"])
        ref = _kl_net(net)
        assert abs(k0 - ref) <= 1e-5 * abs(ref)
        ptrs = [m.W_mask.data_ptr() for m in _layers(net)]
        bbb.prune_by_snr(net, 0.9)                          # in place: the next replay reads it
        assert [m.W_mask.data_ptr() for m in _layers(net)] == ptrs
        k1 = float(eng(x)["kl"])
        ref = _kl_net(net)
        assert abs(k1 - ref) <= 1e-5 * abs(ref), (cache_prep, k1, ref)
        for m in _layers(net):
            m.set_weight_mask(torch.ones_like(m.W_mu, dtype=torch.bool))
        assert float(eng(x)["kl"]) == float(mc.MCForward(net, x, S, seed=SEED, cache_prep=cache_prep)(x)["kl"])
        bbb.prune_by_snr(net, 0.5)
    # the engines evaluate() / mc_forward keep on the net are rebuilt after a clear
    ev0 = mc.evaluate(net, loader, S, train_size=100.0, seed=SEED)
    for m in _layers(net):
        m.clear_weight_mask()
    ev1 = mc.evaluate(net, loader, S, train_size=100.0, seed=SEED)
    ref = _kl_net(net)
    assert abs(ev1["klsum"] / S - ref) <= 1e-5 * abs(ref)
    assert ev0["klsum"] != ev1["klsum"]

"""Per-weight Gaussian priors on the GPU: every KL path of the engine with a tensor prior (bbb_prior).

1. Constant fill, bitwise: a tensor prior filled with the desc's scalars gives the scalar call's y, act_std and KL bit for
   bit -- on every case of tests/forward_ref.CASES (fp32, tf32, bf16 and bf16 activations; BBB and LRT; folded and
   unfolded; a nonzero first image), on the fused BBBAlexNet chain (LRT and BBB, folded, through MCForward) and on the
   stand-alone kl_forward / kl_backward (KLFn), gradients included.
2. Random priors, mu_p = W_mu + N(0, 0.05), sigma_p = softplus(W_rho + N(0, 0.5)), in both KL conventions: the KL
   against float64 within 1e-5 relative on the same paths, and the KL backward against float64 autograd within
   1e-5 M per element (M: the sum of the absolute values of the terms of the derivative).
3. Continual learning: BBBLeNet (LRT) trained on a synthetic task A with MCTrainStep(fold=True), then posterior_as_prior:
   every layer's KL is ~0, and a task-B step's gradients match float64 oracle autograd of the ELBO under that prior.
4. Captured engines: MCForward (captured, and with steps in flight) with tensor priors gives the eager KL and head, and
   an in-place set_prior after capture moves the KL of the next replay.  The engines mc_forward and evaluate() keep on
   the net follow posterior_as_prior / clear_prior; a captured MCForward or GraphedForward refuses to replay once a
   layer's prior buffers were replaced or removed (they would otherwise read freed memory)."""
import ctypes as C

import pytest
import torch

from oracle import bbb_oracle as O
from tests import forward_ref as R
from tests.util import CFG_PRIORS, load_params_into, scale_err

pytestmark = pytest.mark.gpu
PM, PS = 0.05, 0.1                 # the desc's scalar prior in the constant-fill checks
MC_NS, SEED = 1 << 63, 41


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _softplus(t):
    return torch.log1p(torch.exp(t))


def _const_prior(W_mu, b_mu, pm=PM, ps=PS):
    return (torch.full_like(W_mu, pm), torch.full_like(W_mu, ps),
            None if b_mu is None else torch.full_like(b_mu, pm), None if b_mu is None else torch.full_like(b_mu, ps))


def _random_prior(W_mu, W_rho, b_mu, b_rho, seed):
    g = torch.Generator(device=W_mu.device).manual_seed(seed)
    rn = lambda t, s: t + s * torch.randn(t.shape, generator=g, device=t.device)
    return (rn(W_mu, 0.05).contiguous(), _softplus(rn(W_rho, 0.5)).contiguous(),
            None if b_mu is None else rn(b_mu, 0.05).contiguous(), None if b_mu is None else _softplus(rn(b_rho, 0.5)).contiguous())


def _kl64(W_mu, W_rho, b_mu, b_rho, prior, conv):
    """float64 KL of a layer against the tensor prior: the weight and the bias part, each against its own tensors."""
    f = O.kl_loss if conv == "reference" else O.kl_textbook
    d = lambda t: None if t is None else t.double()
    kl = f(d(W_mu), d(W_rho), None, None, d(prior[0]), d(prior[1]))
    if b_mu is not None:
        kl = kl + f(d(b_mu), d(b_rho), None, None, d(prior[2]), d(prior[3]))
    return kl


# ------------------------------------------------------------------------- (1, 2) the per-layer forward, every case
def _layer(cs, variant, math, inp, prior, conv, first_image, bf16_act=False, seed=7, stream=3):
    """One sampling layer call with in-kernel noise, as BayesLayerFn.forward makes it; None when the desc is refused."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    x, W_mu, W_rho, b_mu, b_rho = inp
    dev = x.device
    fold = None if cs.fold is None else (cs.fold[0], R.FOLD_STRIDE)
    d = Fn.make_desc(tuple(x.shape), tuple(W_mu.shape), R.conv_of(cs), L.VARIANT_LRT if variant == "lrt" else L.VARIANT_BBB,
                     True, b_mu is not None, PM, PS, L.MATH_BY_NAME[math], L.KL_BY_NAME[conv], L.ACT_BY_NAME[cs.act],
                     fold=fold, first_image=first_image)
    if bf16_act:
        ok, _ = Fn.layer_io(d, torch.bfloat16)
        if not ok:
            return None
        x = x.to(torch.bfloat16)
    if L.lib().bbb_forward_supported(C.byref(d)) != 0:
        return None
    y = torch.empty(R.y_shape(cs, x.shape[0]), dtype=x.dtype, device=dev)
    std = torch.empty(R.y_shape(cs, x.shape[0]), dtype=torch.float32, device=dev) if variant == "lrt" else None
    kl = torch.full((), float("nan"), dtype=torch.float32, device=dev)
    ws = Fn.workspace(dev, d)
    fn = L.lib().bbb_linear_forward_prior if R.conv_of(cs) is None else L.lib().bbb_conv2d_forward_prior
    rc = fn(C.byref(d), Fn._ptr(x), Fn._ptr(W_mu), Fn._ptr(W_rho), Fn._ptr(b_mu), Fn._ptr(b_rho), Fn._ptr(y),
            Fn._ptr(kl), Fn._ptr(std), None, None, C.c_uint64(seed), C.c_uint64(stream), None, Fn._ptr(ws),
            C.c_size_t(ws.numel()), Fn._stream(dev), Fn.prior_arg(prior))
    L.check(rc, "layer forward (prior)")
    torch.cuda.synchronize()
    return y, std, kl


def _first_image(cs):
    if cs.fold is not None and cs.fold[1]:
        return cs.fold[1]
    return 5


@pytest.mark.parametrize("cs", R.CASES, ids=[c.name for c in R.CASES])
def test_layer_forward_with_a_tensor_prior(dev, cs):
    ran = 0
    for variant in cs.variants:
        g = torch.Generator(device=dev).manual_seed(11)
        x, W_mu, W_rho, b_mu, b_rho, _ = R.make_inputs(cs, variant, g, device=dev)
        inp = (x, W_mu, W_rho, b_mu, b_rho)
        const = _const_prior(W_mu, b_mu)
        fi = _first_image(cs)
        for math in R.MATHS:
            for bf16_act in ((False, True) if math == "bf16" else (False,)):
                a = _layer(cs, variant, math, inp, None, cs.kl, fi, bf16_act)
                if a is None:
                    continue
                b = _layer(cs, variant, math, inp, const, cs.kl, fi, bf16_act)
                assert torch.equal(a[0], b[0]), (cs.name, variant, math, bf16_act, "y")
                if a[1] is not None:
                    assert torch.equal(a[1], b[1]), (cs.name, variant, math, bf16_act, "act_std")
                assert torch.equal(a[2], b[2]), (cs.name, variant, math, bf16_act, float(a[2]), float(b[2]))
                ran += 1
                if bf16_act:
                    continue
                for k, conv in enumerate(("reference", "textbook")):
                    prior = _random_prior(W_mu, W_rho, b_mu, b_rho, 100 + k)
                    _, _, kl = _layer(cs, variant, math, inp, prior, conv, fi)
                    ref = float(_kl64(W_mu, W_rho, b_mu, b_rho, prior, conv))
                    assert abs(float(kl) - ref) <= 1e-5 * abs(ref), (cs.name, variant, math, conv, float(kl), ref)
    if not cs.refuse or len(cs.refuse) < len(R.MATHS):
        assert ran > 0, cs.name


# ----------------------------------------------------------------------------- (1, 2) the stand-alone KL and its backward
def _kl_grad_terms(mu, rho, pm, ps, conv):
    """float64 d kl / d mu and d kl / d rho of every element, and M: the sum of the absolute values of their terms."""
    mu, rho, pm, ps = mu.double(), rho.double(), pm.double(), ps.double()
    s, sg, d = _softplus(rho), torch.sigmoid(rho), mu - pm
    if conv == "reference":
        dm, Mm = d / s ** 2, d.abs() / s ** 2
        t = (1 / s, -ps ** 2 / s ** 3, -d ** 2 / s ** 3)
    else:
        dm, Mm = d / ps ** 2, d.abs() / ps ** 2
        t = (-1 / s, s / ps ** 2)
    return dm, sum(t) * sg, Mm, sum(x.abs() for x in t) * sg


@pytest.mark.parametrize("conv", ["reference", "textbook"])
def test_kl_forward_and_backward_with_a_tensor_prior(dev, conv):
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import _lib as L
    for shape, bias in (((192, 64, 5, 5), True), ((1000, 1000), True), ((10, 84), False), ((7, 3, 3, 3), True)):
        m = (bbb.BBBConv2d(shape[1], shape[0], shape[2:]) if len(shape) == 4 else bbb.BBBLinear(shape[1], shape[0], bias=bias)).to(dev)
        m.prior_mu, m.prior_sigma, m.kl_convention = PM, PS, conv
        params = [m.W_mu, m.W_rho] + ([m.bias_mu, m.bias_rho] if bias else [])

        def kl_and_grads(prior):
            k = bbb.functional.KLFn.apply(m.W_mu, m.W_rho, m.bias_mu, m.bias_rho, PM, PS, L.KL_BY_NAME[conv], prior)
            gs = torch.autograd.grad(k * 3.0, params)
            return k.detach(), gs
        k0, g0 = kl_and_grads(None)
        k1, g1 = kl_and_grads(_const_prior(m.W_mu.detach(), m.bias_mu.detach() if bias else None))
        assert torch.equal(k0, k1), (shape, conv)
        for a, b in zip(g0, g1):
            assert torch.equal(a, b), (shape, conv)
        prior = _random_prior(m.W_mu.detach(), m.W_rho.detach(), m.bias_mu.detach() if bias else None,
                              m.bias_rho.detach() if bias else None, 7)
        k2, g2 = kl_and_grads(prior)
        ref = float(_kl64(m.W_mu, m.W_rho, m.bias_mu, m.bias_rho, prior, conv))
        assert abs(float(k2) - ref) <= 1e-5 * abs(ref), (shape, conv, float(k2), ref)
        parts = [(m.W_mu, m.W_rho, prior[0], prior[1])] + ([(m.bias_mu, m.bias_rho, prior[2], prior[3])] if bias else [])
        for i, (mu, rho, pm, ps) in enumerate(parts):
            dm, dr, Mm, Mr = _kl_grad_terms(mu.detach(), rho.detach(), pm, ps, conv)
            # float64 autograd of the oracle, and the restated derivative with its magnitude
            mu64, rho64 = mu.detach().double().requires_grad_(True), rho.detach().double().requires_grad_(True)
            f = O.kl_loss if conv == "reference" else O.kl_textbook
            am, ar = torch.autograd.grad(3.0 * f(mu64, rho64, None, None, pm.double(), ps.double()), (mu64, rho64))
            assert float((am - 3.0 * dm).abs().max()) <= 1e-9 * float(3.0 * Mm.max())
            assert float((g2[2 * i] - am).abs().sub(1e-5 * 3.0 * Mm).max()) <= 0, (shape, conv, i, "mu")
            assert float((g2[2 * i + 1] - ar).abs().sub(1e-5 * 3.0 * Mr).max()) <= 0, (shape, conv, i, "rho")


# ----------------------------------------------------------------------------------------- (1, 2) the fused chain
def _alexnet(variant, dev, math="auto"):
    from pytorch_bayesiancnn_b200 import models as M
    params = O.init_params("alexnet", 10, 3, CFG_PRIORS, seed=123)
    net = load_params_into(M.BBBAlexNet(10, 3, CFG_PRIORS, variant, "softplus"), params).to(dev).train()
    net.set_flag("math", math)
    return net


def _layers(net):
    return [m for m in net.modules() if hasattr(m, "W_mu")]


@pytest.mark.parametrize("variant", ["lrt", "bbb"])
def test_fused_chain_with_a_tensor_prior(dev, variant):
    from pytorch_bayesiancnn_b200 import mc
    B = 128
    x = torch.randn(B, 3, 32, 32, generator=torch.Generator().manual_seed(2)).to(dev)
    labels = torch.randint(0, 10, (B,), generator=torch.Generator().manual_seed(3)).to(dev)
    net = _alexnet(variant, dev)
    kw = dict(want_uncertainty=True, with_labels=True, train_size=100.0, beta=0.5, seed=SEED, graph=False)
    # the folded MC step (fused chain over 4 samples in one pass) against the same step with a constant tensor prior
    outs = []
    for prior in (False, True):
        for m in _layers(net):
            m.clear_prior()
            m.prior_mu = PM
            if prior:
                m.set_prior(PM, PS, PM, PS)
            m.prior_sigma = PS
        eng = mc.MCForward(net, x, 4, **kw)
        out = eng(x, labels)
        torch.cuda.synchronize()
        outs.append({k: v.clone() for k, v in out.items()})
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), (variant, k)
    # random priors: each layer's KL from the fused chain's prep kernels against float64, both conventions
    for k, conv in enumerate(("reference", "textbook")):
        net.set_flag("kl_convention", conv)
        priors = []
        for i, m in enumerate(_layers(net)):
            p = _random_prior(m.W_mu.detach(), m.W_rho.detach(), m.bias_mu.detach(), m.bias_rho.detach(), 50 + 10 * k + i)
            m.set_prior(*p)
            priors.append(p)
        with torch.no_grad():
            _, kl_sum = net(x)
        assert net._fused_plans.get(tuple(x.shape)) is not None, "the fused chain did not run"
        total = 0.0
        for m, p in zip(_layers(net), priors):
            ref = float(_kl64(m.W_mu, m.W_rho, m.bias_mu, m.bias_rho, p, conv))
            kl_m, versions, _ = m._kl_cache               # the scalar the chain's prep kernel wrote
            assert versions == m._versions()
            got = float(kl_m)
            assert abs(got - ref) <= 1e-5 * abs(ref), (variant, conv, got, ref)
            total += ref
        assert abs(float(kl_sum) - total) <= 1e-5 * abs(total)


# ----------------------------------------------------------------------------------------- (3) continual learning
def _oracle_elbo_grads(params, priors, x, labels, eps_per_sample, train_size, beta):
    """main_bayesian.py:46-58 through float64 autograd on the oracle, with each layer's KL against its tensor prior."""
    P = [{k: v.double().clone().requires_grad_(True) for k, v in p.items()} for p in params]
    outs = [O.net_forward("lenet", P, x.double(), [e.double() for e in eps], "lrt", "softplus", 0.0, 0.1, 10)[0]
            for eps in eps_per_sample]
    kl = sum(_kl64(p["W_mu"], p["W_rho"], p["bias_mu"], p["bias_rho"], q, "reference") for p, q in zip(P, priors))
    nll = torch.nn.functional.nll_loss(O.mc_combine(outs), labels, reduction="mean")
    (nll * train_size + beta * kl).backward()
    return nll.detach(), kl.detach(), [p[k].grad for p in P for k in ("W_mu", "W_rho", "bias_mu", "bias_rho")]


def test_continual_learning_run(dev):
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import mc, models as M
    from tests.test_gpu_mc import _engine_eps
    B, S, train_size, beta = 64, 4, 50.0, 1.0
    params = O.init_params("lenet", 10, 3, CFG_PRIORS, seed=9)
    net = load_params_into(M.BBBLeNet(10, 3, CFG_PRIORS, "lrt", "softplus"), params).to(dev).train()
    net.set_flag("math", "tf32")
    g = torch.Generator().manual_seed(1)
    # task A: labels a fixed function of the image (the sign pattern of 10 random projections)
    proj = torch.randn(10, 3 * 32 * 32, generator=g)
    xa = torch.rand(B, 3, 32, 32, generator=g)
    la = (xa.flatten(1) @ proj.t()).argmax(1)
    xa, la = xa.to(dev), la.to(dev)
    step = mc.MCTrainStep(net, xa, S, train_size=train_size, seed=SEED, fold=True)
    assert step.layer_fold is not None
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    for _ in range(5):
        step(xa, la, beta=beta)
        opt.step()
    bbb.posterior_as_prior(net)
    for m in _layers(net):
        n = m.W_mu.numel() + m.bias_mu.numel()
        assert abs(float(m.kl_loss())) <= 1e-6 * n, float(m.kl_loss())          # the stand-alone KL kernel
    with torch.no_grad(), bbb.functional.layer_fold(B, 1 << 40):
        net(torch.cat([xa, xa]))                                                # a folded forward: the prep kernels' KL
    for m in _layers(net):
        n = m.W_mu.numel() + m.bias_mu.numel()
        assert abs(float(m._kl_cache[0])) <= 1e-6 * n, float(m._kl_cache[0])
    # one task-B step against float64 oracle autograd of the ELBO under the posterior-of-A prior
    xb = torch.rand(B, 3, 32, 32, generator=g).to(dev)
    lb = torch.randint(0, 10, (B,), generator=g).to(dev)
    step_b = mc.MCTrainStep(net, xb, S, train_size=train_size, seed=SEED + 1, fold=True)
    out = step_b(xb, lb, beta=beta)
    torch.cuda.synchronize()
    got = [p.grad.clone() for m in _layers(net) for p in (m.W_mu, m.W_rho, m.bias_mu, m.bias_rho)]
    eps = [[e.to(dev) for e in _engine_eps(bbb, "lenet", 10, 3, "lrt", B, SEED + 1, MC_NS | (j << 40), dev)]
           for j in range(S)]
    cur = [{k: getattr(m, k).detach() for k in ("W_mu", "W_rho", "bias_mu", "bias_rho")} for m in _layers(net)]
    ref_nll, ref_kl, ref_grads = _oracle_elbo_grads(cur, [m.prior_tensors() for m in _layers(net)], xb, lb, eps,
                                                    train_size, beta)
    # head = {nll * train_size + beta * kl, nll, accuracy, beta * kl}: the NLL at the tf32 bar of tests/test_gpu_train_fold.py;
    # the KL, a sum of ~62k terms that are each ~0 here, at the bar of a KL at its minimum (1e-6 per element)
    assert abs(float(out["head"][1]) - float(ref_nll)) <= 2e-5 * abs(float(ref_nll)), (float(out["head"][1]), float(ref_nll))
    n_all = sum(m.W_mu.numel() + m.bias_mu.numel() for m in _layers(net))
    assert abs(float(out["head"][3]) - beta * float(ref_kl)) <= beta * 1e-6 * n_all, (float(out["head"][3]), float(ref_kl))
    errs = [scale_err(a, b) for a, b in zip(got, ref_grads)]
    assert max(errs) <= 2.5e-2, errs                      # the tf32 bar of tests/test_gpu_train_fold.py


# ------------------------------------------------------------------------------------------- (4) captured engines
def test_captured_engines_read_the_tensor_prior(dev):
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import functional as Fn, mc
    from pytorch_bayesiancnn_b200.graph import _STRIDE
    net = _alexnet("lrt", dev)
    B = 128
    x = torch.randn(B, 3, 32, 32, generator=torch.Generator().manual_seed(6)).to(dev)
    labels = torch.randint(0, 10, (B,), generator=torch.Generator().manual_seed(7)).to(dev)
    for i, m in enumerate(_layers(net)):
        m.set_prior(*_random_prior(m.W_mu.detach(), m.W_rho.detach(), m.bias_mu.detach(), m.bias_rho.detach(), 200 + i))
    kw = dict(want_uncertainty=True, with_labels=True, train_size=100.0, beta=0.5, seed=SEED)
    cap = mc.MCForward(net, x, 4, **kw)
    fly = mc.MCForward(net, x, 4, overlap=True, inflight=2, **kw)

    def eager_kl():
        with Fn.stream_base(torch.zeros(1, dtype=torch.int64, device=dev)), Fn.mc_sample(0, SEED), torch.no_grad():
            return float(net(x)[1])

    for rnd in range(2):
        out = cap(x, labels)
        torch.cuda.synchronize()
        o1 = {k: v.clone() for k, v in out.items()}
        of = fly(x, labels)
        fly.wait()
        torch.cuda.synchronize()
        for k in o1:
            assert torch.equal(o1[k], of[k]), (rnd, k)
        kl = eager_kl()
        assert abs(float(o1["kl"]) - kl) <= 1e-6 * abs(kl), (rnd, float(o1["kl"]), kl)
        nll = float(torch.nn.functional.nll_loss(o1["log_outputs"], labels))
        assert abs(float(o1["head"][3]) - 0.5 * kl) <= 1e-6 * abs(0.5 * kl)
        assert abs(float(o1["head"][0]) - (nll * 100.0 + 0.5 * kl)) <= 1e-4 * abs(nll * 100.0 + 0.5 * kl)
        if rnd == 0:
            before = float(o1["kl"])
            ptrs = [m.W_prior_mu.data_ptr() for m in _layers(net)]
            for i, m in enumerate(_layers(net)):                 # in place: the captured graphs keep their addresses
                m.set_prior(*_random_prior(m.W_mu.detach(), m.W_rho.detach(), m.bias_mu.detach(), m.bias_rho.detach(), 300 + i))
            assert [m.W_prior_mu.data_ptr() for m in _layers(net)] == ptrs
    assert float(o1["kl"]) != before
    assert cap.timeouts() == 0 and fly.timeouts() == 0


def _kl_total(net):
    return sum(float(_kl64(m.W_mu, m.W_rho, m.bias_mu, m.bias_rho,
                           m.prior_tensors() or _const_prior(m.W_mu, m.bias_mu, float(m.prior_mu), float(m.prior_sigma)),
                           "reference")) for m in _layers(net))


def test_cached_engines_follow_the_prior(dev):
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import _lib as L, mc
    net = _alexnet("lrt", dev)
    B, S = 128, 2
    g = torch.Generator().manual_seed(8)
    loader = [(torch.randn(B, 3, 32, 32, generator=g), torch.randint(0, 10, (B,), generator=g)) for _ in range(2)]
    x = loader[0][0].to(dev)
    n_all = sum(m.W_mu.numel() + m.bias_mu.numel() for m in _layers(net))

    def both():
        ev = mc.evaluate(net, loader, S, train_size=100.0, seed=SEED)
        _, kl = mc.mc_forward(net, x, S, seed=SEED)
        torch.cuda.synchronize()
        return ev["klsum"] / S, float(kl)

    ref = _kl_total(net)                                     # the scalar prior
    for got in both():
        assert abs(got - ref) <= 1e-5 * abs(ref), (got, ref)
    held = mc.MCForward(net, x, S, seed=SEED)                # captured on the scalar prior
    graphed = bbb.GraphedForward(net, x)
    bbb.posterior_as_prior(net)                              # the cached engines (same keys) must not keep the scalar
    for got in both():
        assert abs(got) <= 1e-6 * n_all, got
    with pytest.raises(L.EngineError, match="prior"):
        held(x)
    with pytest.raises(L.EngineError, match="prior"):
        graphed(x)
    for i, m in enumerate(_layers(net)):                     # in place: the cached engines are kept and read it
        m.set_prior(*_random_prior(m.W_mu.detach(), m.W_rho.detach(), m.bias_mu.detach(), m.bias_rho.detach(), 400 + i))
    engines = dict(net._mc_engines)
    ref = _kl_total(net)
    for got in both():
        assert abs(got - ref) <= 1e-5 * abs(ref), (got, ref)
    assert net._mc_engines == engines
    tensor_eng = mc.MCForward(net, x, S, seed=SEED)           # captured on the tensor prior
    for m in _layers(net):
        m.clear_prior()                                      # frees nothing a captured graph reads: the replay is refused
    torch.cuda.empty_cache()
    with pytest.raises(L.EngineError, match="prior"):
        tensor_eng(x)
    ref = _kl_total(net)                                     # the scalar prior again, in new engines
    for got in both():
        assert abs(got - ref) <= 1e-5 * abs(ref), (got, ref)

"""The scale-mixture prior on the GPU: the Monte-Carlo KL kernels against the float64 restatement (tests/kl_mc_ref.py) on
the engine's own normals, and every path that returns a KL for nets whose layers have such a prior.

1. Kernels: value (1e-5 relative) and gradients (1e-4 scale-relative) at every layer shape of the three models, with
   and without bias, 1 and 4 draws, 16-byte-aligned and unaligned pointers; extreme parameters stay finite and within
   the bar; draw d of a multi-draw call (4 draws, and 20: more than one launch takes) equals the single-draw call on
   stream + d * stride bit for bit.
2. Layers: the prior does not move the layer's own noise -- y and the input gradient are bitwise those of the
   scalar-prior layer -- and the layer's KL is the stand-alone draw on the next stream id.
3. MCForward on BBBAlexNet (fused chain, folded) and BBBLeNet (per-layer fold): kl bitwise the sample loop's and the mean
   of the per-sample stand-alone draws on the expected streams; every replay of a captured engine draws anew, serial or
   with steps in flight; GraphedForward likewise; a net with Gaussian and mixture layers side by side.
4. MCTrainStep, sample loop and folded: kl, and the KL's share of the parameter gradients against the float64 restatement.
5. Two GPUs (skipped on one): the same kl on both ranks and as on one GPU."""
import math
import os

import pytest
import torch

from tests import kl_mc_ref as K
from tests.util import CFG_PRIORS, load_params_into, scale_err

pytestmark = pytest.mark.gpu
MC_NS, SEED = 1 << 63, 29
MIX = (0.5, 1.0, math.exp(-6))
MODELS = {"alexnet": 3, "lenet": 3, "3conv3fc": 1}


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _net(key, variant, dev, math_="bf16", mixture=MIX, only=None):
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import models as M
    from oracle import bbb_oracle as O
    cls = {"alexnet": M.BBBAlexNet, "lenet": M.BBBLeNet, "3conv3fc": M.BBB3Conv3FC}[key]
    params = O.init_params(key, 10, MODELS[key], CFG_PRIORS, seed=123)
    net = load_params_into(cls(10, MODELS[key], CFG_PRIORS, variant, "softplus"), params).to(dev).train()
    net.set_flag("math", math_)
    layers = _layers(net)
    for i, m in enumerate(layers):
        if mixture is not None and (only is None or i in only):
            m.set_mixture_prior(*mixture)
    return net


def _layers(net):
    return [m for m in net.children() if hasattr(m, "W_mu")]


def _f32(mix):
    return tuple(torch.tensor(mix, dtype=torch.float32).tolist())


def _forward(W_mu, W_rho, b_mu, b_rho, mix, seed, stream, n_draws=1, stride=0):
    from pytorch_bayesiancnn_b200 import functional as Fn
    kl = torch.empty(n_draws, dtype=torch.float32, device=W_mu.device)
    Fn.kl_mc_forward(kl, W_mu, W_rho, b_mu, b_rho, mix, seed, stream, None, stride)
    return kl


def _backward(mu, rho, first, mix, seed, stream, gkl, stride=0):
    import ctypes as C
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    g_mu, g_rho = torch.zeros_like(mu), torch.zeros_like(rho)
    rc = L.lib().bbb_kl_mc_backward(Fn._ptr(mu), Fn._ptr(rho), mu.numel(), first, Fn.mixture_arg(mix), seed, stream, None,
                                    gkl.numel(), C.c_uint64(stride), Fn._ptr(gkl), Fn._ptr(g_mu), Fn._ptr(g_rho),
                                    Fn._stream(mu.device))
    L.check(rc, "bbb_kl_mc_backward")
    return g_mu, g_rho


def _eps(n, seed, stream, offset, dev):
    import pytorch_bayesiancnn_b200 as bbb
    return bbb.philox_normal(n, seed, stream, offset, device=dev)


def _ref(W_mu, W_rho, b_mu, b_rho, mix, seed, stream):
    """float64 value of one draw on (seed, stream), from the engine's normals at the draw indices."""
    pi, s1, s2 = _f32(mix)
    parts = [(W_mu.reshape(-1), W_rho.reshape(-1), _eps(W_mu.numel(), seed, stream, 0, W_mu.device))]
    if b_mu is not None:
        parts.append((b_mu, b_rho, _eps(b_mu.numel(), seed, stream, W_mu.numel(), W_mu.device)))
    return K.kl_mc(parts, pi, s1, s2)


def _layer_ref(m, seed, stream, mix=MIX):
    return _ref(m.W_mu.detach(), m.W_rho.detach(), m.bias_mu.detach(), m.bias_rho.detach(), mix, seed, stream)


def _unaligned(t):
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    buf[1:].copy_(t.reshape(-1))
    return buf[1:]


# ------------------------------------------------------------------------------------------------ (1) the kernels
@pytest.mark.parametrize("aligned", [True, False], ids=["aligned", "unaligned"])
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("key", list(MODELS))
def test_kernels_match_float64(dev, key, bias, aligned):
    net = _net(key, "lrt", dev, mixture=None)
    stride = 1 << 40
    for li, m in enumerate(_layers(net)):
        fix = (lambda t: t) if aligned else _unaligned
        W_mu, W_rho = fix(m.W_mu.detach().reshape(-1)), fix(m.W_rho.detach().reshape(-1))
        b_mu, b_rho = (fix(m.bias_mu.detach()), fix(m.bias_rho.detach())) if bias else (None, None)
        for n_draws in (1, 4):
            stream = 100 + li
            kl = _forward(W_mu, W_rho, b_mu, b_rho, MIX, SEED, stream, n_draws, stride)
            gkl = torch.linspace(0.5, 1.5, n_draws, device=dev)
            want_mu, want_rho = torch.zeros_like(W_mu, dtype=torch.float64), torch.zeros_like(W_mu, dtype=torch.float64)
            for d in range(n_draws):
                ref = _ref(W_mu, W_rho, b_mu, b_rho, MIX, SEED, stream + d * stride)
                assert abs(float(kl[d]) - float(ref)) <= 1e-5 * abs(float(ref)), (key, li, n_draws, d, float(kl[d]), float(ref))
                gm, gr = K.kl_mc_grads(W_mu, W_rho, _eps(W_mu.numel(), SEED, stream + d * stride, 0, dev), *_f32(MIX))
                want_mu += float(gkl[d]) * gm
                want_rho += float(gkl[d]) * gr
            g_mu, g_rho = _backward(W_mu, W_rho, 0, MIX, SEED, stream, gkl, stride)
            assert scale_err(g_mu, want_mu) < 1e-4 and scale_err(g_rho, want_rho) < 1e-4, (key, li, n_draws)
            if bias and n_draws == 4:
                nw = W_mu.numel()
                g_mu, g_rho = _backward(b_mu, b_rho, nw, MIX, SEED, stream, gkl, stride)
                wm, wr = torch.zeros_like(b_mu, dtype=torch.float64), torch.zeros_like(b_mu, dtype=torch.float64)
                for d in range(n_draws):
                    gm, gr = K.kl_mc_grads(b_mu, b_rho, _eps(b_mu.numel(), SEED, stream + d * stride, nw, dev), *_f32(MIX))
                    wm += float(gkl[d]) * gm
                    wr += float(gkl[d]) * gr
                assert scale_err(g_mu, wm) < 1e-4 and scale_err(g_rho, wr) < 1e-4, (key, li, "bias")


@pytest.mark.parametrize("rho", [-12.0, 5.0])
@pytest.mark.parametrize("mix", [(0.5, 1.0, math.exp(-8)), (1.0, 0.1, 1.0), (0.25, 0.5, math.exp(-6))])
def test_extreme_parameters_stay_finite(dev, rho, mix):
    n = 10007
    g = torch.Generator(device=dev).manual_seed(5)
    mu = (torch.rand(n, generator=g, device=dev) * 6.0 - 3.0).contiguous()           # |mu| up to 3
    mu[:4] = torch.tensor([3.0, -3.0, 0.0, 1e-6], device=dev)
    rh = torch.full((n,), rho, device=dev)
    kl = _forward(mu, rh, mu[:64].clone(), rh[:64].clone(), mix, SEED, 7)
    ref = _ref(mu, rh, mu[:64].clone(), rh[:64].clone(), mix, SEED, 7)
    assert torch.isfinite(kl).all() and abs(float(kl) - float(ref)) <= 1e-5 * abs(float(ref)), (float(kl), float(ref))
    g_mu, g_rho = _backward(mu, rh, 0, mix, SEED, 7, torch.ones(1, device=dev))
    gm, gr = K.kl_mc_grads(mu, rh, _eps(n, SEED, 7, 0, dev), *_f32(mix))
    assert torch.isfinite(g_mu).all() and torch.isfinite(g_rho).all()
    assert scale_err(g_mu, gm) < 1e-4 and scale_err(g_rho, gr) < 1e-4


@pytest.mark.parametrize("n_draws", [4, 20])
def test_draw_d_is_the_single_draw_call_on_its_stream(dev, n_draws):
    m = _layers(_net("lenet", "bbb", dev, mixture=None))[2]                          # fc1: 48000 weights + 120 bias
    args = (m.W_mu.detach(), m.W_rho.detach(), m.bias_mu.detach(), m.bias_rho.detach(), MIX, SEED)
    stride = 3 << 40
    many = _forward(*args, MC_NS + 11, n_draws, stride)
    again = _forward(*args, MC_NS + 11, n_draws, stride)
    assert torch.equal(many, again) and len(set(many.tolist())) == n_draws
    gkl = torch.rand(n_draws, device=dev)
    g_many = _backward(args[0], args[1], 0, MIX, SEED, MC_NS + 11, gkl, stride)
    acc = [torch.zeros_like(args[0]), torch.zeros_like(args[0])]
    for d in range(n_draws):
        one = _forward(*args, MC_NS + 11 + d * stride)
        assert torch.equal(one[0], many[d]), d
        g = _backward(args[0], args[1], 0, MIX, SEED, MC_NS + 11 + d * stride, gkl[d:d + 1])
        acc = [a + b for a, b in zip(acc, g)]
    assert scale_err(g_many[0], acc[0]) < 1e-6 and scale_err(g_many[1], acc[1]) < 1e-6


# ------------------------------------------------------------------------------------------------- (2) the layers
@pytest.mark.parametrize("math_", ["fp32", "bf16", "tf32"])
@pytest.mark.parametrize("variant", ["bbb", "lrt"])
def test_the_prior_does_not_move_the_layer_noise(dev, variant, math_):
    import pytorch_bayesiancnn_b200 as bbb
    conv = (bbb.BBBConv2d if variant == "bbb" else bbb.BBBLRTConv2d)(16, 64, 3, padding=1, priors=CFG_PRIORS).to(dev)
    lin = (bbb.BBBLinear if variant == "bbb" else bbb.BBBLRTLinear)(256, 128, priors=CFG_PRIORS).to(dev)
    for layer, shape in ((conv, (128, 16, 8, 8)), (lin, (128, 256))):
        layer.set_flag("math", math_)
        x = torch.randn(shape, generator=torch.Generator().manual_seed(1)).to(dev).requires_grad_(True)
        res = []
        for mix in (None, MIX):
            layer.clear_prior() if mix is None else layer.set_mixture_prior(*mix)
            bbb.manual_seed(SEED, 40)
            y = layer(x)
            kl = layer.kl_loss()
            assert kl is layer.kl_loss()                                   # the forward's draw, not a second one
            gx, = torch.autograd.grad(y, x, torch.ones_like(y))
            res.append((y.detach().clone(), gx.clone(), kl))
        assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
        kl = res[1][2]
        ref = _layer_ref(layer, SEED, 41)                                  # the id behind the layer's own (40)
        assert kl.dim() == 0 and abs(float(kl.detach()) - float(ref)) <= 1e-5 * abs(float(ref))
        # gradients through the layer's KL, and a kl_loss() without a forward draws on the next stream id (42)
        g = torch.autograd.grad(kl, [layer.W_mu, layer.W_rho, layer.bias_mu, layer.bias_rho])
        pi, s1, s2 = _f32(MIX)
        want = K.kl_mc_grads(layer.W_mu.detach().reshape(-1), layer.W_rho.detach().reshape(-1),
                             _eps(layer.W_mu.numel(), SEED, 41, 0, dev), pi, s1, s2)
        assert scale_err(g[0].reshape(-1), want[0]) < 1e-4 and scale_err(g[1].reshape(-1), want[1]) < 1e-4
        wb = K.kl_mc_grads(layer.bias_mu.detach(), layer.bias_rho.detach(),
                           _eps(layer.bias_mu.numel(), SEED, 41, layer.W_mu.numel(), dev), pi, s1, s2)
        assert scale_err(g[2], wb[0]) < 1e-4 and scale_err(g[3], wb[1]) < 1e-4
        with torch.no_grad():
            layer.W_mu.add_(0.0)                                           # a new parameter version: the cache is stale
        fresh = layer.kl_loss()
        ref = _layer_ref(layer, SEED, 42)
        assert abs(float(fresh.detach()) - float(ref)) <= 1e-5 * abs(float(ref))


# -------------------------------------------------------------------------------------------- (3) MCForward, graphs
def _expected_kl(net, seed, ids, replay, mixed=None):
    """Mean over the samples `ids` of the net's KL in float64: mixture layers from stand-alone draws on the streams a layer
    call of sample j takes at replay `replay` (layer stream, then the KL's), Gaussian layers (`mixed`) from kl_loss()."""
    from pytorch_bayesiancnn_b200.graph import _STRIDE
    tot = 0.0
    for j in ids:
        sid = (MC_NS | (j << 40)) + replay * _STRIDE
        for m in _layers(net):
            sid += 1                                                       # the layer's own noise stream
            if m.mixture_values() is None:
                m._kl_cache = None
                tot += float(m.kl_loss().detach())
            else:
                tot += float(_layer_ref(m, seed, sid, m.mixture_values()))
                sid += 1
    return tot / len(ids)


@pytest.mark.parametrize("key,variant,B", [("alexnet", "lrt", 64), ("alexnet", "bbb", 128), ("lenet", "lrt", 64),
                                           ("lenet", "bbb", 128)])
def test_mc_forward_fold_equals_loop_and_the_expected_draws(dev, key, variant, B):
    from pytorch_bayesiancnn_b200 import mc
    S = 4
    net = _net(key, variant, dev)
    x = torch.rand(B, MODELS[key], 32, 32, generator=torch.Generator().manual_seed(2)).to(dev)
    labels = torch.randint(0, 10, (B,), generator=torch.Generator().manual_seed(3)).to(dev)
    kw = dict(with_labels=True, train_size=1000.0, beta=0.1, seed=SEED)
    folded = mc.MCForward(net, x, S, **kw)
    loop = mc.MCForward(net, x, S, fold=False, **kw)
    flight = mc.MCForward(net, x, S, overlap=True, inflight=2, **kw)
    assert (folded.fold_steps is not None) if key == "alexnet" else (folded.layer_fold is not None or variant == "bbb")
    assert loop.fold_steps is None and loop.layer_fold is None
    kls = []
    for replay in range(3):
        a = {k: v.clone() for k, v in folded(x, labels).items()}
        b = {k: v.clone() for k, v in loop(x, labels).items()}
        flight(x, labels)
        c = {k: v.clone() for k, v in flight.wait().items()}
        torch.cuda.synchronize()
        for k in ("kl", "log_outputs", "head"):
            assert torch.equal(a[k], b[k]) and torch.equal(a[k], c[k]), (replay, k)
        want = _expected_kl(net, SEED, range(S), replay)
        assert abs(float(a["kl"]) - want) <= 2e-6 * abs(want), (replay, float(a["kl"]), want)
        kls.append(float(a["kl"]))
    assert len(set(kls)) == 3                                               # every replay draws anew
    eager = mc.MCForward(net, x, S, graph=False, **kw)(x, labels)
    assert torch.equal(eager["kl"].cpu(), torch.tensor(kls[0]))
    # new values are kernel arguments: the captured engines refuse to replay, the cached ones are rebuilt
    _layers(net)[0].set_mixture_prior(0.5, 1.0, math.exp(-7))
    with pytest.raises(Exception, match="prior"):
        folded(x, labels)


def test_mixed_net_and_graphed_forward(dev):
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import mc
    from pytorch_bayesiancnn_b200.graph import _STRIDE
    net = _net("lenet", "lrt", dev, only=(1, 3))
    net.fc3.set_prior(0.01, 0.2)                                            # Gaussian scalar, mixture and tensor priors
    x = torch.rand(64, 3, 32, 32, generator=torch.Generator().manual_seed(2)).to(dev)
    folded = mc.MCForward(net, x, 3, seed=SEED)
    loop = mc.MCForward(net, x, 3, seed=SEED, fold=False)
    a, b = folded(x)["kl"].clone(), loop(x)["kl"].clone()
    want = _expected_kl(net, SEED, range(3), 0)
    assert torch.equal(a, b) and abs(float(a) - want) <= 1e-5 * abs(want)      # the Gaussian terms: the KL parity bar
    # GraphedForward: replay r draws first_stream + r * 2^20 + (layer, KL, layer, KL, ...)
    net = _net("alexnet", "lrt", dev)
    x = torch.rand(32, 3, 32, 32, generator=torch.Generator().manual_seed(2)).to(dev)
    bbb.manual_seed(SEED)
    gf = bbb.GraphedForward(net, x, first_stream=5)
    for r in range(2):
        _, kl = gf(x)
        want = sum(float(_layer_ref(m, SEED, 5 + r * _STRIDE + 2 * i + 1)) for i, m in enumerate(_layers(net)))
        assert abs(float(kl) - want) <= 2e-6 * abs(want), r
    # and the plain eager forward, fused and layer by layer, on the same streams
    for fuse in (True, False):
        net.set_flag("fuse", fuse)
        bbb.manual_seed(SEED, 5)
        with torch.no_grad():
            _, kl = net(x)
        want = sum(float(_layer_ref(m, SEED, 5 + 2 * i + 1)) for i, m in enumerate(_layers(net)))
        assert kl.dim() == 0 and abs(float(kl) - want) <= 2e-6 * abs(want), fuse


def test_evaluate_with_a_mixture_prior(dev):
    from pytorch_bayesiancnn_b200 import mc
    net = _net("lenet", "lrt", dev)
    g = torch.Generator().manual_seed(6)
    data = [(torch.rand(32, 3, 32, 32, generator=g), torch.randint(0, 10, (32,), generator=g)) for _ in range(3)]
    m = mc.evaluate(net, data, num_ens=2, train_size=1000.0, seed=SEED, inflight=2)
    want = sum(2 * _expected_kl(net, SEED, range(2), r) for r in range(3)) / 3      # klsum: sum_j kl_j, mean over steps
    assert m["steps"] == 3 and abs(m["klsum"] - want) <= 2e-6 * abs(want)


# ----------------------------------------------------------------------------------------------- (4) MCTrainStep
@pytest.mark.parametrize("fold", [False, True], ids=["loop", "fold"])
def test_training_step_kl_and_gradients(dev, fold):
    from pytorch_bayesiancnn_b200 import mc
    B, S, beta = 64, 2, 1.0
    net = _net("lenet", "lrt", dev)
    x = torch.rand(B, 3, 32, 32, generator=torch.Generator().manual_seed(4)).to(dev)
    labels = torch.randint(0, 10, (B,), generator=torch.Generator().manual_seed(5)).to(dev)
    grads, outs = {}, {}
    for b_ in (0.0, beta):                                  # fresh engines: both draw noise block 0
        step = mc.MCTrainStep(net, x, S, train_size=60000.0, seed=SEED, fold=fold)
        assert (step.layer_fold is not None) == fold
        out = step(x, labels, b_)
        torch.cuda.synchronize()
        grads[b_] = [p.grad.clone() for p in step.params]
        outs[b_] = {k: v.clone() for k, v in out.items()}
    want = _expected_kl(net, SEED, range(S), 0)
    assert torch.equal(outs[0.0]["kl"], outs[beta]["kl"]) and torch.equal(outs[0.0]["log_outputs"], outs[beta]["log_outputs"])
    assert abs(float(outs[beta]["kl"]) - want) <= 2e-6 * abs(want)
    assert abs(float(outs[beta]["head"][3]) - beta * want) <= 2e-6 * abs(beta * want)
    # the KL's share of the gradients, beta / S * sum_j d KL_j: the difference of the two steps against the restatement
    pi, s1, s2 = _f32(MIX)
    names = [n for n, p in net.named_parameters() if p.requires_grad]
    by_name = {n: g1 - g0 for n, g0, g1 in zip(names, grads[0.0], grads[beta])}
    worst = 0.0
    for li, (lname, m) in enumerate((n, m) for n, m in net.named_children() if hasattr(m, "W_mu")):
        nw = m.W_mu.numel()
        for mu, rho, first, pn in ((m.W_mu, m.W_rho, 0, "W"), (m.bias_mu, m.bias_rho, nw, "bias")):
            wm = torch.zeros(mu.numel(), dtype=torch.float64, device=dev)
            wr = torch.zeros_like(wm)
            for j in range(S):
                e = _eps(mu.numel(), SEED, (MC_NS | (j << 40)) + 2 * li + 1, first, dev)
                gm, gr = K.kl_mc_grads(mu.detach().reshape(-1), rho.detach().reshape(-1), e, pi, s1, s2)
                wm += beta / S * gm
                wr += beta / S * gr
            # the difference of two fp32 gradients carries the rounding of the likelihood's share
            for got, ref, g0 in ((by_name[f"{lname}.{pn}_mu"], wm, grads[0.0][names.index(f"{lname}.{pn}_mu")]),
                                 (by_name[f"{lname}.{pn}_rho"], wr, grads[0.0][names.index(f"{lname}.{pn}_rho")])):
                tol = 1e-4 * float(ref.abs().max()) + 4e-7 * float(g0.abs().max() + ref.abs().max())
                worst = max(worst, float((got.reshape(-1).double() - ref).abs().max()) / tol)
    assert worst <= 1.0, worst


def test_folded_training_step_equals_the_sample_loop_with_a_mixture(dev):
    from pytorch_bayesiancnn_b200 import mc
    net = _net("lenet", "lrt", dev, only=(0, 2, 4))                          # Gaussian layers in between
    x = torch.rand(64, 3, 32, 32, generator=torch.Generator().manual_seed(4)).to(dev)
    labels = torch.randint(0, 10, (64,), generator=torch.Generator().manual_seed(5)).to(dev)
    res = []
    for fold in (False, True):
        step = mc.MCTrainStep(net, x, 5, train_size=60000.0, seed=SEED, fold=fold, fold_group=2 if fold else None)
        out = step(x, labels, 0.3)
        torch.cuda.synchronize()
        res.append(({k: v.clone() for k, v in out.items()}, [p.grad.clone() for p in step.params]))
    for k in ("kl", "log_outputs", "head"):
        assert torch.equal(res[0][0][k], res[1][0][k]), k
    for a, b in zip(res[0][1], res[1][1]):
        assert scale_err(b, a) < 1e-4


# --------------------------------------------------------------------------------------------------- (5) two GPUs
def _mp_worker(rank, world, port, out_path):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from pytorch_bayesiancnn_b200 import mc
    res = {}
    for rb in (1, 2):
        net = _net("lenet", "lrt", dev)
        x = torch.rand(64, 3, 32, 32, generator=torch.Generator().manual_seed(3)).to(dev)
        y = torch.randint(0, 10, (64,), generator=torch.Generator().manual_seed(4)).to(dev)
        ts = mc.MCTrainStep(net, x, 4, train_size=1000.0, seed=9, batch_shards=rb, fold=True)
        out = ts(x, y, beta=0.1)
        torch.cuda.synchronize()
        res[rb] = out["kl"].cpu()
        ts.close()
    torch.save(res, out_path + f".{rank}")
    dist.destroy_process_group()


def test_two_gpus_give_the_kl_of_one(dev):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import socket
    import tempfile
    import torch.multiprocessing as mp
    from pytorch_bayesiancnn_b200 import mc
    world = 2
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out_path = os.path.join(tempfile.mkdtemp(), "kl_mc")
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_mp_worker, args=(r, world, port, out_path)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0
    outs = [torch.load(out_path + f".{r}") for r in range(world)]
    net = _net("lenet", "lrt", dev)
    x = torch.rand(64, 3, 32, 32, generator=torch.Generator().manual_seed(3)).to(dev)
    y = torch.randint(0, 10, (64,), generator=torch.Generator().manual_seed(4)).to(dev)
    one = mc.MCTrainStep(net, x, 4, train_size=1000.0, seed=9, fold=True)(x, y, beta=0.1)["kl"].cpu()
    for rb in (1, 2):
        assert torch.equal(outs[0][rb], outs[1][rb]), rb                     # the same bits on both ranks
        # the per-sample estimates do not depend on the sharding; the ranks' partial sums are added in another order
        assert abs(float(outs[0][rb]) - float(one)) <= 1e-6 * abs(float(one)), rb

"""The folded training step on the GPU: bbb_lrt_noise_grad, autograd through layer_fold(grad=True), and
MCTrainStep(fold=True) against the sample loop and float64 oracle autograd -- at the LRT layer geometries of the three
models (tests/backward_ref.py's tables)."""
import ctypes as C
import os
from types import SimpleNamespace

import pytest
import torch

from tests import backward_ref as R
from tests.util import CFG_PRIORS, load_params_into, scale_err

pytestmark = pytest.mark.gpu
MC_NS = 1 << 63
STRIDE = 1 << 40
SEED = 31


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _geometries():
    """(name, cin, cout, k, s, p, hw) of every Bayesian layer of the three models; k = None: linear."""
    out = []
    for prefix, table in (("alexnet", R._ALEXNET), ("lenet", R._LENET), ("3conv3fc", R._3CONV3FC)):
        for tag, cin, cout, k, s, p, hw in table:
            out.append((f"{prefix}_{tag}", cin, cout, k, s, p, hw))
    return out


GEOMS = _geometries()
GEOM_IDS = [g[0] for g in GEOMS]


def _conv(g):
    _, _, _, k, s, p, _ = g
    return None if k is None else ((s, s), (p, p), (1, 1))


def _x_shape(g, B):
    _, cin, _, k, _, _, hw = g
    return (B, cin) if k is None else (B, cin, hw, hw)


def _w_shape(g):
    _, cin, cout, k, _, _, _ = g
    return (cout, cin) if k is None else (cout, cin, k, k)


def _y_shape(g, B):
    from pytorch_bayesiancnn_b200 import functional as Fn
    _, _, cout, k, _, _, hw = g
    return (B, cout) if k is None else (B, cout) + Fn.out_hw(hw, hw, k, k, _conv(g))


def _eps(shape, seed, stream, first_image, dev):
    """The eps the forward of a layer call of output `shape` draws (NHWC element index from its first image), NCHW."""
    from pytorch_bayesiancnn_b200 import functional as Fn
    B = shape[0]
    per = 1
    for d in shape[1:]:
        per *= d
    z = Fn.philox_normal(B * per, seed, stream, first_image * per, device=dev)
    if len(shape) == 2:
        return z.view(shape)
    return z.view(B, shape[2], shape[3], shape[1]).permute(0, 3, 1, 2)


def _desc(g, B, math, fold=None, first=0):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    return Fn.make_desc(_x_shape(g, B), _w_shape(g), _conv(g), L.VARIANT_LRT, True, True, 0.0, 0.1, math,
                        fold=fold, first_image=first)


# --------------------------------------------------------------------------------------------------- (1) the kernel
@pytest.mark.parametrize("geom", GEOMS, ids=GEOM_IDS)
def test_noise_grad_kernel_is_the_elementwise_chain(dev, geom):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    gen = torch.Generator(device=dev).manual_seed(3)
    B, G = 5, 3
    for first, base_val, fold in ((0, None, False), (37, None, False), (0, 11, False), (123, 7, False),
                                  (0, None, True), (41, 5, True)):
        rows = G * B if fold else B
        ys = _y_shape(geom, rows)
        gy = torch.randn(ys, device=dev, generator=gen)
        act_std = torch.rand(ys, device=dev, generator=gen) + 0.05
        base = None if base_val is None else torch.tensor([base_val], dtype=torch.int64, device=dev)
        stream = 1000 + 3 * first
        d = _desc(geom, rows, L.MATH_BF16_TC, fold=(B, STRIDE) if fold else None, first=first)
        gv = Fn.lrt_noise_grad(d, gy, act_std, SEED, stream, base)
        s0 = stream + (base_val or 0)
        if fold:
            eps = torch.cat([_eps(_y_shape(geom, B), SEED, s0 + j * STRIDE, first, dev) for j in range(G)])
        else:
            eps = _eps(ys, SEED, s0, first, dev)
        ref = gy * eps / (2.0 * act_std)
        torch.cuda.synchronize()
        assert torch.equal(gv, ref), (geom[0], first, base_val, fold, (gv - ref).abs().max().item())


# ------------------------------------------------------------------------ (2) the unfolded backward, as the parent
def _layer_forward(geom, B, math, first, base, dev, gen):
    """A forward of an LRT layer call through the C ABI: (x, W_mu, W_rho, bias_mu, bias_rho, act_std, desc)."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    ws = _w_shape(geom)
    x = torch.randn(_x_shape(geom, B), device=dev, generator=gen)
    W_mu = torch.randn(ws, device=dev, generator=gen) * 0.1
    W_rho = torch.randn(ws, device=dev, generator=gen) * 0.1 - 5.0
    b_mu = torch.randn(ws[0], device=dev, generator=gen) * 0.1
    b_rho = torch.randn(ws[0], device=dev, generator=gen) * 0.1 - 5.0
    d = _desc(geom, B, math, first=first)
    ys = _y_shape(geom, B)
    y, act_std = torch.empty(ys, device=dev), torch.empty(ys, device=dev)
    kl = torch.empty((), device=dev)
    wsp = Fn.workspace(dev, d)
    fn = L.lib().bbb_linear_forward if geom[3] is None else L.lib().bbb_conv2d_forward
    L.check(fn(C.byref(d), Fn._ptr(x), Fn._ptr(W_mu), Fn._ptr(W_rho), Fn._ptr(b_mu), Fn._ptr(b_rho), Fn._ptr(y),
               Fn._ptr(kl), Fn._ptr(act_std), None, None, C.c_uint64(SEED), C.c_uint64(77), Fn._ptr(base),
               Fn._ptr(wsp), C.c_size_t(wsp.numel()), Fn._stream(dev)), "forward")
    return x, W_mu, W_rho, b_mu, b_rho, act_std, d


@pytest.mark.parametrize("math", ["bf16", "tf32"])
@pytest.mark.parametrize("geom", GEOMS, ids=GEOM_IDS)
def test_unfolded_tc_backward_is_bit_identical_to_the_aten_chain(dev, geom, math):
    """The LRT tensor-core backward with gv from bbb_lrt_noise_grad == the computation it replaces: eps from
    philox_normal, the NHWC -> NCHW permute and gy * eps / (2 act_std) in aten ops, the same contractions."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    gen = torch.Generator(device=dev).manual_seed(5)
    m = L.MATH_BY_NAME[math]
    for first, base_val in ((0, None), (29, 4)):
        base = None if base_val is None else torch.tensor([base_val], dtype=torch.int64, device=dev)
        x, W_mu, W_rho, b_mu, b_rho, act_std, d = _layer_forward(geom, 6, m, first, base, dev, gen)
        gy = torch.randn(act_std.shape, device=dev, generator=gen)
        cfg = {"conv": _conv(geom), "variant": L.VARIANT_LRT, "sample": True, "math": m}
        ctx = SimpleNamespace(saved_tensors=(x, W_mu, W_rho, b_mu, b_rho, act_std, None, None), cfg=cfg, desc=d,
                              noise=(SEED, 77, base), first_image=first, needs_input_grad=(True,) * 5, has_bias=True,
                              fold=None)
        got = Fn.BayesLayerFn._backward_tc(ctx, gy)
        # the parent's computation
        conv = _conv(geom)
        stream_id = 77 + (int(base.item()) if base is not None else 0)
        eps = _eps(gy.shape, SEED, stream_id, first, dev)
        sig, dsig = torch.log1p(torch.exp(W_rho)), torch.sigmoid(W_rho)
        red = (0,) if conv is None else (0, 2, 3)
        gw_mu = Fn._tc_wgrad(x, gy, conv, W_mu.shape)
        gv = gy * eps / (2.0 * act_std)
        gw_rho = Fn._tc_wgrad(x * x, gv, conv, W_mu.shape) * (2.0 * sig * dsig)
        gx = Fn._tc_dgrad(gy, W_mu, conv, x.shape) + 2.0 * x * Fn._tc_dgrad(gv, sig * sig, conv, x.shape)
        gb_mu = gy.sum(red)
        gb_rho = gv.sum(red) * (2.0 * torch.log1p(torch.exp(b_rho)) * torch.sigmoid(b_rho))
        torch.cuda.synchronize()
        for name, a, b in zip(("gx", "gw_mu", "gw_rho", "gb_mu", "gb_rho"), got, (gx, gw_mu, gw_rho, gb_mu, gb_rho)):
            assert torch.equal(a, b), (geom[0], math, first, name)


# --------------------------------------------------------------------- (3) a folded layer against per-sample calls
def _layer(geom, dev, math):
    from pytorch_bayesiancnn_b200 import modules as M
    _, cin, cout, k, s, p, _ = geom
    torch.manual_seed(11)
    layer = M.BBBLRTLinear(cin, cout, priors=CFG_PRIORS) if k is None else \
        M.BBBLRTConv2d(cin, cout, k, stride=s, padding=p, priors=CFG_PRIORS)
    layer = layer.to(dev).train()
    layer.set_flag("math", math)
    return layer


@pytest.mark.parametrize("math", ["bf16", "tf32"])
@pytest.mark.parametrize("geom", GEOMS, ids=GEOM_IDS)
def test_folded_layer_backward_equals_per_sample_backwards(dev, geom, math):
    from pytorch_bayesiancnn_b200 import functional as Fn
    layer = _layer(geom, dev, math)
    params = [layer.W_mu, layer.W_rho, layer.bias_mu, layer.bias_rho]
    B, G = 8, 3
    gen = torch.Generator(device=dev).manual_seed(7)
    x = torch.randn(_x_shape(geom, B), device=dev, generator=gen)
    gy = torch.randn(_y_shape(geom, G * B), device=dev, generator=gen)
    for b0 in (0, 45):
        for p in params:
            p.grad = None
        xf = x.repeat((G,) + (1,) * (x.dim() - 1)).requires_grad_(True)
        with Fn.mc_sample(2, SEED), Fn.first_image(b0), Fn.layer_fold(B, STRIDE, grad=True):
            yf = layer(xf)
        yf.backward(gy)
        folded = [p.grad.clone() for p in params]
        acc = [torch.zeros_like(p) for p in params]
        for j in range(G):
            for p in params:
                p.grad = None
            xj = x.clone().requires_grad_(True)
            with Fn.mc_sample(2 + j, SEED), Fn.first_image(b0):
                yj = layer(xj)
            yj.backward(gy[j * B:(j + 1) * B])
            for a, p in zip(acc, params):
                a += p.grad
            assert torch.equal(yj, yf[j * B:(j + 1) * B].detach()), (geom[0], b0, j)
            assert torch.equal(xj.grad, xf.grad[j * B:(j + 1) * B]), (geom[0], b0, j)
        for i, (a, b) in enumerate(zip(folded, acc)):
            assert scale_err(a, b) < 1e-4, (geom[0], math, b0, i, scale_err(a, b))


# ------------------------------------------------------------------- (4) MCTrainStep(fold=True) against fold=False
def _net(key, variant, dev, math, inputs):
    from pytorch_bayesiancnn_b200 import models as M
    from oracle import bbb_oracle as O
    cls = {"alexnet": M.BBBAlexNet, "lenet": M.BBBLeNet, "3conv3fc": M.BBB3Conv3FC}[key]
    params = O.init_params(key, 10, inputs, CFG_PRIORS, seed=123)
    net = load_params_into(cls(10, inputs, CFG_PRIORS, variant, "softplus"), params).to(dev).train()
    net.set_flag("math", math)
    return net, params


def _run(step, x, labels, beta):
    """Two consecutive steps; (kernels of the second, outputs and per-sample logits of each, gradients of the second)."""
    from pytorch_bayesiancnn_b200 import _lib as L
    res = []
    for _ in range(2):
        n0 = L.launch_count()
        out = step(x, labels, beta=beta)
        torch.cuda.synchronize()
        res.append(({k: v.clone() for k, v in out.items()}, step.logits.clone(), L.launch_count() - n0))
    return res, [p.grad.clone() for p in step.params]


# (relative error of the loss, scale-relative error of every parameter gradient) against float64 oracle autograd: the
# bars of tests/test_gpu_backward_geometry.py's training test
TRAIN_BAR = {"bf16": (9e-4, 5e-2), "tf32": (2e-5, 2.5e-2)}
NETS = (("lenet", 3), ("3conv3fc", 1), ("alexnet", 3))


@pytest.mark.parametrize("math", ["bf16", "tf32"])
@pytest.mark.parametrize("key,inputs", NETS)
def test_folded_training_step_equals_the_sample_loop(dev, key, inputs, math):
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import mc
    from pytorch_bayesiancnn_b200.graph import _STRIDE
    from tests.test_gpu_mc import _engine_eps, _oracle_train_grads
    B, S, beta, train_size = 96, 4, 0.1, 5000.0
    net, params = _net(key, "lrt", dev, math, inputs)
    x = torch.rand(B, inputs, 32, 32, generator=torch.Generator().manual_seed(4)).to(dev)
    labels = torch.randint(0, 10, (B,), generator=torch.Generator().manual_seed(5)).to(dev)
    loop = mc.MCTrainStep(net, x, S, train_size=train_size, seed=SEED)
    folded = mc.MCTrainStep(net, x, S, train_size=train_size, seed=SEED, fold=True)
    assert loop.layer_fold is None and folded.layer_fold == (S, 1)
    ra, ga = _run(loop, x, labels, beta)
    rb, gb = _run(folded, x, labels, beta)
    for (oa, la, na), (ob, lb, nb) in zip(ra, rb):
        assert torch.equal(la, lb)
        for k in ("log_outputs", "kl", "head"):
            assert torch.equal(oa[k], ob[k]), k
        assert nb < na, (nb, na)
    for i, (a, b) in enumerate(zip(ga, gb)):
        assert scale_err(b, a) < 1e-4, (key, math, i, scale_err(b, a))
    # the second step (noise block 1) against float64 oracle autograd on the same noise
    eps = [[e.to(dev) for e in _engine_eps(bbb, key, 10, inputs, "lrt", B, SEED, (MC_NS | (j << 40)) + _STRIDE, dev)]
           for j in range(S)]
    P = [{k: v.to(dev) for k, v in p.items()} for p in params]
    ref_loss, ref_grads = _oracle_train_grads(key, P, x, labels, eps, "lrt", 10, train_size, beta, dtype=torch.float64)
    e_loss = abs(float(rb[1][0]["head"][0]) - float(ref_loss)) / abs(float(ref_loss))
    errs = [scale_err(a, b) for a, b in zip(gb, ref_grads)]
    assert e_loss <= TRAIN_BAR[math][0], e_loss
    assert max(errs) <= TRAIN_BAR[math][1], errs


def test_uneven_groups(dev):
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", "lrt", dev, "bf16", 3)
    x = torch.rand(64, 3, 32, 32, generator=torch.Generator().manual_seed(1)).to(dev)
    labels = torch.randint(0, 10, (64,), generator=torch.Generator().manual_seed(2)).to(dev)
    loop = mc.MCTrainStep(net, x, 5, train_size=1000.0, seed=SEED)
    folded = mc.MCTrainStep(net, x, 5, train_size=1000.0, seed=SEED, fold=True, fold_group=2)
    assert folded.layer_fold == (2, 3) and folded._groups == [(0, 2), (2, 2), (4, 1)]
    ra, ga = _run(loop, x, labels, 0.3)
    rb, gb = _run(folded, x, labels, 0.3)
    for (oa, la, _), (ob, lb, _) in zip(ra, rb):
        assert torch.equal(la, lb)
        for k in ("log_outputs", "kl", "head"):
            assert torch.equal(oa[k], ob[k]), k
    for a, b in zip(ga, gb):
        assert scale_err(b, a) < 1e-4


# ------------------------------------------------------------------------------- (5) refusals and unchanged paths
def test_layer_fold_grad_refusals(dev):
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    x = torch.randn(256, 3, 32, 32, device=dev)
    for variant, math, msg in (("bbb", "bf16", "BBB layer"), ("lrt", "fp32", "fp32")):
        net, _ = _net("lenet", variant, dev, math, 3)
        with pytest.raises(L.EngineError, match=msg), Fn.layer_fold(128, STRIDE, grad=True):
            net(x)
    net, _ = _net("lenet", "lrt", dev, "bf16", 3)
    with pytest.raises(L.EngineError, match="no external eps"), Fn.layer_fold(128, STRIDE, grad=True), \
            bbb.external_eps([torch.zeros(256, 6, 28, 28)]):
        net(x)
    with pytest.raises(L.EngineError, match="forward-only"), Fn.layer_fold(128, STRIDE):
        net(x)                                                        # grad=False keeps refusing autograd
    assert not Fn.layer_fold_active()


@pytest.mark.parametrize("variant,math", [("bbb", "bf16"), ("lrt", "fp32")])
def test_fold_true_keeps_the_sample_loop_where_it_cannot_fold(dev, variant, math):
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", variant, dev, math, 3)
    x = torch.rand(64, 3, 32, 32, generator=torch.Generator().manual_seed(1)).to(dev)
    labels = torch.randint(0, 10, (64,), generator=torch.Generator().manual_seed(2)).to(dev)
    a = mc.MCTrainStep(net, x, 3, train_size=1000.0, seed=SEED)
    b = mc.MCTrainStep(net, x, 3, train_size=1000.0, seed=SEED, fold=True)
    assert b.layer_fold is None
    ra, ga = _run(a, x, labels, 0.1)
    rb, gb = _run(b, x, labels, 0.1)
    for (oa, la, na), (ob, lb, nb) in zip(ra, rb):
        assert torch.equal(la, lb) and na == nb
        for k in oa:
            assert torch.equal(oa[k], ob[k]), k
    # the tensor-core backward is deterministic; the CUDA-core one (math='fp32') accumulates with float atomics, so two
    # runs of the same sample loop differ in the order of their sums
    for x_, y_ in zip(ga, gb):
        assert torch.equal(x_, y_) if math != "fp32" else scale_err(y_, x_) < 1e-5


# ------------------------------------------------------------------------------------------------- (6) two GPUs
def _mp_worker(rank, world, port, out_path):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from pytorch_bayesiancnn_b200 import mc
    res = {}
    for rb in (1, 2):
        net, _ = _net("lenet", "lrt", dev, "bf16", 3)
        x = torch.rand(64, 3, 32, 32, generator=torch.Generator().manual_seed(3)).to(dev)
        y = torch.randint(0, 10, (64,), generator=torch.Generator().manual_seed(4)).to(dev)
        ts = mc.MCTrainStep(net, x, 4, train_size=1000.0, seed=9, batch_shards=rb, fold=True)
        assert ts.layer_fold is not None
        out = ts(x, y, beta=0.1)
        torch.cuda.synchronize()
        res[rb] = (out["head"].cpu(), [p.grad.cpu() for p in net.parameters()])
        ts.close()
    torch.save(res, out_path + f".{rank}")
    dist.destroy_process_group()


def test_two_gpus_folded_equals_one_gpu(dev):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import socket
    import tempfile
    import torch.multiprocessing as mp
    from pytorch_bayesiancnn_b200 import mc
    world = 2
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out_path = os.path.join(tempfile.mkdtemp(), "train_fold")
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_mp_worker, args=(r, world, port, out_path)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0
    outs = [torch.load(out_path + f".{r}") for r in range(world)]
    net, _ = _net("lenet", "lrt", dev, "bf16", 3)
    x = torch.rand(64, 3, 32, 32, generator=torch.Generator().manual_seed(3)).to(dev)
    y = torch.randint(0, 10, (64,), generator=torch.Generator().manual_seed(4)).to(dev)
    ts = mc.MCTrainStep(net, x, 4, train_size=1000.0, seed=9, fold=True)
    out = ts(x, y, beta=0.1)
    torch.cuda.synchronize()
    for rb in (1, 2):
        head, grads = outs[0][rb]
        assert (out["head"].cpu() - head).abs().max() <= 1e-4 * float(head.abs().max()), rb
        for p, g in zip(net.parameters(), grads):
            assert scale_err(p.grad, g) < 1e-4, rb

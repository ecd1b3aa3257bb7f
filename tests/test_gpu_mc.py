"""The Monte-Carlo step above the Bayesian layers on the GPU product path (SURVEY.md 8e, f3, f4) and the BASELINE
configurations at full size (C2, C4, C5) -- through the package API (-> ctypes -> C ABI), checked against the oracle on
IDENTICAL noise: the engine draws its Philox streams in-kernel, the test draws the same streams on the host side of
the boundary (bbb_philox_normal_fill) and feeds them to the oracle as the reference's eps tensors.

Multi-rank logic on ONE GPU: `world` emulated ranks = `world` receive buffers + `world` launches of bbb_mc_exchange on
`world` streams, which really wait for each other's flags.  The real multi-process NCCL/IPC test is at the bottom
(needs >= 2 GPUs)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests.util import CFG_PRIORS, load_params_into, scale_err

pytestmark = pytest.mark.gpu
MC_NS = 1 << 63


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _exchange(dev, logits_per_rank, S_total, labels=None, moments=True, normalized=False, train_size=1.0, beta=0.0,
              kl=None):
    """Run bbb_mc_exchange for len(logits_per_rank) emulated ranks on one device; returns the outputs of every rank."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    lib = L.lib()
    world = len(logits_per_rank)
    B, Cc = next(l for l in logits_per_rank if l is not None).shape[1:]
    flags = (L.MC_MOMENTS if moments else 0) | (L.MC_NORMALIZED if normalized else 0)
    nbytes = int(lib.bbb_mc_buffer_bytes(B, Cc, flags, world))
    bufs = [torch.zeros(nbytes, dtype=torch.uint8, device=dev) for _ in range(world)]
    peers = (C.c_void_p * world)(*[b.data_ptr() for b in bufs])
    states = [torch.zeros(int(lib.bbb_mc_state_bytes()), dtype=torch.uint8, device=dev) for _ in range(world)]
    outs = []
    streams = [torch.cuda.Stream(device=dev) for _ in range(world)]
    klt = torch.tensor(float(kl if kl is not None else 0.0), device=dev)
    lab = labels.to(dev) if labels is not None else None
    torch.cuda.synchronize()
    for rep in range(2):                                    # twice: the second call exercises slot/sequence reuse
        outs = []
        for r in range(world):
            lg = logits_per_rank[r]
            f32 = dict(dtype=torch.float32, device=dev)
            o = {"lo": torch.empty(B, Cc, **f32), "kl": torch.empty((), **f32), "pred": torch.empty(B, Cc, **f32),
                 "epi": torch.empty(B, Cc, **f32), "ale": torch.empty(B, Cc, **f32), "ent": torch.empty(B, **f32),
                 "head": torch.full((4,), float("nan"), **f32)}
            with torch.cuda.stream(streams[r]):
                rc = lib.bbb_mc_exchange(
                    Fn._ptr(lg), 0 if lg is None else lg.shape[0], S_total, B, Cc, Fn._ptr(klt), 1, flags, Fn._ptr(lab),
                    C.c_float(train_size), C.c_float(beta), r, world, peers, Fn._ptr(states[r]), Fn._ptr(o["lo"]),
                    Fn._ptr(o["kl"]), *(Fn._ptr(o[k]) if moments else None for k in ("pred", "epi", "ale", "ent")),
                    Fn._ptr(o["head"]) if lab is not None else None, None, 0, Fn._stream(dev))
                L.check(rc, "bbb_mc_exchange")
            outs.append(o)
        torch.cuda.synchronize()
    for st in states:
        assert int(st[8:12].view(torch.int32).item()) == 0, "an exchange wait timed out"
    return outs


def test_mc_exchange_matches_oracle_single_and_emulated_ranks(dev):
    from oracle import bbb_oracle as O
    g = torch.Generator().manual_seed(2)
    for (S, B, Cc, world) in [(1, 5, 10, 1), (7, 33, 10, 3), (25, 64, 100, 8), (3, 700, 10, 4), (2, 9, 10, 4)]:
        base_logits = torch.randn(S, B, Cc, generator=g) * 4
        labels = torch.randint(0, Cc, (B,), generator=g)
        kl = 1234.5
        for normalized in (False, True):
            logits = base_logits.clone()
            if not normalized:        # classes whose softmax underflows fp32 in EVERY sample: logmeanexp must stay finite
                logits[:, 0, :] = torch.tensor([-200.0] * (Cc - 1) + [0.0])
            per_rank = []
            for r in range(world):
                ids = list(range(r, S, world))
                per_rank.append(logits[ids].contiguous().to(dev) if ids else None)
            outs = _exchange(dev, per_rank, S, labels, True, normalized, train_size=50000.0, beta=0.1, kl=kl)
            pred, epi, ale, ent = O.uncertainty(list(logits), normalized=normalized)
            if normalized:
                pr = torch.nn.functional.softplus(logits.double())
                lp = torch.log(pr / pr.sum(2, keepdim=True))
                ref = O.logmeanexp(lp.permute(1, 2, 0), 2)
            else:
                ref = O.mc_combine(list(logits)).double()
            for o in outs:
                assert torch.isfinite(o["lo"]).all()
                assert (o["lo"].double().cpu() - ref).abs().max() < 2e-5 * max(1.0, float(ref.abs().max())), (S, B, Cc, world)
                assert abs(float(o["kl"]) - kl) < 1e-3                       # sum_j kl_j / S == kl (main_bayesian.py:51)
                assert (o["pred"].double().cpu() - pred).abs().max() < 2e-6 * max(1.0, float(pred.abs().max())) * S
                assert (o["epi"].double().cpu() - epi).abs().max() < 2e-6
                assert (o["ale"].double().cpu() - ale).abs().max() < 2e-6
                assert (o["ent"].double().cpu() - ent).abs().max() < 1e-5
                nll = torch.nn.functional.nll_loss(ref.float(), labels)      # metrics.py:12-14
                acc = float((ref.argmax(1) == labels).float().mean())       # metrics.py:23-24
                head = o["head"].cpu()
                assert abs(float(head[1]) - float(nll)) < 1e-4 * max(1.0, abs(float(nll)))
                assert abs(float(head[0]) - (float(nll) * 50000.0 + 0.1 * kl)) < 1e-4 * abs(float(nll) * 50000.0 + 0.1 * kl)
                assert abs(float(head[2]) - acc) < 1e-6 and abs(float(head[3]) - 0.1 * kl) < 1e-3
            for o in outs[1:]:                                               # fixed rank order: bitwise identical on every rank
                assert torch.equal(o["lo"], outs[0]["lo"]) and torch.equal(o["epi"], outs[0]["epi"])


def _net(key, classes, inputs, variant, dev, math):
    from pytorch_bayesiancnn_b200 import models as M
    from oracle import bbb_oracle as O
    cls = {"alexnet": M.BBBAlexNet, "lenet": M.BBBLeNet, "3conv3fc": M.BBB3Conv3FC}[key]
    params = O.init_params(key, classes, inputs, CFG_PRIORS, seed=123)
    net = load_params_into(cls(classes, inputs, CFG_PRIORS, variant, "softplus"), params).to(dev).train()
    net.set_flag("math", math)
    return net, params


def _engine_eps(bbb, key, classes, inputs, variant, batch, seed, stream0, dev):
    """The eps tensors the engine's kernels draw for one net(x) whose first layer call uses Philox stream `stream0`
    (layer l uses stream0 + l), in the reference's draw order and layout -- for the oracle."""
    from oracle import bbb_oracle as O
    shapes = O.eps_shapes(key, classes, inputs, variant, batch)
    eps, layer = [], 0
    it = iter(shapes)
    for shp in it:
        if variant == "lrt":
            z = bbb.philox_normal(int(np.prod(shp)), seed, stream0 + layer, 0, device=dev)
            if len(shp) == 4:                                            # NHWC-flat element index (include/bbb_b200.h)
                Bn, Cn, H, W = shp
                z = z.view(Bn, H, W, Cn).permute(0, 3, 1, 2).contiguous()
            eps.append(z.view(shp).cpu())
        else:
            nw = int(np.prod(shp))
            bshape = next(it)
            eps.append(bbb.philox_normal(nw, seed, stream0 + layer, 0, device=dev).view(shp).cpu())
            eps.append(bbb.philox_normal(bshape[0], seed, stream0 + layer, nw, device=dev).cpu())
        layer += 1
    return eps


def test_c2_lenet_b256_bbb(dev):
    """BASELINE configs[1] (C2): BBBLeNet, CIFAR-10 shape, batch 256, 1 MC sample, bbb variant -- in-kernel Philox,
    exact-arithmetic kernels at the 1e-3 fp32 bar (measured ~1e-6) and the default 'auto' path at the 1e-2 bar."""
    import pytorch_bayesiancnn_b200 as bbb
    from oracle import bbb_oracle as O
    x = torch.rand(256, 3, 32, 32, generator=torch.Generator().manual_seed(3))      # ToTensor()-like inputs in [0,1]
    for math, tol in (("fp32", 1e-4), ("auto", 1e-2)):
        net, params = _net("lenet", 10, 3, "bbb", dev, math)
        bbb.manual_seed(77, 1000)
        with torch.no_grad():
            logits, kl = net(x.to(dev))
        eps = _engine_eps(bbb, "lenet", 10, 3, "bbb", 256, 77, 1000, dev)
        ref, refkl = O.net_forward("lenet", params, x, eps, "bbb", "softplus", 0.0, 0.1, 10)
        e = scale_err(logits, ref)
        print("C2 lenet bbb B=256", math, "scale err", e)
        assert e < tol, (math, e)
        assert abs(float(kl) - float(refkl)) <= 1e-5 * abs(float(refkl))


def _sharded_engine_logits(bbb, net, x, num_ens, world, seed):
    """What MCForward does on each rank, for all emulated ranks of one process: rank r runs samples r, r+world, ..."""
    from pytorch_bayesiancnn_b200 import functional as Fn, mc
    per_rank, kl = [], None
    for r in range(world):
        outs = []
        for j in mc.local_samples(num_ens, world, r):
            with Fn.mc_sample(j, seed), torch.no_grad():
                lg, kl = net(x)
            outs.append(lg.clone())
        per_rank.append(torch.stack(outs) if outs else None)
    return per_rank, kl


def test_c4_alexnet100_b1024_s25_over_8_ranks(dev):
    """BASELINE configs[3] (C4): BBBAlexNet CIFAR-100, batch 1024, 25 MC samples sharded 4,3,3,3,3,3,3,3 over 8 ranks,
    lrt, fused tensor-core chain + the NVLink-exchange kernel (8 emulated ranks on this GPU) vs the oracle's
    main_bayesian.py:46-53 on the same noise."""
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import mc
    from oracle import bbb_oracle as O
    B, S, world, seed = 1024, 25, 8, 4242
    assert [len(mc.local_samples(S, world, r)) for r in range(world)] == [4, 3, 3, 3, 3, 3, 3, 3]
    net, params = _net("alexnet", 100, 3, "lrt", dev, "auto")
    x = torch.randn(B, 3, 32, 32, generator=torch.Generator().manual_seed(5))
    xd = x.to(dev)
    per_rank, kl = _sharded_engine_logits(bbb, net, xd, S, world, seed)
    assert net._fused_plans[(B, 3, 32, 32)] is not None
    labels = torch.randint(0, 100, (B,), generator=torch.Generator().manual_seed(6))
    outs = _exchange(dev, per_rank, S, labels, moments=False, train_size=50000.0, beta=0.1, kl=float(kl))
    ref_logits = []
    for j in range(S):
        eps = _engine_eps(bbb, "alexnet", 100, 3, "lrt", B, seed, MC_NS | (j << 40), dev)
        lg, refkl = O.net_forward("alexnet", params, x, eps, "lrt", "softplus", 0.0, 0.1, 100)
        ref_logits.append(lg)
        got = per_rank[j % world][j // world]
        e = scale_err(got, lg)
        assert e < 1e-2, (j, e)                                           # bf16 chain bar, every one of the 25 samples
    ref = O.mc_combine(ref_logits)
    lo = outs[0]["lo"].cpu()
    err = float((lo - ref).abs().max())
    print("C4 log_outputs max abs err", err, "of scale", float(ref.abs().max()))
    assert err < 1e-2 * float(ref.abs().max())
    assert abs(float(outs[0]["kl"]) - float(refkl)) <= 1e-5 * abs(float(refkl))
    nll = float(torch.nn.functional.nll_loss(ref, labels))
    assert abs(float(outs[0]["head"][1]) - nll) < 2e-2 * abs(nll)
    # sharding does not change the result: one rank with all 25 samples
    one, _ = _sharded_engine_logits(bbb, net, xd, S, 1, seed)
    o1 = _exchange(dev, one, S, labels, moments=False, kl=float(kl))
    assert (o1[0]["lo"] - outs[0]["lo"]).abs().max() < 1e-4


def test_c5_3conv3fc_b2048_uncertainty(dev):
    """BASELINE configs[4] (C5): BBB3Conv3FC, 1x32x32 (SURVEY D2), batch 2048, lrt; pred / epistemic / aleatoric
    (uncertainty_estimation.py:70-96; + H[p_bar], SURVEY D3).  Oracle parity on identical noise with 2 samples at the
    full batch; the 100-sample run sharded 13,13,13,13,12,12,12,12 over 8 emulated ranks equals the unsharded one."""
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import mc
    from oracle import bbb_oracle as O
    B, seed = 2048, 99
    net, params = _net("3conv3fc", 10, 1, "lrt", dev, "auto")
    x = torch.rand(B, 1, 32, 32, generator=torch.Generator().manual_seed(8))
    xd = x.to(dev)
    per_rank, kl = _sharded_engine_logits(bbb, net, xd, 2, 2, seed)
    ref_logits = []
    for j in range(2):
        eps = _engine_eps(bbb, "3conv3fc", 10, 1, "lrt", B, seed, MC_NS | (j << 40), dev)
        lg, refkl = O.net_forward("3conv3fc", params, x, eps, "lrt", "softplus", 0.0, 0.1, 10)
        ref_logits.append(lg)
        e = scale_err(per_rank[j][0], lg)
        print("C5 sample", j, "scale err", e)
        assert e < 1e-2, (j, e)
    for normalized in (False, True):
        o = _exchange(dev, per_rank, 2, None, True, normalized, kl=float(kl))[0]
        pred, epi, ale, ent = O.uncertainty(ref_logits, normalized=normalized)
        sc = float(pred.abs().max())
        assert (o["pred"].double().cpu() - pred).abs().max() < 1e-2 * sc
        assert (o["epi"].double().cpu() - epi).abs().max() < 1e-2 and (o["ale"].double().cpu() - ale).abs().max() < 1e-2
        assert (o["ent"].double().cpu() - ent).abs().max() < 2e-2
    assert abs(float(o["kl"]) - float(refkl)) <= 1e-5 * abs(float(refkl))
    S = 100
    assert [len(mc.local_samples(S, 8, r)) for r in range(8)] == [13, 13, 13, 13, 12, 12, 12, 12]
    sh, kl = _sharded_engine_logits(bbb, net, xd, S, 8, seed)
    un = [torch.cat([sh[j % 8][j // 8][None] for j in range(S)])]                 # the same samples on one rank
    a = _exchange(dev, sh, S, None, True, False, kl=float(kl))[0]
    b = _exchange(dev, un, S, None, True, False, kl=float(kl))[0]
    for k in ("lo", "pred", "epi", "ale", "ent"):
        assert (a[k] - b[k]).abs().max() < 1e-4, k
    assert (a["epi"] >= -1e-6).all() and (a["ale"] >= -1e-6).all() and torch.isfinite(a["ent"]).all()


def test_mc_forward_product_path_single_gpu(dev):
    """mc.mc_forward(net, x, S) on the engine (captured graph, world 1): equals the per-sample engine runs combined
    by the oracle; replays draw fresh noise; the training noise counter is untouched."""
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import functional as Fn, mc
    from oracle import bbb_oracle as O
    net, _ = _net("alexnet", 10, 3, "lrt", dev, "auto")
    x = torch.randn(96, 3, 32, 32, device=dev)
    labels = torch.randint(0, 10, (96,), device=dev)
    bbb.manual_seed(5, 17)
    eng = mc.MCForward(net, x, 4, want_uncertainty=True, with_labels=True, train_size=100.0, beta=0.5, seed=31)
    assert Fn._noise.counter == 17 and Fn._noise.seed == 5                  # MC evaluation left the training stream alone
    out = eng(x, labels)
    torch.cuda.synchronize()
    first = {k: v.clone() for k, v in out.items()}
    out = eng(x, labels)
    torch.cuda.synchronize()
    assert not torch.equal(first["log_outputs"], out["log_outputs"])        # fresh noise per replay
    assert torch.equal(first["kl"], out["kl"])
    # replay r draws streams base_r + sample namespace: reproduce replay 1 (the second) sample by sample, eagerly
    from pytorch_bayesiancnn_b200.graph import _STRIDE
    logits = []
    base = torch.full((1,), _STRIDE, dtype=torch.int64, device=dev)         # replay 0 ran at base 0, replay 1 at base 2^20 (moved by the head kernel of each replay)
    for j in range(4):
        with Fn.stream_base(base), Fn.mc_sample(j, 31), torch.no_grad():
            lg, kl = net(x)
        logits.append(lg.cpu())
    ref = O.mc_combine(logits)
    assert (out["log_outputs"].cpu() - ref).abs().max() < 1e-4
    assert abs(float(out["kl"]) - float(kl)) <= 1e-6 * abs(float(kl))
    nll = float(torch.nn.functional.nll_loss(ref, labels.cpu()))
    assert abs(float(out["head"][0]) - (nll * 100.0 + 0.5 * float(kl))) < 1e-3 * abs(nll * 100.0 + 0.5 * float(kl))
    assert eng.timeouts() == 0 and eng.kernels_per_step is not None


def test_mc_forward_overlapped_exchange_equals_serial(dev):
    """overlap=True (exchange kernel of step t on its own stream beside the chain of step t+1; logits / KL terms / labels
    double buffered) gives bit-identical results to the serial step, step for step, with no synchronisation between steps."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("alexnet", 10, 3, "lrt", dev, "auto")
    x = torch.randn(128, 3, 32, 32, device=dev)
    labs = [torch.randint(0, 10, (128,), device=dev) for _ in range(5)]
    a = mc.MCForward(net, x, 3, want_uncertainty=True, with_labels=True, train_size=10.0, beta=0.2, seed=3)
    b = mc.MCForward(net, x, 3, want_uncertainty=True, with_labels=True, train_size=10.0, beta=0.2, seed=3, overlap=True)
    # inflight=2: even / odd steps on two streams with their own layer workspaces and Philox counters
    c = mc.MCForward(net, x, 3, want_uncertainty=True, with_labels=True, train_size=10.0, beta=0.2, seed=3, overlap=True, inflight=2)
    d = mc.MCForward(net, x, 3, want_uncertainty=True, with_labels=True, train_size=10.0, beta=0.2, seed=3, overlap=True, inflight=3)
    assert b.overlap and b.result_stream is not None and c.inflight == 2 and d.inflight == 3
    for n in (1, 2, 5):                                                      # compare after 1, 3 and 8 steps in total
        for i in range(n):
            oa = a(x, labs[i])
        ra = {k: v.clone() for k, v in oa.items()}
        for eng in (b, c, d):
            for i in range(n):
                ob = eng(x, labs[i])
            eng.wait()
            rb = {k: v.clone() for k, v in ob.items()}
            torch.cuda.synchronize()
            for k in ra:
                assert torch.equal(ra[k], rb[k]), (n, k, eng.inflight)
    assert b.timeouts() == 0 and c.timeouts() == 0 and d.timeouts() == 0


def test_mc_sample_folding_equals_sample_loop(dev):
    """LRT: S local samples folded into ONE pass of the fused chain (each row drawing from its own sample's Philox
    stream) == S passes, one per sample -- same logits, same combine (what makes C3/C4-style steps 2x faster)."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("alexnet", 10, 3, "lrt", dev, "auto")
    x = torch.randn(200, 3, 32, 32, device=dev)                              # not a multiple of the 128-row tile: samples share tiles
    a = mc.MCForward(net, x, 5, want_uncertainty=True, seed=11, fold=True)
    b = mc.MCForward(net, x, 5, want_uncertainty=True, seed=11, fold=False)
    assert a.fold_steps is not None and b.fold_steps is None
    oa, ob = a(x), b(x)
    torch.cuda.synchronize()
    assert (a.logits - b.logits).abs().max() <= 1e-6 * b.logits.abs().max()
    for k in ("log_outputs", "kl", "pred", "epistemic", "aleatoric", "entropy"):
        assert (oa[k] - ob[k]).abs().max() <= 1e-5 * max(1.0, float(ob[k].abs().max())), k
    assert a.kernels_per_step < b.kernels_per_step


def _oracle_train_grads(key, params, x, labels, eps_per_sample, variant, classes, train_size, beta, dtype=torch.float32):
    """main_bayesian.py:46-58 through torch autograd on the oracle, in `dtype` on the device of the tensors given:
    grads of every parameter."""
    from oracle import bbb_oracle as O
    P = [{k: v.to(dtype).clone().requires_grad_(True) for k, v in p.items()} for p in params]
    x = x.to(dtype)
    outs, kl = [], 0.0
    for eps in eps_per_sample:
        lg, _kl = O.net_forward(key, P, x, [e.to(dtype) for e in eps], variant, "softplus", 0.0, 0.1, classes)
        outs.append(lg)
        kl = kl + _kl
    kl = kl / len(eps_per_sample)
    log_outputs = O.mc_combine(outs)
    loss = torch.nn.functional.nll_loss(log_outputs, labels, reduction="mean") * train_size + beta * kl    # metrics.py:12-14
    loss.backward()
    return loss.detach(), [p[k].grad for p in P for k in ("W_mu", "W_rho", "bias_mu", "bias_rho")]


def test_training_step_matches_oracle_autograd(dev):
    """Row f1: the sharded training step (one rank here) == main_bayesian.train_model's math on identical noise:
    loss, and the gradient of every W_mu / W_rho / bias_mu / bias_rho, for 3 MC samples, both variants."""
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import mc
    for variant in ("lrt", "bbb"):
        net, params = _net("lenet", 10, 3, variant, dev, "fp32")
        x = torch.rand(48, 3, 32, 32, generator=torch.Generator().manual_seed(4))
        labels = torch.randint(0, 10, (48,), generator=torch.Generator().manual_seed(5))
        step = mc.MCTrainStep(net, x.to(dev), 3, train_size=5000.0, seed=21)
        out = step(x.to(dev), labels.to(dev), beta=0.1)
        eps = [_engine_eps(bbb, "lenet", 10, 3, variant, 48, 21, MC_NS | (j << 40), dev) for j in range(3)]
        ref_loss, ref_grads = _oracle_train_grads("lenet", params, x, labels, eps, variant, 10, 5000.0, 0.1)
        assert abs(float(out["head"][0]) - float(ref_loss)) <= 1e-4 * abs(float(ref_loss)), (variant, float(out["head"][0]), float(ref_loss))
        got = [g for m in net.children() if hasattr(m, "W_mu") for g in (m.W_mu.grad, m.W_rho.grad, m.bias_mu.grad, m.bias_rho.grad)]
        assert len(got) == len(ref_grads)
        for i, (a, b) in enumerate(zip(got, ref_grads)):
            e = scale_err(a, b)
            assert e < 2e-4, (variant, i, e)


# --------------------------------------------------------------------------- #
# real multi-process run: NCCL for the handshake, CUDA-IPC peer buffers for the exchange
# --------------------------------------------------------------------------- #
def _mp_worker(rank, world, port, num_ens, out_path):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("alexnet", 10, 3, "lrt", dev, "auto")
    x = torch.randn(256, 3, 32, 32, generator=torch.Generator().manual_seed(1)).to(dev)
    labels = torch.randint(0, 10, (256,), generator=torch.Generator().manual_seed(2)).to(dev)
    eng = mc.MCForward(net, x, num_ens, want_uncertainty=True, with_labels=True, train_size=50000.0, beta=0.1, seed=77)
    for _ in range(3):
        out = eng(x, labels)
    torch.cuda.synchronize()
    assert eng.timeouts() == 0
    res = {k: v.cpu() for k, v in out.items()}
    eng.close()
    # the same three steps with the exchange of step t overlapped with the chain of step t+1 (double-buffered samples)
    eng2 = mc.MCForward(net, x, num_ens, want_uncertainty=True, with_labels=True, train_size=50000.0, beta=0.1, seed=77, overlap=True)
    other = torch.randint(0, 10, (256,), generator=torch.Generator().manual_seed(5)).to(dev)
    for i in range(3):
        o2 = eng2(x, labels if i == 2 else other)                   # back to back, no synchronisation in between
    eng2.wait()
    torch.cuda.synchronize()
    for k, v in res.items():
        assert torch.equal(o2[k].cpu(), v), k
    for _ in range(40):
        eng2(x, labels)
    torch.cuda.synchronize()
    assert eng2.timeouts() == 0
    eng2.close()
    eng3 = mc.MCForward(net, x, num_ens, want_uncertainty=True, with_labels=True, train_size=50000.0, beta=0.1, seed=77, overlap=True,
                        inflight=2)
    for i in range(3):
        o3 = eng3(x, labels if i == 2 else other)
    eng3.wait()
    torch.cuda.synchronize()
    for k, v in res.items():
        assert torch.equal(o3[k].cpu(), v), ("inflight2", k)
    for _ in range(40):
        eng3(x, labels)
    torch.cuda.synchronize()
    assert eng3.timeouts() == 0
    eng3.close()
    # sharded training step (row f1): gradients after ONE all-reduce
    tnet, _ = _net("lenet", 10, 3, "lrt", dev, "fp32")
    xt = torch.rand(64, 3, 32, 32, generator=torch.Generator().manual_seed(3)).to(dev)
    yt = torch.randint(0, 10, (64,), generator=torch.Generator().manual_seed(4)).to(dev)
    ts = mc.MCTrainStep(tnet, xt, 4, train_size=1000.0, seed=9)
    tout = ts(xt, yt, beta=0.1)
    torch.cuda.synchronize()
    res["train_loss"] = tout["head"].cpu()
    res["train_grads"] = [p.grad.cpu() for p in tnet.parameters()]
    ts.close()
    torch.save(res, out_path + f".{rank}")
    dist.destroy_process_group()


@pytest.mark.parametrize("num_ens", [5])
def test_mc_forward_multi_gpu_equals_single_gpu(dev, num_ens):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import socket
    import tempfile
    import torch.multiprocessing as mp
    from pytorch_bayesiancnn_b200 import mc
    world = 2
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out_path = os.path.join(tempfile.mkdtemp(), "mc")
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_mp_worker, args=(r, world, port, num_ens, out_path)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0
    outs = [torch.load(out_path + f".{r}") for r in range(world)]
    for k in outs[0]:
        if k == "train_grads":
            assert all(torch.equal(a, b) for a, b in zip(outs[0][k], outs[1][k]))
        else:
            assert torch.equal(outs[0][k], outs[1][k]), k                  # every rank holds the same result
    # single GPU, same global sample seeds, same replay index (the third)
    net, _ = _net("alexnet", 10, 3, "lrt", dev, "auto")
    x = torch.randn(256, 3, 32, 32, generator=torch.Generator().manual_seed(1)).to(dev)
    labels = torch.randint(0, 10, (256,), generator=torch.Generator().manual_seed(2)).to(dev)
    eng = mc.MCForward(net, x, num_ens, want_uncertainty=True, with_labels=True, train_size=50000.0, beta=0.1, seed=77)
    for _ in range(3):
        one = eng(x, labels)
    torch.cuda.synchronize()
    for k in ("log_outputs", "pred", "epistemic", "aleatoric", "entropy", "kl", "head"):
        a, b = one[k].cpu(), outs[0][k]
        assert (a - b).abs().max() <= 1e-4 * max(1.0, float(b.abs().max())), k
    # the sharded training step: 2 ranks x 2 samples == 1 rank x 4 samples (same global sample streams)
    tnet, _ = _net("lenet", 10, 3, "lrt", dev, "fp32")
    xt = torch.rand(64, 3, 32, 32, generator=torch.Generator().manual_seed(3)).to(dev)
    yt = torch.randint(0, 10, (64,), generator=torch.Generator().manual_seed(4)).to(dev)
    ts = mc.MCTrainStep(tnet, xt, 4, train_size=1000.0, seed=9)
    tout = ts(xt, yt, beta=0.1)
    torch.cuda.synchronize()
    assert (tout["head"].cpu() - outs[0]["train_loss"]).abs().max() <= 1e-4 * float(outs[0]["train_loss"].abs().max())
    for p, gref in zip(tnet.parameters(), outs[0]["train_grads"]):
        assert scale_err(p.grad, gref) < 1e-4

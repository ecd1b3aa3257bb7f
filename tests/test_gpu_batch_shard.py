"""Row-block sharding of the Monte-Carlo step on the GPU: the first image moves the LRT noise so that a block computes
what the whole batch computes at its rows (every forward path and the backward), the row-block exchange kernel on
emulated ranks, and the training step's gradients over row blocks."""
import ctypes as C
import os

import pytest
import torch

from tests.util import CFG_PRIORS, load_params_into, scale_err

pytestmark = pytest.mark.gpu
SEED = 4242


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _net(key, variant, dev, math, classes=10):
    from pytorch_bayesiancnn_b200 import models as M
    from oracle import bbb_oracle as O
    cls = {"alexnet": M.BBBAlexNet, "lenet": M.BBBLeNet, "3conv3fc": M.BBB3Conv3FC}[key]
    params = O.init_params(key, classes, 3, CFG_PRIORS, seed=123)
    net = load_params_into(cls(classes, 3, CFG_PRIORS, variant, "softplus"), params).to(dev).train()
    net.set_flag("math", math)
    return net


BLOCKS = [(0, 130), (130, 261), (261, 300)]          # b0 not a multiple of 128, a ragged last block


# --------------------------------------------------------------------------- #
# (1) noise offset: net(x[b0:b1]) under first_image(b0) == net(x)[b0:b1], bit for bit
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("key,math", [("lenet", "fp32"), ("lenet", "bf16"), ("lenet", "tf32"), ("3conv3fc", "auto"),
                                      ("alexnet", "auto"), ("alexnet", "fp32")])
@pytest.mark.parametrize("variant", ["lrt", "bbb"])
def test_block_forward_equals_full_batch_rows(dev, key, math, variant):
    from pytorch_bayesiancnn_b200 import functional as Fn
    net = _net(key, variant, dev, math)
    x = torch.rand(300, 3, 32, 32, generator=torch.Generator().manual_seed(1)).to(dev)
    with torch.no_grad(), Fn.mc_sample(3, SEED):
        full, kl = net(x)
    if key == "alexnet" and math == "auto":
        assert net._fused_plans.get(tuple(x.shape)) is not None, "the fused chain (stride-4 first layer) did not run"
    for b0, b1 in BLOCKS:
        with torch.no_grad(), Fn.mc_sample(3, SEED), Fn.first_image(b0):
            part, klp = net(x[b0:b1])
        assert torch.equal(part, full[b0:b1]), (key, math, variant, b0)
        assert float(klp) == float(kl)
    if variant == "lrt":                                 # the offset matters: without it the block draws other noise
        with torch.no_grad(), Fn.mc_sample(3, SEED):
            part, _ = net(x[130:261])
        assert not torch.equal(part, full[130:261])


@pytest.mark.parametrize("variant", ["lrt", "bbb"])
def test_fused_fold_with_first_image(dev, variant):
    """The fused chain folding S samples of a row block (stride-4 first layer included) == the full batch per sample."""
    from pytorch_bayesiancnn_b200 import functional as Fn, fused
    net = _net("alexnet", variant, dev, "auto")
    x = torch.rand(300, 3, 32, 32, generator=torch.Generator().manual_seed(2)).to(dev)
    S, b0, nb = 3, 172, 128                              # BBB folds need 128 rows per sample; b0 % 128 != 0
    fold = (nb, 1 << 40)
    with Fn.first_image(b0):
        steps = fused.plan(list(net.children()), (S * nb, 3, 32, 32), fold)
    assert steps is not None
    with torch.no_grad(), Fn.mc_sample(5, SEED), Fn.first_image(b0):
        out, _ = fused._run(steps, x[b0:b0 + nb], True, None, False, None, fold=fold)
    for s in range(S):
        with torch.no_grad(), Fn.mc_sample(5 + s, SEED):
            ref, _ = net(x)
        got, want = out[s * nb:(s + 1) * nb], ref[b0:b0 + nb]
        assert (got - want).abs().max() <= 1e-6 * want.abs().max(), (variant, s)


@pytest.mark.parametrize("variant", ["lrt", "bbb"])
def test_layer_fold_with_first_image(dev, variant):
    """The per-layer fold (BBBLeNet on the tensor-core layer kernels) of a row block == the full batch per sample."""
    from pytorch_bayesiancnn_b200 import functional as Fn
    net = _net("lenet", variant, dev, "bf16")
    net.set_flag("fuse", False)
    x = torch.rand(300, 3, 32, 32, generator=torch.Generator().manual_seed(3)).to(dev)
    S = 3
    b0, nb = (128, 128) if variant == "bbb" else (131, 97)
    xr = x[b0:b0 + nb].repeat(S, 1, 1, 1)
    with torch.no_grad(), Fn.mc_sample(2, SEED), Fn.layer_fold(nb, 1 << 40), Fn.first_image(b0):
        out, _ = net(xr)
    for s in range(S):
        with torch.no_grad(), Fn.mc_sample(2 + s, SEED):
            ref, _ = net(x)
        assert torch.equal(out[s * nb:(s + 1) * nb], ref[b0:b0 + nb]), (variant, s)


# --------------------------------------------------------------------------- #
# (2) the row-block exchange on emulated ranks (one stream per rank)
# --------------------------------------------------------------------------- #
def _exchange(dev, logits, world, rb, labels, flags, kl=321.5, train_size=1000.0, beta=0.1):
    """bbb_mc_exchange_sharded for `world` emulated ranks, batch_shards = rb (1: the default kernel); logits [S, B, C]
    of all samples, rank (g, k) gets those of its samples and rows.  Runs twice (slot / sequence reuse)."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn, mc
    lib = L.lib()
    S, B, Cc = logits.shape
    rs = world // rb
    nbytes = int(lib.bbb_mc_buffer_bytes(B, Cc, flags, rs))
    bufs = [torch.zeros(nbytes, dtype=torch.uint8, device=dev) for _ in range(world)]
    peers = (C.c_void_p * world)(*[b.data_ptr() for b in bufs])
    states = [torch.zeros(int(lib.bbb_mc_state_bytes()), dtype=torch.uint8, device=dev) for _ in range(world)]
    streams = [torch.cuda.Stream(device=dev) for _ in range(world)]
    klt = torch.tensor(kl, device=dev)
    lab = labels.to(dev)
    mine = []
    for r in range(world):
        _, g, k = mc.shard_layout(world, r, rb)
        b0, b1 = mc.row_block(B, rb, k)
        ids = mc.local_samples(S, rs, g)
        mine.append(logits[ids][:, b0:b1].contiguous().to(dev) if ids else None)
    info = bool(flags & L.MC_INFO)
    torch.cuda.synchronize()
    for rep in range(2):
        outs = []
        for r in range(world):
            f32 = dict(dtype=torch.float32, device=dev)
            o = {k_: torch.empty(B, Cc, **f32) for k_ in ("lo", "pred", "epi", "ale")}
            o.update(kl=torch.empty((), **f32), ent=torch.empty(B, **f32), head=torch.empty(4, **f32),
                     ee=torch.empty(B, **f32), mi=torch.empty(B, **f32))
            lg = mine[r]
            with torch.cuda.stream(streams[r]):
                rc = lib.bbb_mc_exchange_sharded(
                    Fn._ptr(lg), 0 if lg is None else lg.shape[0], S, B, Cc, Fn._ptr(klt), 1, flags, Fn._ptr(lab),
                    C.c_float(train_size), C.c_float(beta), r, world, peers, Fn._ptr(states[r]), Fn._ptr(o["lo"]),
                    Fn._ptr(o["kl"]), Fn._ptr(o["pred"]), Fn._ptr(o["epi"]), Fn._ptr(o["ale"]), Fn._ptr(o["ent"]),
                    Fn._ptr(o["head"]), None, 0, Fn._ptr(o["ee"]) if info else None, Fn._ptr(o["mi"]) if info else None,
                    rb, Fn._stream(dev))
                L.check(rc, "bbb_mc_exchange_sharded")
            outs.append(o)
        torch.cuda.synchronize()
    for st in states:
        assert int(st[8:12].view(torch.int32).item()) == 0, "an exchange wait timed out"
    keys = ("lo", "pred", "epi", "ale", "kl", "ent", "head") + (("ee", "mi") if info else ())
    return [{k_: o[k_].cpu() for k_ in keys} for o in outs]


@pytest.mark.parametrize("world", [2, 4, 8])
def test_sharded_exchange_matches_oracle_and_the_sample_only_exchange(dev, world):
    from oracle import bbb_oracle as O
    from pytorch_bayesiancnn_b200 import _lib as L
    g = torch.Generator().manual_seed(world)
    B, Cc = 333, 10
    for S in (1, 5, 25):
        logits = torch.randn(S, B, Cc, generator=g) * 4
        logits[:, 0, :] = torch.tensor([-200.0] * (Cc - 1) + [0.0])      # every sample's softmax underflows there
        labels = torch.randint(0, Cc, (B,), generator=g)
        ref = O.mc_combine(list(logits)).double()
        pred, epi, ale, ent = O.uncertainty(list(logits))
        for flags in (L.MC_MOMENTS, L.MC_MOMENTS | L.MC_INFO):
            for rb in [d for d in range(2, world + 1) if world % d == 0]:
                outs = _exchange(dev, logits, world, rb, labels, flags)
                # the sample-only exchange on Rs ranks holding the same samples: bitwise the same numbers
                base = _exchange(dev, logits, world // rb, 1, labels, flags)[0]
                for o in outs:
                    for k_ in base:
                        assert torch.equal(o[k_], base[k_]), (world, rb, S, k_)
                o = outs[0]
                assert (o["lo"].double() - ref).abs().max() < 2e-5 * max(1.0, float(ref.abs().max()))
                assert abs(float(o["kl"]) - 321.5) < 1e-3
                assert (o["pred"].double() - pred).abs().max() < 2e-6 * max(1.0, float(pred.abs().max())) * S
                assert (o["epi"].double() - epi).abs().max() < 2e-6 and (o["ale"].double() - ale).abs().max() < 2e-6
                assert (o["ent"].double() - ent).abs().max() < 1e-5
                nll = torch.nn.functional.nll_loss(ref.float(), labels)
                assert abs(float(o["head"][1]) - float(nll)) < 1e-4 * max(1.0, abs(float(nll)))
                assert abs(float(o["head"][2]) - float((ref.argmax(1) == labels).float().mean())) < 1e-6


# --------------------------------------------------------------------------- #
# (3) training over emulated row blocks == the full-batch step
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("variant,math", [("lrt", "fp32"), ("bbb", "fp32"), ("lrt", "bf16"), ("bbb", "bf16")])
def test_training_over_row_blocks_equals_full_batch(dev, variant, math):
    """What MCTrainStep(batch_shards=Rb) computes on each rank, summed over the blocks (the all-reduce): the layer
    gradients of the full-batch step, and each block's input-gradient rows."""
    from pytorch_bayesiancnn_b200 import functional as Fn, mc
    B, S, train_size, beta = 300, 2, 5000.0, 0.1
    x = torch.rand(B, 3, 32, 32, generator=torch.Generator().manual_seed(4)).to(dev)
    labels = torch.randint(0, 10, (B,), generator=torch.Generator().manual_seed(5)).to(dev)
    net = _net("lenet", variant, dev, math)
    step = mc.MCTrainStep(net, x, S, train_size=train_size, seed=SEED)
    xf = x.clone().requires_grad_(True)
    out = step(xf, labels, beta=beta)
    full = [p.grad.clone() for p in step.params]
    lo = out["log_outputs"].clone()
    assert (step.sample_shards, step.batch_shards, step.rows) == (1, 1, (0, B))
    acc = [torch.zeros_like(p) for p in step.params]
    for k, (b0, b1) in enumerate(BLOCKS):
        for p in step.params:
            p.grad = None
        xb = x[b0:b1].clone().requires_grad_(True)
        logits, kls = [], []
        for j in range(S):
            with Fn.mc_sample(j, SEED), Fn.first_image(b0):
                lg, kl = net(xb)
            logits.append(lg)
            kls.append(kl)
        idx = labels[b0:b1].view(-1, 1)
        p_bar_y = lo[b0:b1].gather(1, idx).exp()
        grads = []
        for lg in logits:
            sm = torch.softmax(lg.detach().float(), dim=1)
            grads.append(-(train_size / B) * sm.gather(1, idx) / (S * p_bar_y) *
                         (torch.zeros_like(sm).scatter_(1, idx, 1.0) - sm))
        kl_t = kls if k == 0 else []
        torch.autograd.backward(logits + kl_t, grads + [torch.full_like(t, beta / S) for t in kl_t])
        for a, p in zip(acc, step.params):
            a += p.grad
        assert scale_err(xb.grad, xf.grad[b0:b1]) < 1e-4, (variant, math, k)
    for i, (a, b) in enumerate(zip(acc, full)):
        assert scale_err(a, b) < 1e-4, (variant, math, i, scale_err(a, b))


# --------------------------------------------------------------------------- #
# (4) two GPUs: MCForward / MCTrainStep with batch_shards=2 == one GPU
# --------------------------------------------------------------------------- #
def _mp_worker(rank, world, port, out_path):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from pytorch_bayesiancnn_b200 import mc
    net = _net("alexnet", "lrt", dev, "auto")
    x = torch.randn(301, 3, 32, 32, generator=torch.Generator().manual_seed(1)).to(dev)
    labels = torch.randint(0, 10, (301,), generator=torch.Generator().manual_seed(2)).to(dev)
    eng = mc.MCForward(net, x, 5, want_uncertainty=True, with_labels=True, train_size=50000.0, beta=0.1, seed=77,
                       batch_shards=2)
    for _ in range(3):
        out = eng(x, labels)
    torch.cuda.synchronize()
    res = {k: v.cpu() for k, v in out.items()}
    res["rows"], res["logits"], res["timeouts"] = eng.rows, eng.logits.cpu(), eng.timeouts()
    eng.close()
    tnet = _net("lenet", "lrt", dev, "fp32")
    xt = torch.rand(65, 3, 32, 32, generator=torch.Generator().manual_seed(3)).to(dev)
    yt = torch.randint(0, 10, (65,), generator=torch.Generator().manual_seed(4)).to(dev)
    ts = mc.MCTrainStep(tnet, xt, 1, train_size=1000.0, seed=9, batch_shards=2)
    tout = ts(xt, yt, beta=0.1)
    torch.cuda.synchronize()
    res["train_loss"] = tout["head"].cpu()
    res["train_grads"] = [p.grad.cpu() for p in tnet.parameters()]
    res["train_timeouts"] = ts.timeouts()
    ts.close()
    torch.save(res, out_path + f".{rank}")
    dist.destroy_process_group()


def test_batch_sharded_multi_gpu_equals_single_gpu(dev):
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
    procs = [ctx.Process(target=_mp_worker, args=(r, world, port, out_path)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0
    outs = [torch.load(out_path + f".{r}") for r in range(world)]
    assert all(o["timeouts"] == 0 and o["train_timeouts"] == 0 for o in outs)
    net = _net("alexnet", "lrt", dev, "auto")
    x = torch.randn(301, 3, 32, 32, generator=torch.Generator().manual_seed(1)).to(dev)
    labels = torch.randint(0, 10, (301,), generator=torch.Generator().manual_seed(2)).to(dev)
    eng = mc.MCForward(net, x, 5, want_uncertainty=True, with_labels=True, train_size=50000.0, beta=0.1, seed=77)
    for _ in range(3):
        one = eng(x, labels)
    torch.cuda.synchronize()
    for o in outs:
        b0, b1 = o["rows"]
        assert torch.equal(o["logits"], eng.logits[:, b0:b1].cpu())            # per-sample logits, bit for bit
        for k in ("log_outputs", "pred", "epistemic", "aleatoric", "entropy", "kl", "head"):
            a, b = one[k].cpu(), o[k]
            assert (a - b).abs().max() <= 1e-4 * max(1.0, float(b.abs().max())), k
    tnet = _net("lenet", "lrt", dev, "fp32")
    xt = torch.rand(65, 3, 32, 32, generator=torch.Generator().manual_seed(3)).to(dev)
    yt = torch.randint(0, 10, (65,), generator=torch.Generator().manual_seed(4)).to(dev)
    ts = mc.MCTrainStep(tnet, xt, 1, train_size=1000.0, seed=9)
    ts(xt, yt, beta=0.1)
    torch.cuda.synchronize()
    for p, gref in zip(tnet.parameters(), outs[0]["train_grads"]):
        assert scale_err(p.grad, gref) < 1e-4

"""The per-image score log on the GPU: bbb_mc_score_log against the entries formed from its own inputs (tests/ood_ref.py),
appends and overflow, MCForward(score_log=...) in every mode the engine runs, evaluate(score_log=...) and detect_ood
against the float64 ranking metrics, and the logs of two ranks."""
import math
import os

import numpy as np
import pytest
import torch

from tests import ood_ref as R
from tests.test_gpu_mc import _net

pytestmark = pytest.mark.gpu
PLANES = ("confidence", "entropy", "mutual_info", "expected_entropy", "epistemic", "correct")


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _bits(t):
    return t.contiguous().view(torch.int32)


def _inputs(B, Cc, dev, seed=0):
    """Exchange-like outputs with argmax ties, -inf log-probabilities and a row of -inf."""
    g = torch.Generator().manual_seed(seed)
    lo = torch.log_softmax(torch.randn(B, Cc, generator=g) * 3, dim=1)
    if Cc > 1:
        lo[0] = math.log(1.0 / Cc)                                   # every class tied
        if B > 1:
            lo[1, Cc // 2:] = -float("inf")                          # probabilities that are exactly 0
        if B > 2 and Cc > 2:
            lo[2, Cc - 1] = lo[2, 1] = lo[2].max() + 1.0             # tie of two maximal classes: the first wins
    if B > 3:
        lo[3] = -float("inf")                                        # no finite class: class 0
    return {"lo": lo.contiguous().to(dev), "ent": (torch.rand(B, generator=g) * 2).to(dev),
            "mi": (torch.randn(B, generator=g) * 1e-3).to(dev), "ee": torch.rand(B, generator=g).to(dev),
            "epi": (torch.rand(B, Cc, generator=g) * 1e-2).to(dev),
            "lab": torch.randint(0, Cc, (B,), generator=g).to(dev)}


def _launch(lib, inp, planes, pred, cap, cursor, nulls, dev):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    B, Cc = inp["lo"].shape
    opt = (lambda k: None) if nulls else (lambda k: Fn._ptr(inp[k]))
    L.check(lib.bbb_mc_score_log(Fn._ptr(inp["lo"]), opt("ent"), opt("ee"), opt("mi"), opt("epi"), opt("lab"), B, Cc,
                                 Fn._ptr(planes), Fn._ptr(pred), cap, Fn._ptr(cursor), Fn._stream(dev)), "score_log")


def _check_entries(planes, pred, inp, nulls, tag):
    """planes [6, B] / pred [B] of one launch against the entries formed from its inputs."""
    lo = inp["lo"]
    B, Cc = lo.shape
    ref_pred = lo.cpu().argmax(1)                                     # first maximal class (no NaN in the inputs)
    assert torch.equal(pred.cpu().long(), ref_pred), tag
    conf = torch.exp(lo.gather(1, ref_pred.to(lo.device)[:, None])[:, 0])     # expf on the device, as the kernel
    assert torch.equal(_bits(planes[0]), _bits(conf)), tag
    if nulls:
        assert torch.isnan(planes[1:]).all(), tag
        return
    for k, key in ((1, "ent"), (2, "mi"), (3, "ee")):
        assert torch.equal(_bits(planes[k]), _bits(inp[key])), (tag, PLANES[k])
    ref = inp["epi"].double().sum(1).cpu().numpy()
    got = planes[4].double().cpu().numpy()
    assert (np.abs(got - ref) <= np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)).all(), tag
    assert torch.equal(planes[5].cpu(), (ref_pred == inp["lab"].cpu()).float()), tag


@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("Cc", [1, 2, 10, 100])
@pytest.mark.parametrize("B", [1, 7, 512, 2048])
def test_score_log_kernel_matches_its_inputs(dev, B, Cc, nulls):
    from pytorch_bayesiancnn_b200 import _lib as L
    lib = L.lib()
    inp = _inputs(B, Cc, dev, seed=B + Cc)
    planes = torch.full((6, B), 7.0, device=dev)
    pred = torch.full((B,), -5, dtype=torch.int32, device=dev)
    cursor = torch.zeros(2, dtype=torch.int64, device=dev)
    _launch(lib, inp, planes, pred, B, cursor, nulls, dev)
    torch.cuda.synchronize()
    assert cursor.tolist() == [B, 0]
    _check_entries(planes, pred, inp, nulls, (B, Cc, nulls))


def test_score_log_appends_in_order_and_overflow_keeps_guards(dev):
    """Launches append one after another, eagerly and from a replayed graph; past the capacity nothing is written (the
    guard words behind the planes stay) and the images are counted in cursor[1]."""
    from pytorch_bayesiancnn_b200 import _lib as L
    lib = L.lib()
    Cc, sizes, cap, guard = 10, (300, 7, 512, 1, 400), 1000, 4096
    inps = [_inputs(b, Cc, dev, seed=i) for i, b in enumerate(sizes)]
    buf = torch.full((6 * cap + guard,), 7.0, device=dev)
    pbuf = torch.full((cap + guard,), -5, dtype=torch.int32, device=dev)
    cursor = torch.zeros(2, dtype=torch.int64, device=dev)
    for inp in inps:
        _launch(lib, inp, buf, pbuf, cap, cursor, False, dev)
    torch.cuda.synchronize()
    total = sum(sizes)
    assert cursor.tolist() == [total, total - cap]
    assert (buf[6 * cap:] == 7.0).all() and (pbuf[cap:] == -5).all()
    planes, off = buf[:6 * cap].view(6, cap), 0
    for i, inp in enumerate(inps):                       # whatever fits, entry by entry
        n = min(sizes[i], cap - off)
        if n <= 0:
            break
        part = {k: (v[:n] if v.dim() else v) for k, v in inp.items()}
        _check_entries(planes[:, off:off + n], pbuf[off:off + n], part, False, ("append", i))
        off += n
    # a captured graph of two launches, replayed three times: six appends in launch order
    cap2 = 6 * 300 + 3
    buf2 = torch.full((6 * cap2 + guard,), 7.0, device=dev)
    pbuf2 = torch.full((cap2 + guard,), -5, dtype=torch.int32, device=dev)
    cursor2 = torch.zeros(2, dtype=torch.int64, device=dev)
    a, b = _inputs(300, Cc, dev, seed=11), _inputs(300, Cc, dev, seed=12)
    s = torch.cuda.Stream(device=dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr, stream=s):
        _launch(lib, a, buf2, pbuf2, cap2, cursor2, False, dev)
        _launch(lib, b, buf2, pbuf2, cap2, cursor2, False, dev)
    torch.cuda.synchronize()
    assert cursor2.tolist() == [0, 0]                     # capture runs nothing
    for _ in range(3):
        gr.replay()
    torch.cuda.synchronize()
    assert cursor2.tolist() == [1800, 0] and (buf2[6 * cap2:] == 7.0).all() and (pbuf2[cap2:] == -5).all()
    planes2 = buf2[:6 * cap2].view(6, cap2)
    for k in range(6):
        _check_entries(planes2[:, 300 * k:300 * (k + 1)], pbuf2[300 * k:300 * (k + 1)], (a, b)[k % 2], False, ("graph", k))
    assert (planes2[:, 1800:] == 7.0).all()


# --------------------------------------------------------------------------- #
# MCForward(score_log=...)
# --------------------------------------------------------------------------- #
def _batches(n, B, inputs, dev, Cc=10, seed=5):
    g = torch.Generator().manual_seed(seed)
    return ([torch.randn(B, inputs, 32, 32, generator=g).to(dev) for _ in range(n)],
            [torch.randint(0, Cc, (B,), generator=g).to(dev) for _ in range(n)])


def _expected_log(dev, outs, labels, cap):
    """A log fed with the given per-step outputs (clones), as the engine's own launch would append them."""
    from pytorch_bayesiancnn_b200 import mc
    ref = mc.ScoreLog(dev, cap)
    for o, y in zip(outs, labels):
        ref.append(o["log_outputs"], o.get("entropy"), o.get("expected_entropy"), o.get("mutual_info"),
                   o.get("epistemic"), y)
    torch.cuda.synchronize()
    return ref.read()


def _same_log(got, ref, tag):
    assert set(got) == set(ref), tag
    for k in ref:
        assert torch.equal(got[k].view(torch.int32), ref[k].view(torch.int32)), (tag, k)


@pytest.mark.parametrize("key,inputs", [("alexnet", 3), ("lenet", 1)])
def test_mc_forward_score_log_every_mode(dev, key, inputs):
    """Serial graph (fused fold on AlexNet, per-layer fold on LeNet), the sample loop, graph=False, overlap and
    inflight=4: the log equals the per-step outputs appended in order, bit for bit; every output is that of the same
    engine without a log; warm-up steps are not logged; one more kernel per step."""
    from pytorch_bayesiancnn_b200 import EngineError, mc
    net, _ = _net(key, 10, inputs, "lrt", dev, "auto")
    steps, B, S = 5, 128, 3
    xs, ys = _batches(steps, B, inputs, dev)
    kw = dict(with_labels=True, seed=13, want_uncertainty=True, want_information=True, static_inputs=xs)
    with pytest.raises(EngineError, match="MCTrainStep does not log"):
        mc.MCTrainStep(net, xs[0], 2, 1000.0, score_log=mc.ScoreLog(dev, 8))
    # per-step outputs of the serial engine: the reference every captured mode reproduces
    serial_ref = mc.MCForward(net, xs[0], S, **kw)
    ref_outs = []
    for i in range(steps):
        o = serial_ref(labels=ys[i], slot=i)
        ref_outs.append({k: v.clone() for k, v in o.items()})
    torch.cuda.synchronize()
    expected = _expected_log(dev, ref_outs, ys, steps * B)
    modes = {"serial": {}, "loop": dict(fold=False), "overlap": dict(overlap=True),
             "inflight": dict(overlap=True, inflight=4)}
    for name, extra in modes.items():
        log = mc.ScoreLog(dev, steps * B)
        eng = mc.MCForward(net, xs[0], S, score_log=log, **kw, **extra)
        plain = mc.MCForward(net, xs[0], S, **kw, **extra)
        if name == "serial":
            assert (eng.fold_steps is not None) if key == "alexnet" else (eng.layer_fold is not None)
        if name == "loop":
            assert eng.fold_steps is None and eng.layer_fold is None
        torch.cuda.synchronize()
        assert len(log) == 0, name                                  # the warm-up steps are not logged
        assert eng.kernels_per_step == plain.kernels_per_step + 1, (name, eng.kernels_per_step, plain.kernels_per_step)
        for e in (eng, plain):
            for i in range(steps):
                e(labels=ys[i], slot=i)
            e.wait()
        torch.cuda.synchronize()
        for k in plain.out:
            assert torch.equal(eng.out[k], plain.out[k]), (name, k)
            assert torch.equal(eng.out[k], ref_outs[-1][k]), (name, "serial", k)
        _same_log(log.read(), expected, name)
        eng.wait()
        log.reset()
        for i in range(2):                                           # a reset log starts again at entry 0
            eng(labels=ys[i], slot=i)
        eng.wait()
        torch.cuda.synchronize()
        assert len(log) == 2 * B, name
        assert all(e.timeouts() == 0 for e in (eng, plain))


@pytest.mark.parametrize("informed", [True, False])
def test_mc_forward_score_log_eager(dev, informed):
    """graph=False: every call appends its outputs; without uncertainty / labels those planes are NaN."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    xs, ys = _batches(3, 64, 1, dev, seed=8)
    kw = dict(with_labels=informed, seed=4, want_uncertainty=informed, want_information=informed, graph=False)
    log = mc.ScoreLog(dev, 3 * 64)
    eng, plain = mc.MCForward(net, xs[0], 3, score_log=log, **kw), mc.MCForward(net, xs[0], 3, **kw)
    outs = []
    for x, y in zip(xs, ys):
        lab = y if informed else None
        o, p = eng(x, lab), plain(x, lab)
        torch.cuda.synchronize()
        for k in p:
            assert torch.equal(o[k], p[k]), k
        outs.append({k: v.clone() for k, v in o.items()})
    got = log.read()
    _same_log(got, _expected_log(dev, outs, ys if informed else [None] * 3, 3 * 64), informed)
    if not informed:
        for k in PLANES[1:]:
            assert torch.isnan(got[k]).all(), k


def test_mc_forward_score_log_device_check(dev):
    from pytorch_bayesiancnn_b200 import EngineError, mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    with pytest.raises(EngineError, match="score_log"):
        mc.MCForward(net, torch.randn(8, 1, 32, 32, device=dev), 2, score_log=mc.ScoreLog("cpu", 8))


# --------------------------------------------------------------------------- #
# evaluate(score_log=...), detect_ood
# --------------------------------------------------------------------------- #
def _host_batches(n, B, seed, last=None, shift=0.0):
    g = torch.Generator().manual_seed(seed)
    sizes = [B] * n + ([last] if last else [])
    return [(torch.rand(b, 1, 32, 32, generator=g) + shift, torch.randint(0, 10, (b,), generator=g)) for b in sizes]


def test_evaluate_score_log_loader_order_and_same_metrics(dev):
    """A ragged last batch (two engines): the log is in loader order -- the serial engines' outputs appended batch by
    batch -- and the figures are bitwise those of evaluate() without a log."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    batches = _host_batches(4, 128, 8, last=40)
    log = mc.ScoreLog(dev, 2 * (4 * 128 + 40))
    m_log = mc.evaluate(net, batches, 4, 60000.0, "Blundell", seed=21, inflight=4, score_log=log)
    m_plain = mc.evaluate(net, batches, 4, 60000.0, "Blundell", seed=21, inflight=4)
    assert repr(m_log) == repr(m_plain)
    assert len(log) == 4 * 128 + 40
    engines, outs, ys = {}, [], []
    for x, y in batches:                        # evaluate's engines and noise blocks, one serial step per batch
        k = tuple(x.shape)
        if k not in engines:
            engines[k] = mc.MCForward(net, x.to(dev), 4, with_labels=True, train_size=60000.0, seed=21,
                                      first_replay=len(engines) << 16, want_uncertainty=True, want_information=True)
            plain = mc.MCForward(net, x.to(dev), 4, with_labels=True, train_size=60000.0, seed=21,
                                 first_replay=(len(engines) - 1) << 16)
        o = engines[k](x.to(dev), y.to(dev))
        if k == tuple(batches[0][0].shape) and not outs:
            # log_outputs do not depend on the moment flags
            assert torch.equal(o["log_outputs"], plain(x.to(dev), y.to(dev))["log_outputs"])
        outs.append({kk: v.clone() for kk, v in o.items()})
        ys.append(y.to(dev))
    torch.cuda.synchronize()
    _same_log(log.read(), _expected_log(dev, outs, ys, len(log)), "evaluate")
    m_again = mc.evaluate(net, batches, 4, 60000.0, "Blundell", seed=21, inflight=4, score_log=log)
    assert len(log) == 2 * (4 * 128 + 40) and m_again["images"] == 4 * 128 + 40      # appends: reset() starts over


def test_detect_ood_end_to_end(dev):
    """In-distribution rand images against shifted ones: every score's OOD and selective metrics against ood_ref on the
    host copies of the logs; the in-distribution figures are evaluate()'s."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    in_b = _host_batches(3, 128, 1, last=50)
    out_b = _host_batches(2, 128, 2, last=17, shift=3.0)
    res = mc.detect_ood(net, in_b, out_b, 4, score=None, seed=9)
    logs = {k: {p: v.cpu() for p, v in d.items()} for k, d in res["logs"].items()}
    assert logs["in"]["entropy"].numel() == 3 * 128 + 50 and logs["out"]["entropy"].numel() == 2 * 128 + 17
    for nm in mc.OOD_SCORES:
        si, so = [(-d["confidence"] if nm == "confidence" else d[nm]).double().numpy() for d in (logs["in"], logs["out"])]
        ref = R.ood(si, so)
        for k in ref:
            assert abs(res["ood"][nm][k] - ref[k]) <= 1e-12, (nm, k, res["ood"][nm][k], ref[k])
        sref = R.selective(si, logs["in"]["correct"].double().numpy())
        for k in ("aurc", "eaurc", "auroc", "accuracy"):
            a, b = res["selective"][nm][k], sref[k]
            assert (math.isnan(a) and math.isnan(b)) or abs(a - b) <= 1e-12, (nm, k, a, b)
        print(nm, {k: round(v, 4) for k, v in res["ood"][nm].items() if isinstance(v, float)})
    m = mc.evaluate(net, in_b, 4, 1.0, seed=9)
    assert repr(m) == repr(res["in"])
    one = mc.detect_ood(net, in_b, out_b, 4, seed=9)                     # the default score, logs reused
    assert set(one["ood"]) >= {"auroc", "aupr_in", "aupr_out", "fpr_at_95_tpr"}
    assert one["logs"]["in"]["mutual_info"].numel() == 3 * 128 + 50


# --------------------------------------------------------------------------- #
# two GPUs: the logs are identical on every rank
# --------------------------------------------------------------------------- #
def _mp_worker(rank, world, port, out_path):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    xs, ys = _batches(3, 96, 1, dev, seed=3)
    res = {}
    for rb in (1, 2):
        log = mc.ScoreLog(dev, 3 * 96)
        eng = mc.MCForward(net, xs[0], 4, with_labels=True, want_uncertainty=True, want_information=True, seed=5,
                           static_inputs=xs, overlap=True, inflight=2, batch_shards=rb, score_log=log)
        for i in range(3):
            eng(labels=ys[i], slot=i)
        eng.wait()
        res[f"step{rb}"] = {k: v.cpu() for k, v in log.read().items()}
        eng.close()
        elog = mc.ScoreLog(dev, 1000)
        mc.evaluate(net, _host_batches(2, 128, 4, last=30), 4, 1.0, seed=6, batch_shards=rb, score_log=elog)
        res[f"evaluate{rb}"] = {k: v.cpu() for k, v in elog.read().items()}
    torch.save(res, out_path + f".{rank}")
    dist.destroy_process_group()


def test_score_log_two_ranks_identical(dev):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import socket
    import tempfile
    import torch.multiprocessing as mp
    world = 2
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out_path = os.path.join(tempfile.mkdtemp(), "log")
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_mp_worker, args=(r, world, port, out_path)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0
    outs = [torch.load(out_path + f".{r}") for r in range(world)]
    for mode in outs[0]:
        assert outs[0][mode]["entropy"].numel() > 0
        _same_log(outs[0][mode], outs[1][mode], mode)

"""Held-out evaluation on the GPU: the exchange kernel's METRICS instantiation (bbb_mc_exchange_metrics) over emulated
ranks against the float64 restatement tests/eval_ref.py, MCForward(metrics=...) in every mode the engine runs, and
mc.evaluate() against a reference-style loop (one serial step, a host read and host-side calibration per batch)."""
import ctypes as C
import math
import os

import pytest
import torch

from tests import eval_ref as E
from tests.test_gpu_mc import _net
from tests.test_gpu_mc_info import CASES

pytestmark = pytest.mark.gpu
NB = E.BINS
OUT_KEYS = ("lo", "kl", "pred", "epi", "ale", "ent", "head", "ee", "mi")


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _run_ranks(dev, per_rank, S_total, B, Cc, labels, flags, batch_shards, metrics):
    """bbb_mc_exchange_metrics (metrics=True) or bbb_mc_exchange_sharded for len(per_rank) emulated ranks, each on its
    own stream, twice; the outputs and the accumulator of every rank."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn, mc
    lib = L.lib()
    world = len(per_rank)
    rs = world // batch_shards
    nbytes = int(lib.bbb_mc_buffer_bytes(B, Cc, flags, rs))
    bufs = [torch.zeros(nbytes, dtype=torch.uint8, device=dev) for _ in range(world)]
    peers = (C.c_void_p * world)(*[b.data_ptr() for b in bufs])
    states = [torch.zeros(int(lib.bbb_mc_state_bytes()), dtype=torch.uint8, device=dev) for _ in range(world)]
    accs = [mc.new_metrics(dev) for _ in range(world)]
    streams = [torch.cuda.Stream(device=dev) for _ in range(world)]
    klt = torch.tensor(1234.5, device=dev)
    lab = labels.to(dev)
    f32 = dict(dtype=torch.float32, device=dev)
    torch.cuda.synchronize()
    for rep in range(2):
        outs = []
        for r in range(world):
            lg = per_rank[r]
            o = {"lo": torch.empty(B, Cc, **f32), "kl": torch.empty((), **f32), "pred": torch.empty(B, Cc, **f32),
                 "epi": torch.empty(B, Cc, **f32), "ale": torch.empty(B, Cc, **f32), "ent": torch.empty(B, **f32),
                 "head": torch.full((4,), float("nan"), **f32), "ee": torch.full((B,), float("nan"), **f32),
                 "mi": torch.full((B,), float("nan"), **f32)}
            args = (Fn._ptr(lg), 0 if lg is None else lg.shape[0], S_total, B, Cc, Fn._ptr(klt), 1, flags, Fn._ptr(lab),
                    C.c_float(50000.0), C.c_float(0.1), r, world, peers, Fn._ptr(states[r]), Fn._ptr(o["lo"]),
                    Fn._ptr(o["kl"]), *(Fn._ptr(o[k]) for k in ("pred", "epi", "ale", "ent", "head")), None, 0,
                    Fn._ptr(o["ee"]), Fn._ptr(o["mi"]), batch_shards)
            with torch.cuda.stream(streams[r]):
                if metrics:
                    L.check(lib.bbb_mc_exchange_metrics(*args, Fn._ptr(accs[r]), Fn._stream(dev)), "metrics")
                else:
                    L.check(lib.bbb_mc_exchange_sharded(*args, Fn._stream(dev)), "sharded")
            outs.append(o)
        torch.cuda.synchronize()
    for st in states:
        assert int(st[8:12].view(torch.int32).item()) == 0, "an exchange wait timed out"
    return outs, accs


def check_against_ref(m, sums, tag=""):
    """read_metrics' dict against eval_ref.summarize of the same log_outputs: counts exactly, sums within 1e-6
    relative; an image within 1e-6 of a bin edge may sit in either neighbouring bin (counted)."""
    ref = E.summarize(sums)
    assert m["images"] == ref["images"], tag
    for k in ("nll", "accuracy", "brier"):
        assert math.isclose(m[k], ref[k], rel_tol=1e-6, abs_tol=1e-12), (tag, k, m[k], ref[k])
    conf = torch.cat([s["conf"] for s in sums])
    k = (conf * NB).round()
    edge = ((conf * NB - k).abs() < 1e-6 * NB) & (k >= 1) & (k <= NB - 1)    # 0 and 1 have one neighbouring bin only
    n_edge = int(edge.sum())
    cnt = torch.tensor(m["bin_count"], dtype=torch.float64)
    fixed = torch.zeros(NB, dtype=torch.float64).index_add_(0, E.bin_of(conf[~edge]), torch.ones(int((~edge).sum()),
                                                                                                  dtype=torch.float64))
    extra = cnt - fixed
    assert (extra >= 0).all() and int(extra.sum()) == n_edge, (tag, m["bin_count"], fixed.tolist())
    allowed = set()
    for c in conf[edge].tolist():
        k = round(c * NB)
        allowed |= {k - 1, k}
    assert all(extra[b] == 0 or b in allowed for b in range(NB)), tag
    if n_edge == 0:
        assert m["bin_count"] == ref["bin_count"], tag
        for k in ("bin_confidence", "bin_accuracy"):
            for a, b in zip(m[k], ref[k]):
                assert (math.isnan(a) and math.isnan(b)) or math.isclose(a, b, rel_tol=1e-6), (tag, k)
        assert math.isclose(m["ece"], ref["ece"], rel_tol=1e-6, abs_tol=1e-9), (tag, m["ece"], ref["ece"])
    return n_edge


@pytest.mark.parametrize("batch_shards", [1, 2])
@pytest.mark.parametrize("normalized", [False, True])
@pytest.mark.parametrize("S,B,Cc,world", CASES)
def test_exchange_metrics_matches_reference_and_sharded_outputs(dev, S, B, Cc, world, normalized, batch_shards):
    """Rs sample groups x batch_shards row blocks (batch_shards = 2: the case's ranks as Rs = world / 2 groups of two
    blocks, or twice its ranks when world is odd); every output bitwise that of bbb_mc_exchange_sharded, the
    accumulator (two steps) against eval_ref on the returned log_outputs, bitwise equal on every rank."""
    from pytorch_bayesiancnn_b200 import _lib as L, mc
    g = torch.Generator().manual_seed(3)
    logits = torch.randn(S, B, Cc, generator=g) * 4
    labels = torch.randint(0, Cc, (B,), generator=g)
    logits[:, 0, :] = torch.tensor([-200.0] * (Cc - 1) + [0.0])
    if B > 2:
        logits[:, 1, :] = 0.0                                       # a tie over every class: argmax 0
    rs = world if batch_shards == 1 or world % 2 else world // 2
    per_rank = []
    for r in range(rs * batch_shards):
        ids = list(range(r % rs, S, rs))
        b0, b1 = mc.row_block(B, batch_shards, r // rs)
        per_rank.append(logits[ids][:, b0:b1].contiguous().to(dev) if ids else None)
    flags = L.MC_MOMENTS | L.MC_INFO | (L.MC_NORMALIZED if normalized else 0)
    outs, accs = _run_ranks(dev, per_rank, S, B, Cc, labels, flags, batch_shards, True)
    base, _ = _run_ranks(dev, per_rank, S, B, Cc, labels, flags, batch_shards, False)
    for o, b in zip(outs, base):
        for k in OUT_KEYS:
            torch.testing.assert_close(o[k], b[k], rtol=0, atol=0, equal_nan=True, msg=k)
    for a in accs[1:]:
        assert torch.equal(a[:64], accs[0][:64])                     # every rank holds the same accumulator
    m = mc.read_metrics(accs[0])
    assert m["steps"] == 2 and m["images"] == 2 * B
    s = E.batch_sums(outs[0]["lo"].cpu(), labels)
    n_edge = check_against_ref(m, [s, s], (S, B, Cc, world, normalized, batch_shards))
    a = accs[0].cpu()
    head = outs[0]["head"].cpu()
    kl_sum = float(outs[0]["kl"]) * S
    assert math.isclose(float(a[4]) / 2, kl_sum, rel_tol=1e-6)      # sum_j kl_j, not divided by num_ens
    assert math.isclose(float(a[2]) / 2, float(head[1]), rel_tol=1e-6)            # the head's nll and accuracy
    assert math.isclose(float(a[3]) / 2, float(head[2]), rel_tol=1e-6, abs_tol=1e-12)
    print("bin-edge images", n_edge)


# --------------------------------------------------------------------------- #
# MCForward(metrics=...)
# --------------------------------------------------------------------------- #
def _batches(n, B, inputs, Cc=10, seed=5):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(B, inputs, 32, 32, generator=g), torch.randint(0, Cc, (B,), generator=g)) for _ in range(n)]


def _run(eng, batches, dev):
    ys = [y.to(dev) for _, y in batches]          # alive until every step has copied its labels on its own stream
    for i, y in enumerate(ys):
        eng(labels=y, slot=i)                       # inputs resident in static_inputs: steps in flight never share one
    eng.wait()
    torch.cuda.synchronize()
    del ys


def test_mc_forward_metrics_needs_labels_and_an_accumulator(dev):
    from pytorch_bayesiancnn_b200 import EngineError, mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    x = torch.randn(16, 1, 32, 32, device=dev)
    with pytest.raises(EngineError, match="with_labels"):
        mc.MCForward(net, x, 2, metrics=mc.new_metrics(dev))
    with pytest.raises(EngineError, match="float64"):
        mc.MCForward(net, x, 2, with_labels=True, metrics=torch.zeros(8, dtype=torch.float64, device=dev))


@pytest.mark.parametrize("key,inputs", [("alexnet", 3), ("lenet", 1)])
def test_mc_forward_metrics_every_mode_equals_serial(dev, key, inputs):
    """fused fold (AlexNet) / per-layer fold (LeNet), sample loop, overlap + inflight=4: the accumulator bitwise equals
    the serial engine's over the same batches, and the serial one equals eval_ref on its own log_outputs; eager mode
    against eval_ref; warm-up steps do not count; outputs unchanged by the accumulator."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net(key, 10, inputs, "lrt", dev, "auto")
    batches = _batches(5, 128, inputs)
    xs = [x.to(dev) for x, _ in batches]
    x0 = xs[0]
    kw = dict(with_labels=True, train_size=1000.0, beta=0.1, seed=13, want_uncertainty=True, static_inputs=xs)
    acc = {k: mc.new_metrics(dev) for k in ("serial", "loop", "overlap", "eager")}
    serial = mc.MCForward(net, x0, 5, metrics=acc["serial"], **kw)
    assert (serial.fold_steps is not None) if key == "alexnet" else (serial.layer_fold is not None)
    assert int(acc["serial"][0]) == 0                                    # construction adds nothing
    sums = []
    for i, (_, y) in enumerate(batches):
        out = serial(labels=y.to(dev), slot=i)
        torch.cuda.synchronize()
        sums.append(E.batch_sums(out["log_outputs"].cpu(), y))
    m = mc.read_metrics(acc["serial"])
    assert m["steps"] == 5
    check_against_ref(m, sums, "serial")
    loop = mc.MCForward(net, x0, 5, fold=False, metrics=acc["loop"], **kw)
    assert loop.fold_steps is None and loop.layer_fold is None
    _run(loop, batches, dev)
    ovl = mc.MCForward(net, x0, 5, overlap=True, inflight=4, metrics=acc["overlap"], **kw)
    _run(ovl, batches, dev)
    plain = mc.MCForward(net, x0, 5, overlap=True, inflight=4, **kw)
    _run(plain, batches, dev)
    for k in plain.out:
        assert torch.equal(plain.out[k], ovl.out[k]), k
    for k in serial.out:
        assert torch.equal(serial.out[k], ovl.out[k]), ("last step", k)
    for k in ("loop", "overlap"):
        diff = (acc[k][:64] != acc["serial"][:64]).nonzero().flatten().tolist()
        assert not diff, (k, diff, acc[k][diff].tolist(), acc["serial"][diff].tolist())
    eager = mc.MCForward(net, x0, 5, graph=False, metrics=acc["eager"], **kw)
    esums = []
    for x, y in batches[:2]:
        out = eager(x.to(dev), y.to(dev))
        torch.cuda.synchronize()
        esums.append(E.batch_sums(out["log_outputs"].cpu(), y))
    check_against_ref(mc.read_metrics(acc["eager"]), esums, "eager")
    assert all(e.timeouts() == 0 for e in (serial, loop, ovl, plain, eager))


# --------------------------------------------------------------------------- #
# mc.evaluate
# --------------------------------------------------------------------------- #
def reference_loop(net, batches, num_ens, train_size, beta_type, dev, seed, epoch=None, num_epochs=None):
    """validate_model's loop on the engine: one serial step per batch, a host read of it, calibration on the host.
    The engines and noise blocks are evaluate()'s: one engine per batch shape, the k-th one built from block k * 2^16."""
    from pytorch_bayesiancnn_b200 import mc
    engines, los, ys, kls, sums = {}, [], [], [], []
    for i, (x, y) in enumerate(batches):
        key = tuple(x.shape)
        if key not in engines:
            engines[key] = mc.MCForward(net, x.to(dev), num_ens, with_labels=True, train_size=train_size, seed=seed,
                                        first_replay=len(engines) << 16)
        out = engines[key](x.to(dev), y.to(dev))
        lo = out["log_outputs"].cpu()
        los.append(lo); ys.append(y); kls.append(float(out["kl"].item()) * num_ens)
        sums.append(E.batch_sums(lo, y))
    loss, acc = E.validate(los, ys, kls, train_size, beta_type, epoch, num_epochs)
    return loss, acc, sums


@pytest.mark.parametrize("beta_type", [0.1, "Blundell", "Soenderby"])
def test_evaluate_matches_reference_loop(dev, beta_type):
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    batches = _batches(4, 128, 1, seed=8) + _batches(1, 40, 1, seed=9)          # a ragged last batch
    kw = dict(epoch=3, num_epochs=20)
    m = mc.evaluate(net, batches, 4, 60000.0, beta_type, seed=21, inflight=4, **kw)
    loss, acc, sums = reference_loop(net, batches, 4, 60000.0, beta_type, dev, 21, **kw)
    assert m["steps"] == 5 and m["images"] == 4 * 128 + 40
    assert math.isclose(m["valid_loss"], loss, rel_tol=1e-5), (m["valid_loss"], loss)
    assert math.isclose(m["valid_acc"], acc, rel_tol=1e-5, abs_tol=1e-12), (m["valid_acc"], acc)
    check_against_ref(m, sums, beta_type)
    print(beta_type, {k: m[k] for k in ("valid_loss", "valid_acc", "nll", "accuracy", "brier", "ece")})


def test_evaluate_fused_fold_and_batch_shards_argument(dev):
    """BBBAlexNet on the fused fold, one in flight, with an explicit batch_shards=1."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("alexnet", 10, 3, "lrt", dev, "auto")
    batches = _batches(3, 128, 3, seed=4) + _batches(1, 72, 3, seed=6)
    m = mc.evaluate(net, batches, 3, 50000.0, seed=5, inflight=1, batch_shards=1)
    loss, acc, sums = reference_loop(net, batches, 3, 50000.0, 0.1, dev, 5)
    assert math.isclose(m["valid_loss"], loss, rel_tol=1e-5) and math.isclose(m["valid_acc"], acc, rel_tol=1e-5)
    check_against_ref(m, sums, "alexnet")


def test_evaluate_keeps_its_engines_and_takes_device_batches(dev):
    """A second call reuses the engines kept on the net, starts from a zeroed accumulator and draws fresh noise; batches
    already on the device (no pinned staging) give the same figures as the reference loop."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    batches = _batches(3, 64, 1, seed=2) + _batches(1, 24, 1, seed=3)
    dbatches = [(x.to(dev), y.to(dev)) for x, y in batches]
    m1 = mc.evaluate(net, dbatches, 3, 1000.0, seed=4, inflight=2)
    loss, acc, sums = reference_loop(net, batches, 3, 1000.0, 0.1, dev, 4)
    assert math.isclose(m1["valid_loss"], loss, rel_tol=1e-5) and math.isclose(m1["valid_acc"], acc, rel_tol=1e-5)
    check_against_ref(m1, sums, "device batches")
    (ev,) = net._mc_eval.values()
    engines = {k: e["eng"] for k, e in ev["engines"].items()}
    m2 = mc.evaluate(net, batches, 3, 1000.0, seed=4, inflight=2)
    assert {k: e["eng"] for k, e in ev["engines"].items()} == engines          # the same engine objects
    assert m2["steps"] == 4 and m2["images"] == 3 * 64 + 24                     # a zeroed accumulator
    assert m2["nll"] != m1["nll"]                                              # fresh noise
    assert all(e.timeouts() == 0 for e in engines.values())


# --------------------------------------------------------------------------- #
# two GPUs: evaluate with batch_shards=2 == one GPU
# --------------------------------------------------------------------------- #
def _mp_worker(rank, world, port, out_path):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    batches = _batches(3, 128, 1, seed=8) + _batches(1, 40, 1, seed=9)
    res = {"shards": mc.evaluate(net, batches, 4, 60000.0, "Blundell", seed=21, batch_shards=2),
           "samples": mc.evaluate(net, batches, 4, 60000.0, "Blundell", seed=21)}
    torch.save(res, out_path + f".{rank}")
    dist.destroy_process_group()


def test_evaluate_multi_gpu_equals_single_gpu(dev):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import socket
    import tempfile
    import torch.multiprocessing as mp
    from pytorch_bayesiancnn_b200 import mc
    world = 2
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out_path = os.path.join(tempfile.mkdtemp(), "eval")
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_mp_worker, args=(r, world, port, out_path)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
        assert p.exitcode == 0
    outs = [torch.load(out_path + f".{r}") for r in range(world)]
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    batches = _batches(3, 128, 1, seed=8) + _batches(1, 40, 1, seed=9)
    one = mc.evaluate(net, batches, 4, 60000.0, "Blundell", seed=21)
    for mode in ("shards", "samples"):
        assert repr(outs[0][mode]) == repr(outs[1][mode]), mode        # every rank holds the same result
        for k in ("valid_loss", "valid_acc", "nll", "accuracy", "brier", "ece"):
            assert math.isclose(outs[0][mode][k], one[k], rel_tol=1e-4, abs_tol=1e-9), (mode, k)

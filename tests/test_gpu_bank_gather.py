"""The logit gather of sharded Monte-Carlo steps on the GPU (bbb_mc_logit_gather): on emulated ranks of one device, every
rank's gathered [S, B, C] is the full logits bit for bit, and the banks and fits on it are the one-rank ones; on one
rank a grouped bank changes nothing; on two GPUs, MCForward, acquire and calibrate_temperature with grouped banks give
every rank the single-GPU bank and results."""
import ctypes as C
import os
import subprocess
import sys

import pytest
import torch

from tests.conftest import ROOT
from tests.test_gpu_mc import _net

pytestmark = pytest.mark.gpu
SHAPES = [(1, 1, 2), (7, 33, 10), (25, 1024, 100), (3, 700, 1000), (100, 2048, 10)]
WRAP = 0xFFFFFFFE            # the launches the emulated ranks start after: their next three use 2^32 - 1, 0 and 1


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _logits(S, B, Cc, seed):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(S, B, Cc, generator=g) * 4
    flat = z.view(-1)
    idx = torch.randperm(flat.numel(), generator=g)[:max(4, flat.numel() // 50)]
    for k, v in enumerate((float("nan"), float("inf"), float("-inf"), -0.0)):
        flat[idx[k::4]] = v
    flat.view(torch.int32)[idx[0]] = 0x7fc12345                         # a NaN with a payload
    return z


def _bits(t):
    return t.contiguous().view(torch.int32)


class Ranks:
    """`world` emulated ranks of batch_shards `rb` on one device: a receive buffer, a state and a stream each, the
    buffers and states as after launch WRAP (so the next launches run through both slots and the sequence wrap)."""

    def __init__(self, dev, world, rb, S, B, Cc):
        from pytorch_bayesiancnn_b200 import _lib as L
        lib = L.lib()
        self.dev, self.world, self.rb, self.S, self.B, self.C = dev, world, rb, S, B, Cc
        words = S * B * Cc
        assert lib.bbb_mc_gather_bytes(S, B, Cc) == 16 * words
        tag = lambda seq: (seq << 32) - (1 << 64) if seq >= 1 << 31 else seq << 32
        self.bufs = []
        for _ in range(world):
            b = torch.empty(2, words, dtype=torch.int64, device=dev)
            b[0].fill_(tag(WRAP))
            b[1].fill_(tag(WRAP - 1))
            self.bufs.append(b)
        self.peers = (C.c_void_p * world)(*[b.data_ptr() for b in self.bufs])
        self.states = [torch.zeros(int(lib.bbb_mc_state_bytes()), dtype=torch.uint8, device=dev) for _ in range(world)]
        for st in self.states:
            st[:4].view(torch.int32).fill_(WRAP - (1 << 32))
        self.streams = [torch.cuda.Stream(device=dev) for _ in range(world)]

    def local(self, full, r):
        from pytorch_bayesiancnn_b200 import mc
        rs, g, k = mc.shard_layout(self.world, r, self.rb)
        b0, b1 = mc.row_block(self.B, self.rb, k)
        ids = mc.local_samples(self.S, rs, g)
        return full[ids][:, b0:b1].contiguous() if ids else None

    def launch(self, r, lg, out):
        from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
        with torch.cuda.stream(self.streams[r]):
            L.check(L.lib().bbb_mc_logit_gather(Fn._ptr(lg), 0 if lg is None else lg.shape[0], self.S, self.B, self.C, r,
                                                self.world, self.rb, self.peers, Fn._ptr(self.states[r]), Fn._ptr(out),
                                                Fn._stream(self.dev)), "bbb_mc_logit_gather")

    def timeouts(self, r):
        return int(self.states[r][8:12].view(torch.int32).item())

    def gather(self, locals_, reps=3):
        """Every rank's gather `reps` times, all launched before any sync; the outputs of every launch."""
        torch.cuda.synchronize()
        outs = [[torch.empty(self.S, self.B, self.C, device=self.dev) for _ in range(self.world)] for _ in range(reps)]
        for rep in range(reps):
            for r in range(self.world):
                self.launch(r, locals_[r], outs[rep][r])
        torch.cuda.synchronize()
        for r in range(self.world):
            assert self.timeouts(r) == 0, "a gather wait timed out"
        return outs


def _prob_bank(dev, z, normalized=False):
    from pytorch_bayesiancnn_b200 import mc
    b = mc.ProbBank(dev, z.shape[1], z.shape[0], z.shape[2])
    b.append(z, normalized=normalized)
    return b


def _logit_bank(dev, z, labels=None):
    from pytorch_bayesiancnn_b200 import mc
    b = mc.LogitBank(dev, z.shape[1], z.shape[0], z.shape[2])
    b.append(z, labels)
    return b


def _maps(dev, Cc):
    """(name, map in place on [.., C] logits) of the step's three maps: the kernels MCForward runs."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn, mc
    g = torch.Generator().manual_seed(Cc)
    t = torch.tensor([1.37], device=dev)

    def temper(z):
        L.check(L.lib().bbb_mc_temper(Fn._ptr(z), z.numel(), Fn._ptr(t), Fn._stream(dev)), "bbb_mc_temper")
        return z
    vec = mc.LogitScaling(dev, Cc, "vector")
    vec.params.copy_(torch.stack([torch.rand(Cc, generator=g) + 0.5, torch.randn(Cc, generator=g)]).to(dev))
    out = [("temperature", temper), ("vector", vec.apply_)]
    if Cc <= 128:
        mat = mc.LogitScaling(dev, Cc, "matrix")
        mat.params.copy_((torch.eye(Cc + 1, Cc) + 0.1 * torch.randn(Cc + 1, Cc, generator=g)).to(dev))
        out.append(("matrix", mat.apply_))
    return out


def _emulated(dev, world):
    for si, (S, B, Cc) in enumerate(SHAPES):
        full = _logits(S, B, Cc, seed=world * 10 + si)
        fdev = full.to(dev)
        for rb in sorted({1, 2, world}):
            if world % rb or rb > B:
                continue
            ranks = Ranks(dev, world, rb, S, B, Cc)
            locals_ = [None if lg is None else lg.to(dev) for lg in (ranks.local(full, r) for r in range(world))]
            outs = ranks.gather(locals_)
            for rep, per_rank in enumerate(outs):
                for r, o in enumerate(per_rank):
                    assert torch.equal(_bits(o), _bits(fdev)), (world, rb, (S, B, Cc), rep, r)
            if rb != world and world > 2:
                continue
            # the banks on the gathered logits, and after each map: mapping the gathered logits has the bits of
            # gathering the mapped ones, and of mapping the one-rank step's logits
            got = outs[-1][world - 1]
            if Cc <= 128:
                for normalized in (False, True):
                    want = _prob_bank(dev, fdev, normalized)
                    have = _prob_bank(dev, got, normalized)
                    assert torch.equal(_bits(have._probs), _bits(want._probs)) and torch.equal(
                        have._ee.view(torch.int64), want._ee.view(torch.int64)), (world, rb, normalized)
            labels = torch.randint(0, Cc, (B,), device=dev)
            want, have = _logit_bank(dev, fdev, labels), _logit_bank(dev, got, labels)
            assert torch.equal(_bits(have._logits), _bits(want._logits)) and torch.equal(have._labels, want._labels)
            for name, f in _maps(dev, Cc):
                mapped = ranks.gather([None if lg is None else f(lg.clone()) for lg in locals_], reps=1)[0]
                ref = f(fdev.clone())
                here = f(got.clone())
                for o in mapped:
                    assert torch.equal(_bits(o), _bits(here)) and torch.equal(_bits(here), _bits(ref)), (world, rb, name)
                if Cc <= 128:
                    assert torch.equal(_bits(_prob_bank(dev, here)._probs), _bits(_prob_bank(dev, ref)._probs)), name


@pytest.mark.parametrize("world", [2, 3, 4, 8, 16])
def test_emulated_ranks_gather_the_full_logits(dev, world):
    if world <= 8:
        _emulated(dev, world)
        return
    # 16 ranks need 16 streams that do not share a hardware queue (a rank's gather behind another's would wait for it):
    # a process of its own with CUDA_DEVICE_MAX_CONNECTIONS=32
    code = ("import sys, torch; sys.path.insert(0, sys.argv[1]); from tests.test_gpu_bank_gather import _emulated; "
            f"_emulated(torch.device('cuda:0'), {world})")
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")
    r = subprocess.run([sys.executable, "-c", code, ROOT], env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]


def test_a_lost_peer_costs_one_time_out_per_launch(dev, monkeypatch):
    """Rank 1 of 2 never launches: rank 0's gather gives up after about one time-out, not one per word it owns (with
    100 ms, ~125 words of the lost peer per thread at this shape would take 12 s), counts it, and its next launch, with
    the peer back, waits for it again and gathers the full logits."""
    import time
    S, B, Cc = 100, 2048, 10
    monkeypatch.setenv("BBB_B200_MC_TIMEOUT_MS", "100")
    full = _logits(S, B, Cc, seed=3).to(dev)
    ranks = Ranks(dev, 2, 1, S, B, Cc)
    mine = [ranks.local(full, r) for r in range(2)]
    out = [torch.empty(S, B, Cc, device=dev) for _ in range(2)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ranks.launch(0, mine[0], out[0])
    torch.cuda.synchronize()
    took = time.perf_counter() - t0
    lost = ranks.timeouts(0)
    assert lost > 0 and took < 3.0, (lost, took)
    assert int(ranks.states[0][12:16].view(torch.int32).item()) == lost      # where the next launch starts counting
    ranks.states[1][:4].view(torch.int32).add_(1)                             # rank 1 takes up at rank 0's next launch
    for r in range(2):
        ranks.launch(r, mine[r], out[r])
    torch.cuda.synchronize()
    assert ranks.timeouts(0) == lost and ranks.timeouts(1) == 0
    for o in out:
        assert torch.equal(_bits(o), _bits(full))


def test_fits_on_gathered_banks_are_the_one_rank_fits(dev):
    """fit_temperature, fit_scaling (vector and matrix) and batchbald(seed=) on every emulated rank's banks: the one-rank
    bits."""
    from pytorch_bayesiancnn_b200 import mc
    S, B, Cc, world, rb = 10, 512, 10, 4, 2
    g = torch.Generator().manual_seed(9)
    full = (torch.randn(S, B, Cc, generator=g) * 2 + torch.randn(1, B, Cc, generator=g) * 3).to(dev)
    labels = torch.randint(0, Cc, (B,), generator=g).to(dev)
    ranks = Ranks(dev, world, rb, S, B, Cc)
    outs = ranks.gather([None if lg is None else lg for lg in (ranks.local(full, r) for r in range(world))])[-1]

    def fits(z):
        lb, pb = _logit_bank(dev, z, labels), _prob_bank(dev, z)
        t = mc.fit_temperature(lb).read()["temperature"]
        v = mc.fit_scaling(lb, "vector", iters=50).scaling.params.clone()
        m = mc.fit_scaling(lb, "matrix", iters=50).scaling.params.clone()
        bb = mc.batchbald(pb, 4, num_configs=200, seed=11)
        return t, v, m, bb["indices"], bb["scores"]
    want = fits(full)
    for o in outs:
        t, v, m, idx, sc = fits(o)
        assert t == want[0] and torch.equal(_bits(v), _bits(want[1])) and torch.equal(_bits(m), _bits(want[2]))
        assert torch.equal(idx, want[3]) and torch.equal(sc.view(torch.int64), want[4].view(torch.int64))


# --------------------------------------------------------------------------- #
# one rank: a grouped bank is an ungrouped one
# --------------------------------------------------------------------------- #
@pytest.fixture
def one_rank_group(tmp_path):
    import torch.distributed as dist
    if dist.is_initialized():
        pytest.skip("a process group is already initialised")
    dist.init_process_group("gloo", init_method=f"file://{tmp_path / 'pg'}", rank=0, world_size=1)
    yield dist.group.WORLD
    dist.destroy_process_group()


def test_grouped_bank_on_one_rank_is_the_ungrouped_bank(dev, one_rank_group):
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    g = torch.Generator().manual_seed(3)
    xs = [torch.randn(128, 1, 32, 32, generator=g).to(dev) for _ in range(3)]
    ys = [torch.randint(0, 10, (128,), generator=g).to(dev) for _ in range(3)]
    for mode in (dict(), dict(overlap=True, inflight=4), dict(graph=False)):
        res = []
        for group in (None, one_rank_group):
            pb, lb = mc.ProbBank(dev, 384, 4, 10, group=group), mc.LogitBank(dev, 384, 4, 10, group=group)
            eng = mc.MCForward(net, xs[0], 4, seed=21, with_labels=True, want_uncertainty=True, static_inputs=xs,
                               prob_bank=pb, logit_bank=lb, temperature=1.4, **mode)
            outs = []
            for i in range(3):
                o = eng(labels=ys[i], slot=i) if mode.get("graph", True) else eng(xs[i], labels=ys[i])
                eng.wait()
                outs.append({k: v.clone() for k, v in o.items()})
            torch.cuda.synchronize()
            assert eng.gathered_all is None and eng.timeouts() == 0
            res.append((outs, eng.kernels_per_step, pb.read(), lb.read()))
        (o0, k0, p0, l0), (o1, k1, p1, l1) = res
        assert k0 == k1, mode
        for a, b in zip(o0, o1):
            assert all(torch.equal(_bits(a[k]), _bits(b[k])) for k in a), mode
        assert all(torch.equal(p0[k].view(torch.int32 if p0[k].dtype == torch.float32 else torch.int64),
                               p1[k].view(torch.int32 if p1[k].dtype == torch.float32 else torch.int64)) for k in p0)
        assert torch.equal(_bits(l0["logits"]), _bits(l1["logits"])) and torch.equal(l0["labels"], l1["labels"])
    loader = [(x.cpu(), y.cpu()) for x, y in zip(xs, ys)]
    m0 = mc.calibrate_temperature(net, loader, 4, seed=5)
    m1 = mc.calibrate_temperature(net, loader, 4, seed=5, group=one_rank_group)
    assert m0["fit"]["temperature"] == m1["fit"]["temperature"] and repr(m0["evaluate"]) == repr(m1["evaluate"])
    a0 = mc.acquire(net, loader, 5, 4, num_configs=100, seed=3)
    a1 = mc.acquire(net, loader, 5, 4, num_configs=100, seed=3, group=one_rank_group)
    assert torch.equal(a0["indices"], a1["indices"]) and repr(a0["evaluate"]) == repr(a1["evaluate"])


# --------------------------------------------------------------------------- #
# two GPUs: every rank's bank is the single-GPU bank
# --------------------------------------------------------------------------- #
MODES = [dict(batch_shards=1), dict(batch_shards=2), dict(batch_shards=1, overlap=True),
         dict(batch_shards=2, overlap=True, inflight=4)]


def _data(dev):
    g = torch.Generator().manual_seed(8)
    xs = [torch.randn(130, 3, 32, 32, generator=g).to(dev) for _ in range(3)]
    ys = [torch.randint(0, 10, (130,), generator=g).to(dev) for _ in range(3)]
    return xs, ys


def _fill(net, dev, xs, ys, group, **mode):
    """Three steps of a 5-sample MCForward with a ProbBank and a LogitBank of `group`; (banks read, timeouts)."""
    from pytorch_bayesiancnn_b200 import mc
    pb, lb = mc.ProbBank(dev, 390, 5, 10, group=group), mc.LogitBank(dev, 390, 5, 10, group=group)
    eng = mc.MCForward(net, xs[0], 5, group=group, seed=31, with_labels=True, static_inputs=xs, prob_bank=pb,
                       logit_bank=lb, temperature=1.3, **mode)
    for i in range(3):
        eng(labels=ys[i], slot=i)
    eng.wait()
    torch.cuda.synchronize()
    res = {"probs": pb.read()["probs"].cpu(), "ee": pb.read()["expected_entropy"].cpu(),
           "logits": lb.read()["logits"].cpu(), "labels": lb.read()["labels"].cpu(), "timeouts": eng.timeouts()}
    eng.close()
    return res


def _eval_timeouts(net):
    return sum(e["eng"].timeouts() for ev in net.__dict__.get("_mc_eval", {}).values() for e in ev["engines"].values())


def _mp_worker(rank, world, port, out_path):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from pytorch_bayesiancnn_b200 import mc
    group = dist.group.WORLD
    net, _ = _net("alexnet", 10, 3, "lrt", dev, "auto")
    xs, ys = _data(dev)
    res = {"modes": [_fill(net, dev, xs, ys, group, **m) for m in MODES]}
    loader = [(x.cpu(), y.cpu()) for x, y in zip(xs, ys)]
    res["acquire"] = mc.acquire(net, loader, 5, 5, num_configs=100, seed=3, group=group)["indices"]
    res["acquire_unseeded"] = mc.acquire(net, loader, 5, 5, num_configs=100, group=group)["indices"]
    cal = mc.calibrate_temperature(net, loader, 5, seed=5, group=group)
    res["T"] = cal["temperature"].cpu()
    res["eval_timeouts"] = _eval_timeouts(net)
    torch.save(res, out_path + f".{rank}")
    dist.destroy_process_group()


def test_two_gpus_fill_every_rank_with_the_single_gpu_bank(dev):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    import socket
    import tempfile
    import torch.multiprocessing as mp
    from pytorch_bayesiancnn_b200 import mc
    world = 2
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    out_path = os.path.join(tempfile.mkdtemp(), "bank")
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_mp_worker, args=(r, world, port, out_path)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=900)
        assert p.exitcode == 0
    outs = [torch.load(out_path + f".{r}") for r in range(world)]
    net, _ = _net("alexnet", 10, 3, "lrt", dev, "auto")
    xs, ys = _data(dev)
    one = _fill(net, dev, xs, ys, None)
    loader = [(x.cpu(), y.cpu()) for x, y in zip(xs, ys)]
    acq = mc.acquire(net, loader, 5, 5, num_configs=100, seed=3)["indices"]
    T = mc.calibrate_temperature(net, loader, 5, seed=5)["temperature"].cpu()
    for o in outs:
        assert o["eval_timeouts"] == 0
        for m, got in zip(MODES, o["modes"]):
            assert got["timeouts"] == 0, m
            assert torch.equal(_bits(got["probs"]), _bits(one["probs"])), m
            assert torch.equal(got["ee"].view(torch.int64), one["ee"].view(torch.int64)), m
            assert torch.equal(_bits(got["logits"]), _bits(one["logits"])) and torch.equal(got["labels"], one["labels"])
        assert torch.equal(o["acquire"], acq)
        assert torch.equal(o["acquire_unseeded"], outs[0]["acquire_unseeded"])
        assert torch.equal(_bits(o["T"]), _bits(T))

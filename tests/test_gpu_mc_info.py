"""Expected entropy and mutual information (BBB_MC_INFO) of the Monte-Carlo step on the GPU: the exchange kernel's
INFO instantiation over emulated ranks against the float64 reference, and MCForward(want_information=True) in every
mode the engine runs (fused-chain fold, per-layer fold, sample loop, eager, overlapped / in flight, C5 at full size)."""
import ctypes as C

import pytest
import torch

from tests.info_ref import information
from tests.test_gpu_mc import _exchange, _net

pytestmark = pytest.mark.gpu
INFO_KEYS = ("expected_entropy", "mutual_info")


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _exchange_info(dev, logits_per_rank, S_total, labels, normalized, kl):
    """bbb_mc_exchange_info with BBB_MC_INFO for len(logits_per_rank) emulated ranks on one device, each launch on its
    own stream (twice: the second call reuses the slots); the outputs of every rank, with the keys of _exchange."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    lib = L.lib()
    world = len(logits_per_rank)
    B, Cc = next(l for l in logits_per_rank if l is not None).shape[1:]
    flags = L.MC_MOMENTS | L.MC_INFO | (L.MC_NORMALIZED if normalized else 0)
    nbytes = int(lib.bbb_mc_buffer_bytes(B, Cc, flags, world))
    bufs = [torch.zeros(nbytes, dtype=torch.uint8, device=dev) for _ in range(world)]
    peers = (C.c_void_p * world)(*[b.data_ptr() for b in bufs])
    states = [torch.zeros(int(lib.bbb_mc_state_bytes()), dtype=torch.uint8, device=dev) for _ in range(world)]
    streams = [torch.cuda.Stream(device=dev) for _ in range(world)]
    klt = torch.tensor(float(kl), device=dev)
    lab = labels.to(dev)
    torch.cuda.synchronize()
    for rep in range(2):
        outs = []
        for r in range(world):
            lg = logits_per_rank[r]
            f32 = dict(dtype=torch.float32, device=dev)
            o = {"lo": torch.empty(B, Cc, **f32), "kl": torch.empty((), **f32), "pred": torch.empty(B, Cc, **f32),
                 "epi": torch.empty(B, Cc, **f32), "ale": torch.empty(B, Cc, **f32), "ent": torch.empty(B, **f32),
                 "head": torch.full((4,), float("nan"), **f32), "ee": torch.full((B,), float("nan"), **f32),
                 "mi": torch.full((B,), float("nan"), **f32)}
            with torch.cuda.stream(streams[r]):
                rc = lib.bbb_mc_exchange_info(
                    Fn._ptr(lg), 0 if lg is None else lg.shape[0], S_total, B, Cc, Fn._ptr(klt), 1, flags, Fn._ptr(lab),
                    C.c_float(50000.0), C.c_float(0.1), r, world, peers, Fn._ptr(states[r]), Fn._ptr(o["lo"]),
                    Fn._ptr(o["kl"]), *(Fn._ptr(o[k]) for k in ("pred", "epi", "ale", "ent", "head")), None, 0,
                    Fn._ptr(o["ee"]), Fn._ptr(o["mi"]), Fn._stream(dev))
                L.check(rc, "bbb_mc_exchange_info")
            outs.append(o)
        torch.cuda.synchronize()
    for st in states:
        assert int(st[8:12].view(torch.int32).item()) == 0, "an exchange wait timed out"
    return outs


# the (S, B, C, world) cases of test_gpu_mc.py::test_mc_exchange_matches_oracle_single_and_emulated_ranks: solo,
# 3 ranks, C = 100 over 8 ranks, multi-CTA B = 700, and ranks that own no sample; then C5's shape on one and 8 ranks
# (100 samples per image: the longest per-lane sums)
CASES = [(1, 5, 10, 1), (7, 33, 10, 3), (25, 64, 100, 8), (3, 700, 10, 4), (2, 9, 10, 4), (100, 2048, 10, 1),
         (100, 2048, 10, 8)]


@pytest.mark.parametrize("normalized", [False, True])
@pytest.mark.parametrize("S,B,Cc,world", CASES)
def test_exchange_info_matches_oracle_and_leaves_other_outputs_unchanged(dev, S, B, Cc, world, normalized):
    g = torch.Generator().manual_seed(2)
    logits = torch.randn(S, B, Cc, generator=g) * 4
    labels = torch.randint(0, Cc, (B,), generator=g)
    logits[:, 0, :] = torch.tensor([-200.0] * (Cc - 1) + [0.0])    # probabilities that underflow fp32 in every sample
    if S > 1:
        logits[:, B - 1, :] = logits[0, B - 1, :]                   # identical samples: no mutual information
    per_rank = []
    for r in range(world):
        ids = list(range(r, S, world))
        per_rank.append(logits[ids].contiguous().to(dev) if ids else None)
    outs = _exchange_info(dev, per_rank, S, labels, normalized, kl=1234.5)
    base = _exchange(dev, per_rank, S, labels, True, normalized, train_size=50000.0, beta=0.1, kl=1234.5)
    ree, rmi = information(list(logits), normalized=normalized)
    for o, b in zip(outs, base):
        assert torch.isfinite(o["ee"]).all() and torch.isfinite(o["mi"]).all()
        e_ee = float((o["ee"].double().cpu() - ree).abs().max())
        e_mi = float((o["mi"].double().cpu() - rmi).abs().max())
        assert e_ee < 1e-5 and e_mi < 1e-5, (e_ee, e_mi)
        assert torch.equal(o["mi"], o["ent"] - o["ee"])             # mutual_info = entropy - expected_entropy in fp32
        for k in b:                                                # the INFO kernel changes nothing else, bit for bit
            torch.testing.assert_close(o[k], b[k], rtol=0, atol=0, equal_nan=True, msg=k)
    for o in outs[1:]:                                             # rank order: bitwise identical on every rank
        assert torch.equal(o["ee"], outs[0]["ee"]) and torch.equal(o["mi"], outs[0]["mi"])


def _check_oracle(eng, out, normalized=False, tol=5e-5):
    """The new outputs == the float64 reference on the engine's own per-sample logits (one rank: all samples)."""
    ree, rmi = information(list(eng.logits.cpu()), normalized=normalized)
    e_ee = float((out["expected_entropy"].double().cpu() - ree).abs().max())
    e_mi = float((out["mutual_info"].double().cpu() - rmi).abs().max())
    assert e_ee < tol and e_mi < tol, (e_ee, e_mi)
    assert torch.isfinite(out["expected_entropy"]).all() and torch.isfinite(out["mutual_info"]).all()
    return e_ee, e_mi


NETS = [("alexnet", 3, "lrt"), ("alexnet", 3, "bbb"), ("lenet", 1, "lrt"), ("lenet", 1, "bbb"),
        ("3conv3fc", 1, "lrt"), ("3conv3fc", 1, "bbb")]


@pytest.mark.parametrize("key,inputs,variant", NETS)
def test_mc_forward_information_folded_equals_sample_loop(dev, key, inputs, variant):
    """Fused-chain fold (BBBAlexNet) and per-layer fold (BBBLeNet, BBB3Conv3FC) against the sample loop; both against
    the reference on their own logits; the existing outputs equal an engine built without information."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net(key, 10, inputs, variant, dev, "auto")
    x = torch.randn(256, inputs, 32, 32, device=dev)
    kw = dict(want_uncertainty=True, seed=11)
    a = mc.MCForward(net, x, 5, fold=True, want_information=True, **kw)
    b = mc.MCForward(net, x, 5, fold=False, want_information=True, **kw)
    c = mc.MCForward(net, x, 5, fold=True, **kw)
    assert (a.fold_steps is not None) if key == "alexnet" else (a.layer_fold is not None)
    assert b.fold_steps is None and b.layer_fold is None
    assert a.kernels_per_step == c.kernels_per_step
    oa = {k: v.clone() for k, v in a(x).items()}
    ob = {k: v.clone() for k, v in b(x).items()}
    oc = c(x)
    torch.cuda.synchronize()
    assert set(oa) == set(oc) | set(INFO_KEYS)
    assert torch.equal(a.logits, c.logits)
    for k in oc:
        assert torch.equal(oa[k], oc[k]), k
    assert torch.equal(a.logits, b.logits)
    for k in INFO_KEYS:
        assert torch.equal(oa[k], ob[k]), k
    print(key, variant, "oracle err", _check_oracle(a, oa), _check_oracle(b, ob))
    assert a.timeouts() == 0 and b.timeouts() == 0


@pytest.mark.parametrize("key,inputs", [("alexnet", 3), ("lenet", 1)])
def test_mc_forward_information_overlap_eager_and_replays(dev, key, inputs):
    """overlap + inflight=4 == the serial engine bit for bit, step for step (the new outputs follow result_stream);
    replays draw fresh noise; graph=False runs the same kernel eagerly."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net(key, 10, inputs, "lrt", dev, "auto")
    x = torch.randn(128, inputs, 32, 32, device=dev)
    kw = dict(want_uncertainty=True, want_information=True, seed=3)
    a = mc.MCForward(net, x, 5, **kw)
    d = mc.MCForward(net, x, 5, overlap=True, inflight=4, **kw)
    assert d.inflight == 4 and d.result_stream is not None
    prev = None
    for n in (1, 2, 5):
        for _ in range(n):
            oa = a(x)
        ra = {k: v.clone() for k, v in oa.items()}
        for _ in range(n):
            od = d(x)
        d.wait()
        torch.cuda.synchronize()
        for k in ra:
            assert torch.equal(ra[k], od[k]), (n, k)
        _check_oracle(a, ra)
        if prev is not None:
            for k in INFO_KEYS:
                assert not torch.equal(prev[k], ra[k]), k           # fresh noise per replay
        prev = ra
    e = mc.MCForward(net, x, 5, graph=False, **kw)
    oe = e(x)
    torch.cuda.synchronize()
    _check_oracle(e, oe)
    assert a.timeouts() == 0 and d.timeouts() == 0 and e.timeouts() == 0


def test_mc_forward_information_normalized_and_tuple(dev):
    """softplus-normalised p_hat through MCForward; mc_forward's uncertainty tuple grows to six only on request."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    x = torch.randn(128, 1, 32, 32, device=dev)
    eng = mc.MCForward(net, x, 4, want_uncertainty=True, normalized=True, want_information=True, seed=7)
    out = eng(x)
    torch.cuda.synchronize()
    _check_oracle(eng, out, normalized=True)
    r4 = mc.mc_forward(net, x, 4, want_uncertainty=True, seed=7)
    r6 = mc.mc_forward(net, x, 4, want_uncertainty=True, seed=7, information=True)
    assert len(r4[2]) == 4 and len(r6[2]) == 6


def test_c5_information_full_size(dev):
    """C5 (BBB3Conv3FC, 1x32x32, B = 2048, 100 samples, LRT): finite, equal to the reference on the engine's logits, and
    the same number of kernels per step as without information.  (At this random initialisation BBB3Conv3FC's logits are
    far apart, so most per-sample entropies are 0: the C5 shape with spread-out logits is a case of the exchange test.)"""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("3conv3fc", 10, 1, "lrt", dev, "auto")
    x = torch.rand(2048, 1, 32, 32, device=dev)
    a = mc.MCForward(net, x, 100, want_uncertainty=True, want_information=True, seed=99)
    out = {k: v.clone() for k, v in a(x).items()}
    torch.cuda.synchronize()
    for k, v in out.items():
        assert torch.isfinite(v).all(), k
    print("C5 information oracle err", _check_oracle(a, out), "max expected entropy / mutual info",
          float(out["expected_entropy"].max()), float(out["mutual_info"].max()))
    assert not torch.signbit(out["expected_entropy"]).any()             # H >= 0, and an entropy of 0 is +0
    assert (out["mutual_info"] >= -1e-5).all()
    n_info = a.kernels_per_step
    del a
    b = mc.MCForward(net, x, 100, want_uncertainty=True, seed=99)
    assert b.kernels_per_step == n_info

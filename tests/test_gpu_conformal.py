"""Split conformal prediction on the GPU: bbb_mc_conformal_log against the float64 reference (tests/conformal_ref.py)
at every class count band it takes, its cursor, MCForward(conformal=...) in every mode the engine runs,
evaluate(conformal=...) and mc.conformal end to end."""
import math

import numpy as np
import pytest
import torch

from tests import conformal_ref as R
from tests.test_gpu_mc import _net

pytestmark = pytest.mark.gpu
METHOD_ID = {R.LAC: 0, R.APS: 1, R.RAPS: 2}
VARIANTS = [(R.LAC, False, 0.0, 0), (R.APS, False, 0.0, 0), (R.APS, True, 0.0, 0), (R.RAPS, True, 0.05, 2),
            (R.RAPS, False, 0.01, 0)]
SEED, STREAM = 0x9E3779B97F4A7C15, (1 << 33) + 7


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _rows(B, C, seed):
    """Log-probabilities with ties, peaked rows (one class at log 0, the rest -inf or -1e30) and a NaN row; labels
    on the peak of every peaked row, so that a randomised APS score there is u itself."""
    g = np.random.default_rng(seed)
    lo = np.log(g.dirichlet(np.full(C, 0.5), size=B)).astype(np.float32)
    y = g.integers(0, C, B)
    lo[B // 3:B // 2] = np.round(lo[B // 3:B // 2] * 2) / 2                     # many ties
    for b in range(0, B, 5):                                                   # peaked
        lo[b] = -np.inf if b % 10 == 0 else -1e30
        lo[b, b % C] = 0.0
        y[b] = b % C
    if B > 3:
        lo[3, :] = math.log(1.0 / C)                                           # every class tied
        lo[1, 1 % C] = np.nan
    return lo, y


def _launch(lo, y, opts, qhat, per_class, cap, cursor, out, dev):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    import ctypes as C
    method, randomized, lam, k_reg = opts
    L.check(L.lib().bbb_mc_conformal_log(
        Fn._ptr(lo), Fn._ptr(y), lo.shape[0], lo.shape[1], METHOD_ID[method], int(randomized), C.c_double(lam), k_reg,
        C.c_uint64(SEED), C.c_uint64(STREAM), Fn._ptr(qhat), int(per_class), Fn._ptr(out["score"]),
        Fn._ptr(out["size"]), Fn._ptr(out["covered"]), Fn._ptr(out["label"]), Fn._ptr(out["sets"]), cap,
        Fn._ptr(cursor), Fn._stream(dev)), "conformal_log")


def _outputs(cap, C, dev, guard=0):
    w = (C + 31) // 32
    return {"score": torch.full((cap + guard,), 7.0, dtype=torch.float64, device=dev),
            "size": torch.full((cap + guard,), -5, dtype=torch.int32, device=dev),
            "covered": torch.full((cap + guard,), -5, dtype=torch.int32, device=dev),
            "label": torch.full((cap + guard,), -5, dtype=torch.int32, device=dev),
            "sets": torch.full(((cap + guard) * w,), -5, dtype=torch.int32, device=dev)}


def _bits(words, n, C):
    w = (C + 31) // 32
    v = words[:n * w].view(n, w).cpu().numpy().astype(np.uint32)
    return np.unpackbits(v.view(np.uint8), axis=1, bitorder="little")[:, :C].astype(bool)


def _check(out, ref, off, n, C, q, tag):
    score = out["score"][off:off + n].cpu().numpy()
    rs = ref["score"]
    assert np.array_equal(np.isnan(score), np.isnan(rs)), tag
    ok = ~np.isnan(rs)
    assert np.abs(score[ok] - rs[ok]).max(initial=0.0) <= 1e-12, (tag, np.abs(score[ok] - rs[ok]).max())
    assert np.array_equal(out["label"][off:off + n].cpu().numpy(), ref["label"]), tag
    w = (C + 31) // 32
    sets = _bits(out["sets"][off * w:], n, C)
    qq = np.broadcast_to(np.asarray(q, dtype=np.float64).reshape(-1), (C,))
    with np.errstate(invalid="ignore"):
        near = np.abs(ref["E"] - qq[None, :]) <= 1e-12
    assert np.array_equal(sets | near, ref["sets"] | near), tag
    size = out["size"][off:off + n].cpu().numpy()
    cov = out["covered"][off:off + n].cpu().numpy()
    y = ref["label"]
    if np.isnan(qq).any():
        assert (size == -1).all() and (cov == -1).all() and not sets.any(), tag
        return
    assert np.array_equal(size, sets.sum(1)), tag
    has = y >= 0
    assert np.array_equal(cov[has], sets[has, y[has]]) and (cov[~has] == -1).all(), tag
    if qq.min() == qq.max():
        # the invariant: a scored image is covered exactly when its own score is <= q_hat
        assert np.array_equal(cov[has & ok] == 1, score[has & ok] <= qq[0]), tag


@pytest.mark.parametrize("opts", VARIANTS, ids=lambda o: f"{o[0]}-{'rand' if o[1] else 'det'}-{o[2]}-{o[3]}")
@pytest.mark.parametrize("B", [1, 7, 512])
@pytest.mark.parametrize("C", [2, 3, 10, 32, 33, 100, 1000, 1024])
def test_conformal_kernel_against_float64(dev, C, B, opts):
    lo, y = _rows(B, C, 17 * C + B)
    y_t = torch.from_numpy(y).to(dev)
    if B > 2:
        y_t[B // 2] = C + 3                                                    # a label outside [0, C)
    lo_t = torch.from_numpy(lo).to(dev)
    y_np = y_t.cpu().numpy()
    base = R.entries(lo, y_np, *opts, SEED, STREAM, 0, np.nan)
    fin = base["score"][~np.isnan(base["score"])]
    g = np.random.default_rng(C + B)
    thresholds = {"none": (np.array([np.nan]), False), "inf": (np.array([np.inf]), False),
                  "scalar": (np.array([np.median(fin) if fin.size else 0.5]), False),
                  "class": (g.random(C) * (1.5 if opts[0] != R.RAPS else 3.0), True)}
    for name, (q, per_class) in thresholds.items():
        out = _outputs(B, C, dev)
        cursor = torch.zeros(2, dtype=torch.int64, device=dev)
        _launch(lo_t, y_t, opts, torch.from_numpy(q).to(dev), per_class, B, cursor, out, dev)
        torch.cuda.synchronize()
        assert cursor.tolist() == [B, 0]
        ref = R.entries(lo, y_np, *opts, SEED, STREAM, 0, q)
        _check(out, ref, 0, B, C, q, (C, B, opts, name))
    if opts[0] == R.APS and opts[1]:
        # peaked rows with the label on the peak: S = 0 and p = 1, so the score is u, bit for bit
        peaked = np.arange(0, B, 5)
        assert np.array_equal(out["score"][peaked].cpu().numpy(), base["u"][peaked]), (C, B)


@pytest.mark.parametrize("C", [10, 1000])
def test_conformal_cursor_appends_overflow_and_capacity_zero(dev, C):
    """Launches append one after another and take u at their log index; past the capacity nothing is written (the
    guard entries stay) and the images are counted; a log of no capacity counts every image."""
    opts = (R.RAPS, True, 0.02, 1)
    sizes, cap, guard = (300, 7, 512, 1, 400), 1000, 64
    out = _outputs(cap, C, dev, guard)
    cursor = torch.zeros(2, dtype=torch.int64, device=dev)
    q = np.array([0.8])
    q_t = torch.from_numpy(q).to(dev)
    batches = [_rows(b, C, i) for i, b in enumerate(sizes)]
    for lo, y in batches:
        _launch(torch.from_numpy(lo).to(dev), torch.from_numpy(y).to(dev), opts, q_t, False, cap, cursor, out, dev)
    torch.cuda.synchronize()
    total = sum(sizes)
    assert cursor.tolist() == [total, total - cap]
    w = (C + 31) // 32
    for k in ("score", "size", "covered", "label"):
        assert (out[k][cap:] == (7.0 if k == "score" else -5)).all(), k
    assert (out["sets"][cap * w:] == -5).all()
    off = 0
    for lo, y in batches:
        n = min(lo.shape[0], cap - off)
        if n <= 0:
            break
        ref = R.entries(lo[:n], y[:n], *opts, SEED, STREAM, off, q)
        _check(out, ref, off, n, C, q, ("append", off))
        off += n
    zero = _outputs(0, C, dev, 1)
    cz = torch.zeros(2, dtype=torch.int64, device=dev)
    lo, y = batches[0]
    _launch(torch.from_numpy(lo).to(dev), torch.from_numpy(y).to(dev), opts, q_t, False, 0, cz, zero, dev)
    torch.cuda.synchronize()
    assert cz.tolist() == [300, 300] and (zero["size"] == -5).all()


def test_conformal_refuses_out_of_range(dev):
    from pytorch_bayesiancnn_b200 import EngineError
    lo = torch.zeros(4, 10, device=dev)
    y = torch.zeros(4, dtype=torch.int64, device=dev)
    out = _outputs(4, 10, dev)
    q = torch.zeros(1, dtype=torch.float64, device=dev)
    cursor = torch.zeros(2, dtype=torch.int64, device=dev)
    for opts in ((R.RAPS, True, -1.0, 0), (R.RAPS, True, float("inf"), 0), (R.RAPS, True, float("nan"), 0),
                 (R.RAPS, True, 0.0, -1)):
        with pytest.raises(EngineError, match="lam/k_reg"):
            _launch(lo, y, opts, q, False, 4, cursor, out, dev)
    with pytest.raises(EngineError, match="B/C"):
        _launch(lo[:, :1].contiguous(), y, (R.LAC, False, 0.0, 0), q, False, 4, cursor, out, dev)
    with pytest.raises(EngineError, match="capacity"):
        _launch(lo, y, (R.LAC, False, 0.0, 0), q, False, 1 << 48, cursor, out, dev)
    torch.cuda.synchronize()
    assert cursor.tolist() == [0, 0]


# --------------------------------------------------------------------------- #
# MCForward(conformal=...), evaluate(conformal=...)
# --------------------------------------------------------------------------- #
def _expected(dev, outs, labels, log):
    """A log with the same options and threshold, fed the given per-step outputs by append."""
    from pytorch_bayesiancnn_b200 import mc
    ref = mc.ConformalLog(dev, log.capacity, log.num_classes, **log._options())
    if log.threshold is not None:
        ref.set_threshold(log.threshold)
    for o, y in zip(outs, labels):
        ref.append(o["log_outputs"], y)
    torch.cuda.synchronize()
    return ref.read()


def _same(got, ref, tag):
    assert set(got) == set(ref), tag
    for k in ref:
        assert torch.equal(got[k], ref[k]) or (k == "score" and torch.equal(got[k].view(torch.int64),
                                                                             ref[k].view(torch.int64))), (tag, k)


@pytest.mark.parametrize("key,inputs,dtype", [("alexnet", 3, torch.float32), ("lenet", 1, torch.float32),
                                              ("lenet", 1, torch.bfloat16)])
def test_mc_forward_conformal_every_mode(dev, key, inputs, dtype):
    """graph=False, serial graph (fused fold on AlexNet, per-layer fold on LeNet), the sample loop, overlap and
    inflight=4: every output is that of the same engine without a log, bit for bit; the log equals append() on the
    outputs; the warm-up steps are not logged; one more kernel per step."""
    from pytorch_bayesiancnn_b200 import EngineError, mc
    net, _ = _net(key, 10, inputs, "lrt", dev, "auto")
    steps, B, S = 4, 128, 3
    g = torch.Generator().manual_seed(5)
    xs = [torch.randn(B, inputs, 32, 32, generator=g).to(dtype).to(dev) for _ in range(steps)]
    ys = [torch.randint(0, 10, (B,), generator=g).to(dev) for _ in range(steps)]
    kw = dict(with_labels=True, seed=13, static_inputs=xs)
    with pytest.raises(EngineError, match="MCTrainStep does not log conformal"):
        mc.MCTrainStep(net, xs[0], 2, 1000.0, conformal=mc.ConformalLog(dev, 8, 10))
    with pytest.raises(EngineError, match="conformal log holds"):
        mc.MCForward(net, xs[0], S, conformal=mc.ConformalLog(dev, 8, 11), **kw)
    # graph=False
    log = mc.ConformalLog(dev, steps * B, 10, method="raps", lam=0.01, k_reg=2, seed=3)
    log.set_threshold(0.9)
    eng = mc.MCForward(net, xs[0], S, conformal=log, graph=False, **kw)
    plain = mc.MCForward(net, xs[0], S, graph=False, **kw)
    outs = []
    for i in range(steps):
        o, p = eng(xs[i], ys[i]), plain(xs[i], ys[i])
        torch.cuda.synchronize()
        for k in p:
            assert torch.equal(o[k], p[k]), ("eager", k)
        outs.append({k: v.clone() for k, v in o.items()})
    _same(log.read(), _expected(dev, outs, ys, log), "eager")
    # captured modes: the serial engine's per-step outputs are what every mode reproduces
    serial = mc.MCForward(net, xs[0], S, **kw)
    outs = []
    for i in range(steps):
        outs.append({k: v.clone() for k, v in serial(labels=ys[i], slot=i).items()})
    torch.cuda.synchronize()
    modes = {"serial": {}, "loop": dict(fold=False), "overlap": dict(overlap=True),
             "inflight": dict(overlap=True, inflight=4)}
    for name, extra in modes.items():
        log = mc.ConformalLog(dev, steps * B, 10, method="aps", seed=4, stream=1)
        eng = mc.MCForward(net, xs[0], S, conformal=log, **kw, **extra)
        plain = mc.MCForward(net, xs[0], S, **kw, **extra)
        if name == "serial" and dtype == torch.float32:
            assert (eng.fold_steps is not None) if key == "alexnet" else (eng.layer_fold is not None)
        torch.cuda.synchronize()
        assert len(log) == 0, name
        assert eng.kernels_per_step == plain.kernels_per_step + 1, name
        log.set_threshold(torch.linspace(0.5, 1.0, 10, dtype=torch.float64))     # set after capture: read in place
        for e in (eng, plain):
            for i in range(steps):
                e(labels=ys[i], slot=i)
            e.wait()
        torch.cuda.synchronize()
        for k in plain.out:
            assert torch.equal(eng.out[k], plain.out[k]), (name, k)
            assert torch.equal(eng.out[k], outs[-1][k]), (name, "serial", k)
        got = log.read()
        assert (got["size"] >= 0).all(), name
        _same(got, _expected(dev, outs, ys, log), name)
        assert all(e.timeouts() == 0 for e in (eng, plain))


def _host_batches(n, B, seed, last=None):
    g = torch.Generator().manual_seed(seed)
    sizes = [B] * n + ([last] if last else [])
    return [(torch.rand(b, 1, 32, 32, generator=g), torch.randint(0, 10, (b,), generator=g)) for b in sizes]


def test_evaluate_conformal_same_figures(dev):
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    batches = _host_batches(3, 128, 8, last=40)
    log = mc.ConformalLog(dev, 424, 10, seed=1)
    m_log = mc.evaluate(net, batches, 4, 60000.0, "Blundell", seed=21, inflight=4, conformal=log)
    m_plain = mc.evaluate(net, batches, 4, 60000.0, "Blundell", seed=21, inflight=4)
    assert repr(m_log) == repr(m_plain)
    got = log.read()
    assert got["score"].numel() == 424 and not torch.isnan(got["score"]).any()
    assert torch.equal(got["label"].long().cpu(), torch.cat([y for _, y in batches]))
    assert (got["size"] == -1).all()                              # no threshold: a calibration log


def test_conformal_end_to_end_coverage(dev):
    """One distribution for calibration (2000) and test (5000) images, alpha = 0.1: the test coverage lies within a
    4-sigma binomial band of [0.9, 0.9 + 1/2001]; every test set equals the float64 sets of the test log's own scores
    at q_hat (classes within 1e-12 of it excepted), and q_hat is conformal_quantile of the calibration scores."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    g = torch.Generator().manual_seed(0)
    protos = torch.rand(10, 1, 32, 32, generator=g)

    def batches(n, B):
        out = []
        for _ in range(n // B):
            y = torch.randint(0, 10, (B,), generator=g)
            out.append((protos[y] + 0.8 * torch.rand(B, 1, 32, 32, generator=g), y))
        return out
    cal, test = batches(2000, 250), batches(5000, 250)
    res = mc.conformal(net, cal, test, 4, alpha=0.1, method="aps", seed=11)
    n, m, alpha = 2000, 5000, 0.1
    assert res["calibration"]["n"] == n and res["calibration"]["rank"] == math.ceil((n + 1) * 0.9)
    cs = res["logs"]["calibration"]["score"]
    assert float(res["qhat"]) == float(mc.conformal_quantile(cs, alpha))
    tm = res["test"]
    sigma = math.sqrt(0.9 * 0.1 / m)
    print("coverage", tm["coverage"], "mean size", tm["mean_size"], "qhat", float(res["qhat"]))
    assert 0.9 - 4 * sigma <= tm["coverage"] <= 0.9 + 1 / (n + 1) + 4 * sigma
    assert tm["n"] == m and int(tm["size_histogram"].sum()) == m
    assert repr(res["in"]) == repr(mc.evaluate(net, cal, 4, 1.0, seed=11))
    # Mondrian: one threshold per class, and the log's sets follow them
    mon = mc.conformal(net, cal, test, 4, alpha=0.1, method="lac", randomized=False, mondrian=True, seed=11)
    assert mon["qhat"].shape == (10,)
    print("mondrian coverage", mon["test"]["coverage"], "min class", mon["test"]["min_class_coverage"])
    assert mon["test"]["coverage"] >= 0.9 - 4 * sigma

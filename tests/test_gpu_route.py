"""Routing between task experts on the GPU: every expert inside an ExpertStep computes the bits it computes alone, the
routing kernel agrees with the float64 restatement (tests/route_ref.py) on the experts' own planes and on planted ties,
NaN scores and invalid labels, the per-batch step and mc.route in flight give the same log and accumulator bits, and
every score kind runs with and without a log."""
import numpy as np
import pytest
import torch

from tests import route_ref as R
from tests.util import CFG_PRIORS, load_params_into

pytestmark = pytest.mark.gpu
ACC_WORDS = 6 + 2 * R.MAX_EXPERTS


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _experts(key, K, C, inputs, variant, dev, seed0=100):
    """K experts of one architecture with different weights (init seeds seed0 + k)."""
    from pytorch_bayesiancnn_b200 import models as M
    from oracle import bbb_oracle as O
    cls = {"alexnet": M.BBBAlexNet, "lenet": M.BBBLeNet}[key]
    nets = []
    for k in range(K):
        params = O.init_params(key, C, inputs, CFG_PRIORS, seed=seed0 + k)
        net = load_params_into(cls(C, inputs, CFG_PRIORS, variant, "softplus"), params).to(dev).train()
        net.set_flag("math", "auto")                     # the tensor-core path, which folds
        nets.append(net)
    return nets


def _np(outs):
    return [{k: v.detach().cpu().numpy() for k, v in o.items() if v.dim() > 0} for o in outs]


def _check_against_ref(planes, score, got, tag, offsets=None):
    """ExpertStep / route_batch outputs against route_ref on the same planes: decisions exact wherever the top two
    scores differ by more than 1e-12 relative, scores within 1e-6 relative."""
    e, local, pred, S = R.route(planes, score, offsets)
    gs = got["scores"].cpu().numpy().astype(np.float64)
    fin = np.isfinite(S)
    assert np.array_equal(np.isnan(gs), np.isnan(S)), tag
    assert (np.abs(gs[fin] - S[fin]) <= 1e-6 * np.abs(S[fin]) + 1e-30).all(), tag
    srt = np.sort(np.where(np.isnan(S), np.inf, S), axis=1)
    with np.errstate(invalid="ignore"):                 # rows whose scores are all NaN compare as not clear
        clear = np.abs(srt[:, 1] - srt[:, 0]) > 1e-12 * np.maximum(np.abs(srt[:, 0]), np.abs(srt[:, 1]))
    assert clear.mean() > 0.5, tag                       # the comparison is not vacuous
    ge = got["expert"].cpu().numpy()
    gl = (got["local_pred"] if "local_pred" in got else got["local"]).cpu().numpy()
    gp = got["pred"].cpu().numpy()
    assert np.array_equal(ge[clear], e[clear]), tag
    assert np.array_equal(gl[clear], local[clear]), tag
    assert np.array_equal(gp[clear], pred[clear]), tag
    return clear


def _check_acc(acc_t, ref, K, tag):
    a = acc_t[:ACC_WORDS].cpu().numpy()
    assert a[0] == ref["steps"] and a[1] == ref["images"], tag
    assert a[3] == ref["global"] and a[4] == ref["own"] and a[5] == ref["invalid"], tag
    assert np.array_equal(a[6:6 + K], ref["selected"]), tag
    assert abs(a[2] - ref["sum_local_acc"]) <= 1e-12 * max(1.0, abs(ref["sum_local_acc"])), tag
    ts = a[6 + R.MAX_EXPERTS:6 + R.MAX_EXPERTS + K]
    ref_ts = ref["total_score"]
    assert np.array_equal(np.isnan(ts), np.isnan(ref_ts)), tag           # a NaN score makes its expert's sum NaN
    fin = ~np.isnan(ref_ts)
    assert np.all(np.abs(ts[fin] - ref_ts[fin]) <= 1e-12 * np.abs(ref_ts[fin]) + 1e-300), tag
    assert not a[6 + K:6 + R.MAX_EXPERTS].any() and not a[6 + R.MAX_EXPERTS + K:ACC_WORDS].any(), tag


CASES = {
    "lenet-lrt-K2": ("lenet", 2, 1, "lrt", torch.float32),
    "lenet-lrt-K5": ("lenet", 5, 1, "lrt", torch.float32),
    "lenet-bbb-K2": ("lenet", 2, 1, "bbb", torch.float32),
    "alexnet-lrt-K2-fused": ("alexnet", 2, 3, "lrt", torch.float32),
    "lenet-lrt-K2-bf16": ("lenet", 2, 1, "lrt", torch.bfloat16),
}


@pytest.mark.parametrize("case", list(CASES))
def test_experts_unaffected_and_kernel_matches_reference(dev, case):
    """Each expert's out tensors inside an ExpertStep are the bits of a lone MCForward with the same seed and
    first_replay; the routing of those planes, its accumulator and its log agree with route_ref."""
    from pytorch_bayesiancnn_b200 import mc
    key, K, inputs, variant, dtype = CASES[case]
    C, B, S, steps = 10 // K, 256, 10, 3
    nets = _experts(key, K, C, inputs, variant, dev)
    g = torch.Generator().manual_seed(7)
    xs = [torch.randn(B, inputs, 32, 32, generator=g).to(dtype).to(dev) for _ in range(steps)]
    ys = [torch.randint(0, K * C, (B,), generator=g).to(dev) for _ in range(steps)]
    acc = mc.new_route_metrics(dev)
    log = mc.RouteLog(dev, steps * B, K)
    step = mc.ExpertStep(nets, xs[0], S, seed=21, static_inputs=xs, first_replay=3, metrics=acc, log=log)
    if key == "alexnet":
        assert all(e.fold_steps is not None for e in step.engines), "the fused chain did not fold"
    elif variant == "lrt":
        assert all(e.layer_fold is not None for e in step.engines), "the per-layer fold did not run"
    got, experts = [], []
    for i in range(steps):
        out = step(labels=ys[i], slot=i)
        step.wait()
        got.append({k: v.clone() for k, v in out.items() if k != "experts"})
        experts.append([{k: v.clone() for k, v in o.items()} for o in out["experts"]])
    torch.cuda.synchronize()
    ref_acc = R.new_acc(K)
    for k, net in enumerate(nets):
        lone = mc.MCForward(net, xs[0], S, want_uncertainty=True, seed=21, static_inputs=xs, first_replay=3)
        for i in range(steps):
            o = lone(slot=i)
            torch.cuda.synchronize()
            for name in o:
                assert torch.equal(experts[i][k][name], o[name]), (case, k, i, name)
    for i in range(steps):
        planes = _np(experts[i])
        _check_against_ref(planes, "epistemic", got[i], (case, i))
        R.accumulate(ref_acc, planes, "epistemic", ys[i].cpu().numpy())
    _check_acc(acc, ref_acc, K, case)
    entries = log.read()
    assert torch.equal(entries["expert"], torch.cat([r["expert"] for r in got])), case
    assert torch.equal(entries["local"], torch.cat([r["local_pred"] for r in got])), case
    assert torch.equal(entries["pred"], torch.cat([r["pred"] for r in got])), case
    assert torch.equal(entries["scores"], torch.cat([r["scores"] for r in got])), case


def _planes(B, K, C, dev, seed):
    g = torch.Generator().manual_seed(seed)
    outs = []
    for _ in range(K):
        lo = torch.log_softmax(torch.randn(B, C, generator=g) * 2, dim=1)
        outs.append({"pred": torch.randn(B, C, generator=g), "epistemic": torch.rand(B, C, generator=g) * 1e-2,
                     "aleatoric": torch.rand(B, C, generator=g) * 1e-1, "log_outputs": lo,
                     "mutual_info": torch.rand(B, generator=g) * 1e-2})
    # planted cases: an exact tie of every expert (goes to K - 1), a tie of 0 and 1 only, NaN scores, argmax ties
    for o in outs:
        o["epistemic"][0] = 1e-3
        o["aleatoric"][0] = 1e-2
        o["log_outputs"][0] = outs[0]["log_outputs"][0]
        o["mutual_info"][0] = 5e-3
    for name, shift in (("epistemic", -1.0), ("aleatoric", -1.0), ("log_outputs", 5.0)):
        outs[0][name][1] = outs[0][name][1] + shift        # 0 and 1 tie ahead of every other expert
        outs[1][name][1] = outs[0][name][1]
    outs[0]["mutual_info"][1] = outs[1]["mutual_info"][1] = -1.0
    for name in ("epistemic", "aleatoric", "log_outputs"):
        outs[K - 1][name][2, 0] = float("nan")             # NaN score of the last expert: never chosen
        for o in outs:
            o[name][3, 1] = float("nan")                   # every score NaN: K - 1
    outs[K - 1]["mutual_info"][2] = float("nan")
    for o in outs:
        o["mutual_info"][3] = float("nan")
        o["pred"][4] = 0.5                                 # every class tied: the first
        o["pred"][5] = float("nan")                        # no maximal class: 0
    return [{k: v.contiguous().to(dev) for k, v in o.items()} for o in outs]


@pytest.mark.parametrize("score", ["epistemic", "aleatoric", "both", "mutual_info", "confidence"])
@pytest.mark.parametrize("K,C,B", [(2, 5, 256), (5, 2, 7), (16, 10, 1030), (3, 40, 33)])
def test_kernel_ties_nan_and_labels(dev, score, K, C, B):
    """route_batch on planted planes: ties to the highest index, NaN never chosen, argmax ties and NaN rows; global
    labels with an out-of-range one, task labels, and task given against labels that are already global."""
    from pytorch_bayesiancnn_b200 import mc
    outs = _planes(B, K, C, dev, seed=K * 100 + C)
    planes = _np(outs)
    g = torch.Generator().manual_seed(B)
    lab = torch.randint(0, K * C, (B,), generator=g)
    lab[min(6, B - 1)] = K * C                                # outside every range
    local = torch.randint(0, C, (B,), generator=g)
    offsets = [3 * e * C + 1 for e in range(K)]               # gaps between the ranges
    for labels, task, offs in ((lab, None, None), (local, K - 1, None), (lab, 1, None),
                               (torch.tensor([offsets[b % K] + b % C for b in range(B)]), None, offsets)):
        acc = mc.new_route_metrics(dev)
        log = mc.RouteLog(dev, 2 * B - 1, K)                 # the second launch overflows by one image
        res = [mc.route_batch(outs, score, offs, labels.to(dev), task, acc, log) for _ in range(2)]
        torch.cuda.synchronize()
        tag = (score, K, C, B, task, offs is not None)
        for r in res:
            e, lc, pr, S = R.route(planes, score, offs)
            _check_against_ref(planes, score, r, tag, offs)
            # the class sums run in the same order on both sides: planted ties are exact ties there too
            assert np.array_equal(r["expert"].cpu().numpy(), e), tag
            assert r["expert"][0].item() == K - 1 and r["expert"][1].item() == 1, tag
            assert r["expert"][3].item() == K - 1, tag
            if B > 5:
                assert r["local"][5].item() == 0, tag
        ref = R.new_acc(K)
        for _ in range(2):
            R.accumulate(ref, planes, score, labels.numpy(), -1 if task is None else task, offs)
        _check_acc(acc, ref, K, tag)
        assert log._cursor.tolist() == [2 * B, 1] and len(log) == 2 * B - 1
        with pytest.raises(Exception, match="did not fit"):
            log.read()
        assert torch.equal(log._ints[0, :B], res[0]["expert"]), tag
        assert torch.equal(log._scores[B:2 * B - 1].view(torch.int32), res[1]["scores"][:B - 1].view(torch.int32)), tag


def _loader(n, B, seed, K, C):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(B, 1, 32, 32, generator=g), torch.randint(0, K * C, (B,), generator=g)) for _ in range(n)]


def test_ordering_per_batch_and_route_in_flight(dev):
    """Distinct batches: per-batch ExpertStep calls and mc.route with inflight 1 and 4 give the same per-image log and
    accumulator bits -- no exchange overwrites planes a routing still reads -- and the figures are route_ref's."""
    from pytorch_bayesiancnn_b200 import mc
    K, C, B, S, n = 2, 5, 256, 10, 8
    nets = _experts("lenet", K, C, 1, "lrt", dev, seed0=300)
    batches = _loader(n, B, 9, K, C)
    acc = mc.new_route_metrics(dev)
    log = mc.RouteLog(dev, n * B, K)
    slots = [torch.zeros(B, 1, 32, 32, device=dev) for _ in range(2)]
    step = mc.ExpertStep(nets, slots[0], S, seed=5, static_inputs=slots, metrics=acc, log=log)
    ref = R.new_acc(K)
    for x, y in batches:
        out = step(x.to(dev), y.to(dev))
        step.wait()
        planes = _np([{k: v.clone() for k, v in o.items()} for o in out["experts"]])
        torch.cuda.synchronize()
        R.accumulate(ref, planes, "epistemic", y.numpy())
    torch.cuda.synchronize()
    _check_acc(acc, ref, K, "per-batch")
    per_batch = log.read()
    figures = mc.read_route_metrics(acc, K)
    for inflight in (1, 4):
        res = mc.route(nets, batches, S, inflight=inflight, seed=5)
        for k in ("expert", "pred", "scores"):
            assert torch.equal(res["per_image"][k], per_batch[k]), (inflight, k)
        for k in ("steps", "images", "accuracy", "local_accuracy", "routing_accuracy", "selected", "total_score"):
            assert res[k] == figures[k], (inflight, k)          # read from accumulators of the same bits
    # the next call rebuilds nothing (and draws fresh noise)
    cache = nets[0].__dict__["_mc_route"]
    steps_before = [id(e["eng"]) for ent in cache.values() for e in ent["engines"].values()]
    again = mc.route(nets, batches, S, inflight=4, seed=5)
    assert [id(e["eng"]) for ent in cache.values() for e in ent["engines"].values()] == steps_before
    assert again["images"] == n * B and not torch.equal(again["per_image"]["scores"], per_batch["scores"])
    assert figures["local_accuracy"] == pytest.approx(ref["sum_local_acc"] / n, rel=1e-12)


@pytest.mark.parametrize("score,normalized", [(s, False) for s in R.SCORES] + [("epistemic", True)])
def test_every_score_with_and_without_log(dev, score, normalized):
    """Each score kind (and softplus-normalised p_hat) runs; a step with a log gives the outputs of one without."""
    from pytorch_bayesiancnn_b200 import mc
    K, C, B, S, steps = 2, 5, 128, 4, 3
    nets = _experts("lenet", K, C, 1, "lrt", dev, seed0=500)
    g = torch.Generator().manual_seed(3)
    xs = [torch.randn(B, 1, 32, 32, generator=g).to(dev) for _ in range(steps)]
    ys = [torch.randint(0, K * C, (B,), generator=g).to(dev) for _ in range(steps)]
    log = mc.RouteLog(dev, steps * B, K)
    a = mc.ExpertStep(nets, xs[0], S, score=score, normalized=normalized, seed=8, static_inputs=xs, log=log,
                      metrics=mc.new_route_metrics(dev), inflight=2)
    b = mc.ExpertStep(nets, xs[0], S, score=score, normalized=normalized, seed=8, static_inputs=xs)
    if score == "mutual_info":
        assert "mutual_info" in a.engines[0].out
    for i in range(steps):
        # one after the other: two engines over the same layers share their workspaces, as two MCForwards do
        oa = a(labels=ys[i], slot=i)
        a.wait()
        ob = b(slot=i)
        b.wait()
        torch.cuda.synchronize()
        for k in ("expert", "pred", "local_pred", "scores"):
            assert torch.equal(oa[k], ob[k]), (score, i, k)
        for ea, eb in zip(oa["experts"], ob["experts"]):
            for k in eb:
                assert torch.equal(ea[k], eb[k]), (score, i, k)
        _check_against_ref(_np(oa["experts"]), score, oa, (score, i))
    assert len(log) == steps * B


def test_refusals_on_the_device(dev):
    from pytorch_bayesiancnn_b200 import EngineError, mc
    nets = _experts("lenet", 2, 5, 1, "lrt", dev)
    x = torch.zeros(128, 1, 32, 32, device=dev)
    with pytest.raises(EngineError, match="different numbers of classes"):
        mc.ExpertStep(nets + _experts("lenet", 1, 4, 1, "lrt", dev), x, 2)
    with pytest.raises(EngineError, match="one device"):
        mc.ExpertStep(nets + [_experts("lenet", 1, 5, 1, "lrt", torch.device("cpu"))[0]], x, 2)
    with pytest.raises(EngineError, match="the log holds"):
        mc.ExpertStep(nets, x, 2, log=mc.RouteLog(dev, 8, 3))
    step = mc.ExpertStep(nets, x, 2)
    with pytest.raises(ValueError, match="task"):
        step(x, torch.zeros(128, dtype=torch.int64, device=dev), task=2)
    with pytest.raises(ValueError, match="outside every expert's class range"):
        mc.route(nets, [(x.cpu(), torch.full((128,), 10))], 2)
    with pytest.raises(ValueError, match="outside every expert's class range"):
        mc.route(nets, [(x.cpu(), torch.full((128,), 5))], 2, task=0)      # global labels given as task 0's
    with pytest.raises(EngineError, match="no 'mutual_info' plane"):
        mc.route_batch([e.out for e in step.engines], "mutual_info")

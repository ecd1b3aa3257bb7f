"""Active-learning selection on the GPU: the probability bank kernel (bbb_mc_prob_log) against float64, MCForward(prob_bank=...)
in every mode, bbb_joint_entropy against float64 (tests/batchbald_ref.py) over its accepted range, and the greedy
selection (mc.batchbald / mc.bald / mc.acquire) against the float64 greedy on its own trace."""
import numpy as np
import pytest
import torch

from tests import batchbald_ref as R
from tests.test_gpu_mc import _net

pytestmark = pytest.mark.gpu
TF32_REL = 2.0 ** -11


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _is_tf32(t):
    return bool(((t.contiguous().view(torch.int32) & 0x1FFF) == 0).all())


def _ref_probs(logits, normalized):
    """float64 p_hat [S, B, C] of fp32 logits [S, B, C]."""
    l64 = logits.double()
    if normalized:
        sp = torch.nn.functional.softplus(l64)
        return sp / sp.sum(2, keepdim=True)
    return torch.softmax(l64, 2)


# --------------------------------------------------------------------------- #
# the bank kernel
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("normalized", [False, True])
@pytest.mark.parametrize("S,B,C", [(1, 3, 2), (7, 33, 10), (100, 64, 10), (33, 5, 100), (256, 4, 128)])
def test_prob_log_matches_float64(dev, S, B, C, normalized):
    from pytorch_bayesiancnn_b200 import mc
    g = torch.Generator().manual_seed(S * 1000 + C)
    logits = (torch.randn(S, B, C, generator=g) * 4).to(dev)
    logits[0, 0, :] = -200.0                                   # probabilities that underflow to 0 beside the max
    logits[0, 0, 0] = 50.0
    bank = mc.ProbBank(dev, B + 3, S, C)
    bank.append(logits.contiguous(), normalized)
    torch.cuda.synchronize()
    assert len(bank) == B and bank.dropped == 0
    got = bank.read()
    ref = _ref_probs(logits, normalized).permute(1, 0, 2)     # [B, S, C]
    p = got["probs"].double()
    assert _is_tf32(got["probs"])
    tol = ref.abs() * (TF32_REL + 4 * 2.0 ** -24) + 1e-38
    assert bool(((p - ref).abs() <= tol).all()), float(((p - ref).abs() / tol).max())
    # padding and the entries past the cursor are exactly 0
    raw = bank._probs
    assert bool((raw[:, C:, :] == 0).all()) and bool((raw[:, :, S:] == 0).all()) and bool((raw[B:] == 0).all())
    h = -(torch.special.xlogy(ref, ref)).sum(2).mean(1)
    assert torch.allclose(got["expected_entropy"], h, rtol=1e-5, atol=1e-6)


def test_prob_log_cursor_overflow_and_reset(dev):
    from pytorch_bayesiancnn_b200 import EngineError, mc
    S, C = 5, 10
    bank = mc.ProbBank(dev, 100, S, C)
    chunks = [torch.randn(S, b, C, device=dev) for b in (30, 7, 50, 40)]
    for x in chunks:
        bank.append(x)
    torch.cuda.synchronize()
    assert len(bank) == 100 and bank.dropped == 27
    with pytest.raises(EngineError, match="27 images did not fit"):
        bank.read()
    full = torch.cat(chunks, 1)[:, :100]
    ref = _ref_probs(full, False).permute(1, 0, 2)
    p = bank._probs[:, :C, :S].transpose(1, 2).double()
    assert bool(((p - ref).abs() <= ref * 2 * TF32_REL + 1e-30).all())
    bank.reset()
    bank.append(chunks[1])
    torch.cuda.synchronize()
    assert len(bank) == 7 and bank.dropped == 0
    ref1 = _ref_probs(chunks[1], False).permute(1, 0, 2)
    p1 = bank.read()["probs"].double()
    assert bool(((p1 - ref1).abs() <= ref1 * 2 * TF32_REL + 1e-30).all())


# --------------------------------------------------------------------------- #
# MCForward(prob_bank=...), evaluate(prob_bank=...)
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("key,inputs", [("alexnet", 3), ("lenet", 1)])
def test_mc_forward_prob_bank_every_mode(dev, key, inputs, monkeypatch):
    """Every mode: outputs bit-identical to the engine without a bank, the bank equals the per-step logits appended in
    order (a bank filled from the serial engine's per-sample logits), warm-up steps not logged; expected_entropy
    agrees with the exchange's."""
    from pytorch_bayesiancnn_b200 import EngineError, mc
    net, _ = _net(key, 10, inputs, "lrt", dev, "auto")
    steps, B, S = 4, 128, 3
    g = torch.Generator().manual_seed(5)
    xs = [torch.randn(B, inputs, 32, 32, generator=g).to(dev) for _ in range(steps)]
    ys = [torch.randint(0, 10, (B,), generator=g).to(dev) for _ in range(steps)]
    kw = dict(with_labels=True, seed=13, want_uncertainty=True, want_information=True, static_inputs=xs)
    with pytest.raises(EngineError, match="MCTrainStep does not fill a prob_bank"):
        mc.MCTrainStep(net, xs[0], 2, 1000.0, prob_bank=mc.ProbBank(dev, 8, 2, 10))
    with pytest.raises(EngineError, match="prob_bank holds"):
        mc.MCForward(net, xs[0], S, prob_bank=mc.ProbBank(dev, 8, S + 1, 10), **kw)
    with monkeypatch.context() as mp_:
        mp_.setattr(mc, "_dist_info", lambda group: (None, 2, 0))
        with pytest.raises(EngineError, match="one rank"):
            mc.MCForward(net, xs[0], S, prob_bank=mc.ProbBank(dev, 8, S, 10), **kw)
    serial = mc.MCForward(net, xs[0], S, **kw)
    ref_bank, ref_out = mc.ProbBank(dev, steps * B, S, 10), []
    for i in range(steps):
        o = serial(labels=ys[i], slot=i)
        ref_bank.append(serial.logits_all[0].contiguous())
        ref_out.append({k: v.clone() for k, v in o.items()})
    torch.cuda.synchronize()
    expected = ref_bank.read()
    ee_ref = torch.cat([o["expected_entropy"] for o in ref_out]).double()
    assert torch.allclose(expected["expected_entropy"], ee_ref, rtol=1e-5, atol=1e-6)
    # graph=False: its own noise; the bank against the same engine's per-sample logits, step by step
    bank = mc.ProbBank(dev, steps * B, S, 10)
    eng = mc.MCForward(net, xs[0], S, prob_bank=bank, graph=False, **kw)
    plain = mc.MCForward(net, xs[0], S, graph=False, **kw)
    eager_ref = mc.ProbBank(dev, steps * B, S, 10)
    for i in range(steps):
        o, p = eng(xs[i], ys[i]), plain(xs[i], ys[i])
        eager_ref.append(plain.logits_all[0].contiguous())
        torch.cuda.synchronize()
        for k in p:
            assert torch.equal(o[k], p[k]), ("eager", k)
    got, want = bank.read(), eager_ref.read()
    assert torch.equal(got["probs"], want["probs"]) and torch.equal(got["expected_entropy"], want["expected_entropy"])
    modes = {"serial": {}, "loop": dict(fold=False), "overlap": dict(overlap=True),
             "inflight": dict(overlap=True, inflight=4)}
    for name, extra in modes.items():
        bank = mc.ProbBank(dev, steps * B, S, 10)
        eng = mc.MCForward(net, xs[0], S, prob_bank=bank, **kw, **extra)
        plain = mc.MCForward(net, xs[0], S, **kw, **extra)
        if name == "serial":
            assert (eng.fold_steps is not None) if key == "alexnet" else (eng.layer_fold is not None)
        torch.cuda.synchronize()
        assert len(bank) == 0, name                                  # the warm-up steps are not logged
        assert eng.kernels_per_step == plain.kernels_per_step + 1, name
        for e in (eng, plain):
            for i in range(steps):
                e(labels=ys[i], slot=i)
            e.wait()
        torch.cuda.synchronize()
        for k in plain.out:
            assert torch.equal(eng.out[k], plain.out[k]), (name, k)
        got = bank.read()
        assert torch.equal(got["probs"], expected["probs"]), name
        assert torch.equal(got["expected_entropy"], expected["expected_entropy"]), name


def test_evaluate_prob_bank_same_figures(dev):
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    g = torch.Generator().manual_seed(8)
    batches = [(torch.rand(b, 1, 32, 32, generator=g), torch.randint(0, 10, (b,), generator=g)) for b in (128, 128, 40)]
    bank = mc.ProbBank(dev, 296, 4, 10)
    m_bank = mc.evaluate(net, batches, 4, 60000.0, seed=21, prob_bank=bank)
    m_plain = mc.evaluate(net, batches, 4, 60000.0, seed=21)
    assert repr(m_bank) == repr(m_plain)
    assert len(bank) == 296


# --------------------------------------------------------------------------- #
# bbb_joint_entropy against float64
# --------------------------------------------------------------------------- #
def _bank_from_probs(dev, probs):
    """A ProbBank holding the float64 probabilities [N, S, C] (tf32-rounded as the kernel stores them)."""
    from pytorch_bayesiancnn_b200 import mc
    N, S, C = probs.shape
    bank = mc.ProbBank(dev, N, S, C)
    bank._probs[:N, :C, :S] = mc._tf32(probs.transpose(1, 2).to(dev))
    bank._ee[:N] = torch.as_tensor(R.expected_entropy(probs.numpy()), device=dev)
    bank._cursor[0] = N
    return bank


def _pool(N, S, C, seed):
    g = torch.Generator().manual_seed(seed)
    lo = torch.randn(N, S, C, generator=g, dtype=torch.float64) * 3
    p = torch.softmax(lo, 2)
    if N > 2:
        p[1] = 0.0
        p[1, :, C - 1] = 1.0                                        # one-hot rows
        p[2, :, : C // 2] = 0.0                                     # exact zeros
        p[2] /= p[2].sum(1, keepdim=True)
    return p


def _configs(M, S, seed):
    g = torch.Generator().manual_seed(seed)
    w = torch.rand(M, S, generator=g, dtype=torch.float64) ** 4
    if M > 1 and S > 1:
        w[0] = 0.0
        w[0, 0] = 1.0                                               # a one-hot column
    pt = w / w.sum(1, keepdim=True)
    om = torch.rand(M, generator=g, dtype=torch.float64)
    return pt, om / om.sum()


def _run_joint(dev, bank, pt64, om, mask=None):
    from pytorch_bayesiancnn_b200 import mc
    n = len(bank)
    sc = mc._Scorer(bank, n, pt64.shape[0])
    if mask is not None:
        sc.mask.copy_(mask)
    out = sc(pt64.to(dev), om.to(dev)).clone()
    return out, sc.pt[:pt64.shape[0], :bank.num_ens].double().cpu()


GRID = [(1, 2, 1, 1), (7, 10, 63, 333), (8, 16, 64, 129), (100, 10, 65, 1000), (256, 128, 63, 37),
        (100, 100, 64, 70), (20, 100, 1000, 300), (8, 2, 10000, 65), (100, 10, 10000, 257), (7, 128, 65, 3),
        (256, 2, 64, 4099), (1, 16, 1, 2000),
        # S_pad = 216: the last two-stage ring; 224 and 256: one stage refilled every Pt tile, over many tiles
        (209, 16, 200, 50), (217, 10, 1000, 100), (256, 10, 10000, 300)]


@pytest.mark.parametrize("S,C,M,N", GRID)
def test_joint_entropy_against_float64(dev, S, C, M, N):
    probs = _pool(N, S, C, seed=S + C + M + N)
    bank = _bank_from_probs(dev, probs)
    pt64, om = _configs(M, S, seed=M)
    mask = torch.zeros(N, dtype=torch.uint8)
    mask[::7] = 1
    out, pt_stored = _run_joint(dev, bank, pt64, om, mask.to(dev))
    out2, _ = _run_joint(dev, bank, pt64, om, mask.to(dev))
    assert torch.equal(out.view(torch.int64), out2.view(torch.int64))    # same inputs, same bits
    out = out.cpu().numpy()
    stored = bank._probs[:N, :C, :S].transpose(1, 2).double().cpu().numpy()
    S_pad = bank.S_pad
    eps_acc = (S_pad + 2) * 2.0 ** -23
    omn = om.numpy()
    h_t = R.h_m(stored, pt_stored.numpy())                            # tight: the stored (tf32) operands
    h_l = R.h_m(probs.numpy(), pt64.numpy())                          # loose: the unrounded ones
    tight = h_t @ omn
    bound_t = (eps_acc * (1.0 + h_t) + 2.0 ** -20) @ omn
    loose = h_l @ omn
    bound_l = ((eps_acc + 2 * TF32_REL) * (1.0 + h_l) + 2.0 ** -20) @ omn
    m = mask.numpy().astype(bool)
    assert np.isneginf(out[m]).all()
    assert (np.abs(out[~m] - tight[~m]) <= bound_t[~m]).all(), float((np.abs(out - tight) / bound_t)[~m].max())
    assert (np.abs(out[~m] - loose[~m]) <= bound_l[~m]).all(), float((np.abs(out - loose) / bound_l)[~m].max())


def test_joint_entropy_refuses_out_of_range(dev):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    lib = L.lib()
    buf = torch.zeros(1 << 16, device=dev)
    out = torch.zeros(16, dtype=torch.float64, device=dev)
    om = torch.ones(16, dtype=torch.float64, device=dev)
    for N, S, C, M in ((0, 8, 10, 1), (1, 0, 10, 1), (1, 257, 10, 1), (1, 8, 1, 1), (1, 8, 129, 1), (1, 8, 10, 0),
                       (1, 8, 10, (1 << 20) + 1)):
        rc = lib.bbb_joint_entropy(Fn._ptr(buf), Fn._ptr(om), None, Fn._ptr(buf), N, S, C, M, Fn._ptr(out), None, 0,
                                   Fn._stream(dev))
        assert rc == -1, (N, S, C, M)
    assert lib.bbb_joint_entropy_workspace_bytes(60000, 100, 10, 10000) == 0


# --------------------------------------------------------------------------- #
# greedy selection against the float64 greedy, on the device's own trace
# --------------------------------------------------------------------------- #
def _check_trace(dev, bank, probs, res):
    """Every round: every candidate's score within the loose bound of the float64 score on the same configurations, and
    the pick the float64 argmax or within twice the bound of it."""
    stored = bank._probs[:len(bank), :bank.num_classes, :bank.num_ens].transpose(1, 2).double().cpu().numpy()
    eh = bank._ee[:len(bank)].cpu().numpy()
    p = probs.numpy()
    S_pad = bank.S_pad
    chosen = []
    for r, tr in enumerate(res["trace"]):
        if tr["exact"]:
            pt, om, const, cfg = R.exact_configs(stored, chosen)
            assert np.array_equal(cfg, tr["configs"].cpu().numpy()), r
        else:
            pt, om, const = R.sampled_configs(stored, chosen, tr["configs"].cpu().numpy())
        assert abs(float(tr["const"]) - const) <= 1e-9 * max(1.0, abs(const)), (r, float(tr["const"]), const)
        assert np.allclose(tr["omega"].cpu().numpy(), om, rtol=1e-12, atol=0)
        a_ref, h = R.scores(p, pt, om, const, chosen, eh)
        bound = ((S_pad + 2) * 2.0 ** -23 + 2 * TF32_REL) * ((1.0 + h) @ om) + 2.0 ** -20 + 1e-12
        got = tr["scores"].cpu().numpy()
        live = ~np.isneginf(a_ref)
        assert np.isneginf(got[~live]).all()
        assert (np.abs(got[live] - a_ref[live]) <= bound[live]).all(), (r, float((np.abs(got - a_ref) / bound)[live].max()))
        pick = int(res["indices"][r])
        assert pick == int(np.argmax(a_ref)) or a_ref[pick] >= a_ref.max() - 2 * bound.max(), r
        assert float(res["scores"][r]) == got[pick]
        chosen.append(pick)
    return chosen


@pytest.mark.parametrize("N,S,C,k,num_configs", [(300, 20, 10, 4, 1000), (200, 8, 3, 8, 100), (120, 100, 100, 3, 1000)])
def test_batchbald_against_float64_trace(dev, N, S, C, k, num_configs):
    from pytorch_bayesiancnn_b200 import mc
    probs = _pool(N, S, C, seed=N + k)
    bank = _bank_from_probs(dev, probs)
    res = mc.batchbald(bank, k, num_configs=num_configs, seed=3, trace=True)
    assert res["exact"] == [e for _, e in mc.batchbald_plan(C, k, num_configs)]
    assert (not all(res["exact"])) or C ** (k - 1) <= num_configs
    chosen = _check_trace(dev, bank, probs, res)
    assert len(set(chosen)) == k
    again = mc.batchbald(bank, k, num_configs=num_configs, seed=3)
    assert torch.equal(again["indices"], res["indices"])
    assert torch.equal(again["scores"].view(torch.int64), res["scores"].view(torch.int64))
    # round 0 is BALD: the first pick and score are mc.bald's, and the bank's mutual information
    b = mc.bald(bank, k)
    assert int(b["indices"][0]) == int(res["indices"][0]) and float(b["scores"][0]) == float(res["scores"][0])
    pbar = probs.mean(1)
    mi = -(torch.special.xlogy(pbar, pbar)).sum(1) - torch.as_tensor(R.expected_entropy(probs.numpy()))
    # (the bank holds tf32 probabilities: the loose bound of the unrounded pool)
    assert abs(float(b["scores"][0]) - float(mi.max())) <= 2 * TF32_REL * (1.0 + float(mi.max())) + 1e-5
    assert torch.equal(b["indices"], torch.topk(res["trace"][0]["scores"].cpu(), k).indices)


def test_batchbald_first_sampled_round_memory_is_linear(dev):
    """C = 100 with the default num_configs: round 3 is the first sampled one, drawing 10^4 configurations from the
    exact joint over 10^4 x 100 outcomes.  The update holds O(M S C) words (an [M, M_prev C] cumulative sum would be
    80 GB); the trace still matches float64."""
    from pytorch_bayesiancnn_b200 import mc
    probs = _pool(30, 8, 100, seed=9)
    bank = _bank_from_probs(dev, probs)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    res = mc.batchbald(bank, 4, num_configs=10000, seed=2)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev) - before
    assert res["exact"] == [True, True, True, False]
    assert peak < 64 << 20, peak
    res = mc.batchbald(bank, 4, num_configs=10000, seed=2, trace=True)
    _check_trace(dev, bank, probs, res)


def test_batchbald_repeated_pool_follows_float64_greedy(dev):
    """Every image three times: BALD's top-k takes copies, BatchBALD follows the float64 greedy and never takes a copy
    of an image it holds while a distinct one is worth more."""
    from pytorch_bayesiancnn_b200 import mc
    base = _pool(40, 16, 4, seed=7)
    probs = torch.cat([base, base, base])
    bank = _bank_from_probs(dev, probs)
    res = mc.batchbald(bank, 4, num_configs=10000, seed=1, trace=True)
    _check_trace(dev, bank, probs, res)
    ref_idx, _ = R.greedy_exact(bank._probs[:120, :4, :16].transpose(1, 2).double().cpu().numpy(), 4)
    assert len({i % 40 for i in res["indices"].tolist()}) == 4
    assert [i % 40 for i in res["indices"].tolist()] == [i % 40 for i in ref_idx]
    top = mc.bald(bank, 3)["indices"].tolist()
    assert len({i % 40 for i in top}) == 1                          # the three copies of the same image


def test_batchbald_enqueues_without_host_sync(dev):
    from pytorch_bayesiancnn_b200 import mc
    bank = _bank_from_probs(dev, _pool(500, 10, 10, seed=4))
    n = len(bank)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        picks, scores, plan, _ = mc._batchbald_rounds(bank, n, 5, 100, 7, False)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert not all(e for _, e in plan)
    assert len(set(picks.tolist())) == 5 and torch.isfinite(scores).all()


def test_acquire_end_to_end(dev):
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    g = torch.Generator().manual_seed(2)
    pool = [(torch.rand(b, 1, 32, 32, generator=g), torch.randint(0, 10, (b,), generator=g)) for b in (128, 128, 44)]
    for method in ("bald", "batchbald"):
        res = mc.acquire(net, pool, 5, 8, method=method, num_configs=1000, seed=3)
        bank = net.__dict__["_al_bank"]
        assert len(bank) == 300
        assert len(set(res["indices"].tolist())) == 5 and res["evaluate"]["images"] == 300
        m = mc.evaluate(net, pool, 8, 1.0, seed=3)
        assert repr(m) == repr(res["evaluate"])
        ref = mc.bald(bank, 5) if method == "bald" else mc.batchbald(bank, 5, num_configs=1000, seed=3)
        assert torch.equal(ref["indices"], res["indices"]), method

"""Vector scaling on the GPU: the apply kernel (bbb_mc_logit_scale) against torch's z * a + b bit for bit, the scaled
Monte-Carlo step in every mode against the unscaled engine (the identity), float64 (tests/mc_head_ref.py) and itself,
the fit pass (bbb_scaling_nll_grad) against float64 (tests/scaling_ref.py) within its derived bound, the device fit, and
calibrate_scaling end to end."""
import numpy as np
import pytest
import torch

from tests import mc_head_ref as H
from tests import scaling_ref as R
from tests import temperature_ref as TR
from tests.test_gpu_mc import _net
from tests.test_scaling_cpu import planted

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _scaling(dev, C, seed, identity=False, kind="vector"):
    from pytorch_bayesiancnn_b200 import mc
    s = mc.LogitScaling(dev, C, kind)
    if not identity:
        g = torch.Generator().manual_seed(seed)
        with torch.no_grad():
            if kind == "matrix":
                s.W.copy_(torch.diag(torch.rand(C, generator=g) * 1.5 + 0.25) + torch.randn(C, C, generator=g) * 0.1)
            else:
                s.a.copy_(torch.rand(C, generator=g) * 1.5 + 0.25)
            s.b.copy_(torch.randn(C, generator=g))
    return s


def _mapped(sc, z):
    """f(z) with the bits the step computes: torch's z * a + b (vector), the apply kernel itself (matrix, whose result
    test_matrix_apply_within_bound checks against float64)."""
    if sc.kind == "vector":
        return z * sc.a + sc.b
    out = z.contiguous().clone()
    sc.apply_(out)
    torch.cuda.synchronize()
    return out


# --------------------------------------------------------------------------- #
# the apply kernel
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("rows,C,offset", [(1, 2, 0), (3, 10, 1), (7, 3, 3), (1000, 10, 0), (512 * 10, 10, 2),
                                           (1024 * 25, 100, 1), (33, 1000, 3), (5, 1024, 0), (300000, 7, 1)])
def test_apply_is_torch_mul_add(dev, rows, C, offset):
    g = torch.Generator().manual_seed(rows + C)
    n = rows * C
    base = (torch.randn(n + offset, generator=g) * torch.logspace(-3, 3, n + offset)).to(dev)
    for identity in (True, False):
        s = _scaling(dev, C, rows, identity)
        z = base.clone()
        view = z[offset:].view(rows, C)                           # a start that is not 16-byte aligned
        s.apply_(view)
        want = base[offset:].view(rows, C) * s.a + s.b
        torch.cuda.synchronize()
        assert torch.equal(view.reshape(-1).view(torch.int32), want.reshape(-1).view(torch.int32)), (identity, C)
        assert torch.equal(z[:offset], base[:offset])


@pytest.mark.parametrize("rows,C,offset", [(1, 2, 0), (3, 10, 1), (7, 3, 3), (1000, 10, 0), (512 * 10, 10, 2),
                                           (1024 * 25, 100, 1), (33, 128, 3), (300000, 7, 1)])
def test_matrix_apply_within_bound(dev, rows, C, offset):
    """W z + b within the fmaf chain's bound of float64; the identity gives the input's bits; the same bits every
    run."""
    g = torch.Generator().manual_seed(rows + C)
    n = rows * C
    base = (torch.randn(n + offset, generator=g) * 3).to(dev)
    for identity in (True, False):
        s = _scaling(dev, C, rows, identity, "matrix")
        z = base.clone()
        view = z[offset:].view(rows, C)
        s.apply_(view)
        again = base.clone()
        s.apply_(again[offset:].view(rows, C))
        torch.cuda.synchronize()
        assert torch.equal(z, again) and torch.equal(z[:offset], base[:offset])
        if identity:
            assert torch.equal(view.reshape(-1), base[offset:]), C
            continue
        x = base[offset:].view(rows, C).cpu().numpy()
        W, b = s.W.cpu().numpy(), s.b.cpu().numpy()
        err = np.abs(view.cpu().numpy().astype(np.float64) - R.apply_matrix(x, W, b))
        bnd = R.apply_bound(x, W, b)
        assert bool((err <= bnd).all()), float((err / bnd).max())


# --------------------------------------------------------------------------- #
# the scaled step
# --------------------------------------------------------------------------- #
def _case(key, inputs, variant, dev, steps=3, B=128):
    net, _ = _net(key, 10, inputs, variant, dev, "auto")
    g = torch.Generator().manual_seed(5)
    xs = [torch.randn(B, inputs, 32, 32, generator=g).to(dev) for _ in range(steps)]
    ys = [torch.randint(0, 10, (B,), generator=g).to(dev) for _ in range(steps)]
    return net, xs, ys


def _logs(dev, n, S):
    from pytorch_bayesiancnn_b200 import mc
    return dict(logit_bank=mc.LogitBank(dev, n, S, 10), score_log=mc.ScoreLog(dev, n),
                prob_bank=mc.ProbBank(dev, n, S, 10), conformal=mc.ConformalLog(dev, n, 10, seed=17))


def _bits(t):
    """A tensor's bits, so that NaNs compare equal to the same NaNs."""
    return t.view({8: torch.int64, 4: torch.int32}[t.element_size()]) if t.is_floating_point() else t


def _log_tensors(logs):
    return {(name, k): v.clone() for name, lg in logs.items() for k, v in vars(lg).items() if torch.is_tensor(v)}


def _steps(eng, xs, ys, eager):
    outs = []
    for i in range(len(xs)):
        o = eng(xs[i], ys[i]) if eager else eng(labels=ys[i], slot=i)
        if not eng.overlap:
            outs.append({k: v.clone() for k, v in o.items()})
    eng.wait()
    torch.cuda.synchronize()
    return outs


MODES = {"eager": dict(graph=False), "serial": {}, "overlap": dict(overlap=True),
         "inflight": dict(overlap=True, inflight=4)}


@pytest.mark.parametrize("kind", ["vector", "matrix"])
@pytest.mark.parametrize("key,inputs,variant", [("alexnet", 3, "lrt"), ("lenet", 1, "lrt"), ("alexnet", 3, "bbb")])
def test_identity_scaling_every_mode(dev, key, inputs, variant, kind):
    """The identity map gives every output's and every log's untransformed bits, in every mode, with every log
    attached; the logit bank holds the raw logits either way."""
    from pytorch_bayesiancnn_b200 import mc
    net, xs, ys = _case(key, inputs, variant, dev)
    steps, B, S = len(xs), xs[0].shape[0], 3
    kw = dict(with_labels=True, seed=13, want_uncertainty=True, want_information=True, static_inputs=xs)
    for name, extra in MODES.items():
        eager = name == "eager"
        got = {}
        for scaled in (False, True):
            logs = _logs(dev, steps * B, S)
            sc = mc.LogitScaling(dev, 10, kind) if scaled else None
            eng = mc.MCForward(net, xs[0], S, scaling=sc, **logs, **kw, **extra)
            if variant == "lrt" and name == "serial":
                assert (eng.fold_steps is not None) if key == "alexnet" else (eng.layer_fold is not None)
            for lg in logs.values():
                lg.reset()
            outs = _steps(eng, xs, ys, eager)
            got[scaled] = (outs, {k: v.clone() for k, v in eng.out.items()}, _log_tensors(logs), eng.kernels_per_step)
        (o0, last0, l0, k0), (o1, last1, l1, k1) = got[False], got[True]
        if k0 is not None:
            assert k1 == k0 + 1, name
        for a, b in zip(o1, o0):
            for k in b:
                assert torch.equal(a[k], b[k]), (name, k)
        for k in last0:
            assert torch.equal(last1[k], last0[k]), (name, k)
        for k in l0:
            assert torch.equal(_bits(l1[k]), _bits(l0[k])), (name, k)


@pytest.mark.parametrize("kind", ["vector", "matrix"])
@pytest.mark.parametrize("key,inputs,variant", [("alexnet", 3, "lrt"), ("lenet", 1, "lrt"), ("alexnet", 3, "bbb")])
def test_scaled_step_every_mode(dev, key, inputs, variant, kind):
    """A non-identity map: every output within the float64 head's per-element bounds on f(bank) = bank * a + b, the
    same bits in every mode, the logit bank the raw logits and a ProbBank behind the map ProbBank.append(f(bank))."""
    from pytorch_bayesiancnn_b200 import mc
    net, xs, ys = _case(key, inputs, variant, dev)
    steps, B, S = len(xs), xs[0].shape[0], 3
    kw = dict(with_labels=True, seed=13, want_uncertainty=True, want_information=True, static_inputs=xs)
    plain = mc.MCForward(net, xs[0], S, **kw)
    raw = []
    for i in range(steps):
        plain(labels=ys[i], slot=i)
        raw.append(plain.logits_all[0].clone())
    torch.cuda.synchronize()
    raw_bank = torch.cat(raw, 1).permute(1, 0, 2)                  # [steps * B, S, C]
    sc = _scaling(dev, 10, 3, kind=kind)
    mapped = _mapped(sc, raw_bank)
    serial = mc.MCForward(net, xs[0], S, scaling=sc, **kw)
    want = _steps(serial, xs, ys, False)
    for i, o in enumerate(want):
        z = mapped[i * B:(i + 1) * B].permute(1, 0, 2).contiguous()
        ref = H.head(z.cpu(), ys[i].cpu(), [0.0])
        bnd = H.bounds(z.cpu(), ys[i].cpu(), [0.0], S, 1, ref=ref)
        for k, rk in (("log_outputs", "lo"), ("pred", "pred"), ("epistemic", "epi"), ("aleatoric", "ale"),
                      ("entropy", "ent"), ("expected_entropy", "ee"), ("mutual_info", "mi")):
            err = (o[k].double().cpu() - ref[rk]).abs()
            assert bool((err <= bnd[rk]).all()), (k, float((err / bnd[rk]).max()))
    for name, extra in MODES.items():
        bank = mc.LogitBank(dev, steps * B, S, 10)
        pb = mc.ProbBank(dev, steps * B, S, 10)
        eng = mc.MCForward(net, xs[0], S, scaling=sc, logit_bank=bank, prob_bank=pb, **kw, **extra)
        bank.reset()
        pb.reset()
        if name == "eager":                                         # (eager steps draw their own noise)
            plain_e = mc.MCForward(net, xs[0], S, graph=False, **kw)
            zs = []
            for i in range(steps):
                eng(xs[i], ys[i])
                plain_e(xs[i], ys[i])
                zs.append(plain_e.logits_all[0].clone())
                torch.cuda.synchronize()
                assert torch.equal(eng.logits_all[0], _mapped(sc, plain_e.logits_all[0])), name
            assert torch.equal(bank.read()["logits"], torch.cat(zs, 1).permute(1, 0, 2)), name
            continue
        _steps(eng, xs, ys, False)
        for k in eng.out:
            assert torch.equal(eng.out[k], want[-1][k]), (name, k)
        assert torch.equal(bank.read()["logits"], raw_bank), name
        ref_pb = mc.ProbBank(dev, steps * B, S, 10)
        ref_pb.append(mapped.permute(1, 0, 2).contiguous())
        torch.cuda.synchronize()
        assert torch.equal(pb.read()["probs"], ref_pb.read()["probs"]), name


def test_in_place_scaling_is_read_and_evaluate(dev):
    from pytorch_bayesiancnn_b200 import mc
    net, xs, ys = _case("lenet", 1, "lrt", dev, steps=1)
    kw = dict(with_labels=True, seed=3, static_inputs=xs)
    sc = mc.LogitScaling(dev, 10)
    other = _scaling(dev, 10, 8)
    eng = mc.MCForward(net, xs[0], 4, scaling=sc, **kw)
    ref = mc.MCForward(net, xs[0], 4, scaling=other, **kw)
    a = {k: v.clone() for k, v in eng(labels=ys[0]).items()}
    a2 = {k: v.clone() for k, v in ref(labels=ys[0]).items()}
    sc.params.copy_(other.params)                                   # read by the captured graph's next replay
    b = eng(labels=ys[0])
    c = ref(labels=ys[0])
    torch.cuda.synchronize()
    assert not torch.equal(a["log_outputs"], a2["log_outputs"])
    assert torch.equal(b["log_outputs"], c["log_outputs"]) and torch.equal(b["head"], c["head"])
    g = torch.Generator().manual_seed(8)
    batches = [(torch.rand(b_, 1, 32, 32, generator=g), torch.randint(0, 10, (b_,), generator=g)) for b_ in (64, 40)]
    sc.reset()
    m1 = mc.evaluate(net, batches, 4, 1.0, seed=21, scaling=sc)
    m_plain = mc.evaluate(net, batches, 4, 1.0, seed=21)
    assert m1["nll"] == m_plain["nll"] and m1["ece"] == m_plain["ece"]
    sc.params.copy_(other.params)
    m3 = mc.evaluate(net, batches, 4, 1.0, seed=21, scaling=sc)
    # the engines evaluate keeps for a scaling read its parameters in place; a second call draws the noise of the
    # second call of any other key
    mc.evaluate(net, batches, 4, 1.0, seed=21, scaling=other)
    m3o = mc.evaluate(net, batches, 4, 1.0, seed=21, scaling=other)
    assert m3["nll"] != m_plain["nll"] and m3["nll"] == m3o["nll"] and m3["ece"] == m3o["ece"]
    with pytest.raises(ValueError, match="not both"):
        mc.evaluate(net, batches, 4, 1.0, temperature=2.0, scaling=sc)


def test_refusals(dev):
    from pytorch_bayesiancnn_b200 import EngineError, mc
    net, xs, _ = _case("lenet", 1, "lrt", dev, steps=1, B=16)
    sc = mc.LogitScaling(dev, 10)
    with pytest.raises(EngineError, match="MCTrainStep does not scale logits"):
        mc.MCTrainStep(net, xs[0], 2, 1000.0, scaling=sc)
    with pytest.raises(ValueError, match="normalized"):
        mc.MCForward(net, xs[0], 2, normalized=True, scaling=sc)
    with pytest.raises(ValueError, match="not both"):
        mc.MCForward(net, xs[0], 2, temperature=2.0, scaling=sc)
    with pytest.raises(EngineError, match="holds 11 classes"):
        mc.MCForward(net, xs[0], 2, scaling=mc.LogitScaling(dev, 11))


def test_expert_scalings(dev):
    """Each expert of an ExpertStep maps with its own scaling: its out is that of the scaled engine alone."""
    from pytorch_bayesiancnn_b200 import mc
    a, xs, _ = _case("lenet", 1, "lrt", dev, steps=1, B=64)
    b = _net("lenet", 10, 1, "lrt", dev, "auto")[0]
    with torch.no_grad():
        for p in b.parameters():
            p.mul_(1.01)
    sa, sb = _scaling(dev, 10, 1), _scaling(dev, 10, 2)
    step = mc.ExpertStep([a, b], xs[0], 3, seed=4, static_inputs=xs, scalings=[sa, sb])
    res = step()
    step.wait()
    for net, sc, o in zip((a, b), (sa, sb), res["experts"]):
        alone = mc.MCForward(net, xs[0], 3, want_uncertainty=True, seed=4, static_inputs=xs, overlap=True, scaling=sc)
        alone()
        alone.wait()
        torch.cuda.synchronize()
        for k in ("log_outputs", "pred", "epistemic"):
            assert torch.equal(o[k], alone.out[k]), k
    with pytest.raises(ValueError, match="one per expert"):
        mc.ExpertStep([a, b], xs[0], 3, scalings=[sa])


# --------------------------------------------------------------------------- #
# the fit pass and the fit
# --------------------------------------------------------------------------- #
def _bank_of(dev, z, y, capacity=None):
    from pytorch_bayesiancnn_b200 import mc
    n, S, C = z.shape
    bank = mc.LogitBank(dev, capacity or n, S, C)
    bank.append(torch.as_tensor(z).permute(1, 0, 2).contiguous().to(dev), torch.as_tensor(y).to(dev))
    return bank


def _pass(dev, bank, a, b, mu=0.0, lam=0.0, matrix=False):
    """One bbb_scaling_nll_grad pass (no step) at a (vector) or W (matrix) and b: [J, dJ/dtheta] as float64 host
    values."""
    from pytorch_bayesiancnn_b200 import _lib as L
    from pytorch_bayesiancnn_b200 import functional as Fn
    lib = L.lib()
    C = bank.num_classes
    kind = L.SCALING_MATRIX if matrix else L.SCALING_VECTOR
    theta = torch.tensor(np.concatenate([np.ravel(a), b]), dtype=torch.float32, device=dev)
    P = theta.numel()
    state = torch.zeros(3, P, dtype=torch.float64, device=dev)
    best = torch.zeros(P, dtype=torch.float32, device=dev)
    fit = torch.full((3,), float("nan"), dtype=torch.float64, device=dev)
    res = torch.full((1 + P,), float("nan"), dtype=torch.float64, device=dev)
    nbytes = int(lib.bbb_scaling_workspace_bytes(bank.capacity, bank.num_ens, C, kind))
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    L.check(lib.bbb_scaling_nll_grad(Fn._ptr(bank._logits), Fn._ptr(bank._labels), Fn._ptr(bank._cursor),
                                     bank.capacity, bank.num_ens, C, kind, L.SCALING_FIRST,
                                     Fn._ptr(theta), Fn._ptr(state), Fn._ptr(best), Fn._ptr(fit), Fn._ptr(res), None,
                                     lam, mu, 0.0, 1.0, 1.0, Fn._ptr(ws), nbytes, Fn._stream(dev)),
            "bbb_scaling_nll_grad")
    assert bool((ws[:4] == 0).all())                                # the launch leaves its arrival counter zeroed
    assert torch.equal(best, theta)
    return res.cpu().numpy()


@pytest.mark.parametrize("n,S,C,scale", [(1, 1, 2, 1.0), (37, 2, 10, 5.0), (1000, 25, 10, 1.0), (301, 1, 10, 1e2),
                                         (130, 100, 10, 1e-3), (9, 256, 100, 3.0), (3, 25, 1000, 10.0),
                                         (2500, 2, 2, 1.0), (33, 100, 1024, 1.0)])
def test_nll_grad_against_float64(dev, n, S, C, scale):
    rng = np.random.default_rng(n * 7 + S + C)
    z = (rng.standard_normal((n, S, C)) * scale).astype(np.float32)
    y = rng.integers(0, C, n)
    bank = _bank_of(dev, z, y)
    a = rng.uniform(0.3, 2.0, C).astype(np.float32)
    b = (rng.standard_normal(C) * 0.5).astype(np.float32)
    mu = 0.25
    got = _pass(dev, bank, a, b, mu)
    assert np.array_equal(got, _pass(dev, bank, a, b, mu))          # the same bits every run
    J = R.objective(z, y, a, b, mu)
    ga, gb = R.gradient(z, y, a, b, mu)
    bJ, ba, bb = R.bound(z, y, a, b, mu)
    assert abs(got[0] - J) <= bJ, (got[0], J, bJ)
    assert bool((np.abs(got[1:1 + C] - ga) <= ba).all()), float((np.abs(got[1:1 + C] - ga) / ba).max())
    assert bool((np.abs(got[1 + C:] - gb) <= bb).all()), float((np.abs(got[1 + C:] - gb) / bb).max())


def test_nll_grad_bits_do_not_depend_on_capacity(dev):
    """Images past the cursor add nothing: a larger bank (a larger grid) gives the same bits."""
    rng = np.random.default_rng(1)
    z = rng.standard_normal((500, 10, 10)).astype(np.float32)
    y = rng.integers(0, 10, 500)
    a, b = np.full(10, 0.8, np.float32), np.linspace(-1, 1, 10).astype(np.float32)
    small = _pass(dev, _bank_of(dev, z, y), a, b)
    big = _pass(dev, _bank_of(dev, z, y, capacity=5000), a, b)
    assert np.array_equal(small, big)


@pytest.mark.parametrize("n,S,C,scale", [(1, 1, 2, 1.0), (37, 2, 10, 5.0), (1000, 25, 10, 1.0), (301, 1, 10, 10.0),
                                         (130, 100, 10, 1e-3), (9, 256, 100, 3.0), (300, 25, 100, 2.0),
                                         (2500, 2, 2, 1.0), (33, 7, 128, 1.0), (5, 3, 77, 2.0)])
def test_matrix_nll_grad_against_float64(dev, n, S, C, scale):
    """The matrix pass (tf32 wgmma forward and gradient) within the bound of float64 on the fp32 parameters."""
    rng = np.random.default_rng(n * 5 + S + C)
    z = (rng.standard_normal((n, S, C)) * scale).astype(np.float32)
    y = rng.integers(0, C, n)
    bank = _bank_of(dev, z, y)
    W = (np.diag(rng.uniform(0.3, 2.0, C)) + rng.standard_normal((C, C)) * 0.1).astype(np.float32)
    b = (rng.standard_normal(C) * 0.5).astype(np.float32)
    lam, mu = 0.5, 0.25
    got = _pass(dev, bank, W, b, mu, lam, matrix=True)
    assert np.array_equal(got, _pass(dev, bank, W, b, mu, lam, matrix=True))   # the same bits every run
    J = R.objective_m(z, y, W, b, lam, mu)
    gW, gb = R.gradient_m(z, y, W, b, lam, mu)
    bJ, bW, bb = R.bound_m(z, y, W, b, lam, mu)
    assert abs(got[0] - J) <= bJ, (got[0], J, bJ)
    eW = np.abs(got[1:1 + C * C].reshape(C, C) - gW)
    assert bool((eW <= bW).all()), float((eW / bW).max())
    eb = np.abs(got[1 + C * C:] - gb)
    assert bool((eb <= bb).all()), float((eb / bb).max())


def test_matrix_nll_grad_bits_do_not_depend_on_capacity(dev):
    rng = np.random.default_rng(2)
    z = rng.standard_normal((3000, 10, 10)).astype(np.float32)
    y = rng.integers(0, 10, 3000)
    W, b = (np.eye(10) * 0.8 + 0.02).astype(np.float32), np.linspace(-1, 1, 10).astype(np.float32)
    small = _pass(dev, _bank_of(dev, z, y), W, b, matrix=True)
    big = _pass(dev, _bank_of(dev, z, y, capacity=9000), W, b, matrix=True)
    assert np.array_equal(small, big)


def test_matrix_fit(dev):
    """The device matrix fit: never worse than its start (W = I / T from the fitted temperature), the same bits on
    every run, its objective float64's at the parameters it wrote within the bound, as good as the float64 restatement
    within 1e-3, and clearly better than vector scaling on a bank planted with off-diagonal mass; a poisoned bank
    leaves the parameters untouched."""
    from pytorch_bayesiancnn_b200 import mc
    from tests.test_scaling_cpu import planted_m
    z, y, _, _ = planted_m(4000, 4, 10, 3)
    bank = _bank_of(dev, z, y)
    lam = 0.01
    t = mc.fit_temperature(bank)
    out = mc.LogitScaling(dev, 10, "matrix")
    fit = mc.fit_scaling(bank, "matrix", l2_offdiag=lam, init_temperature=t.temperature, out=out)
    r = fit.read()
    assert fit.scaling is out and r == mc.fit_scaling(bank, "matrix", l2_offdiag=lam,
                                                      init_temperature=t.temperature).read()
    assert r["nll"] <= r["nll_start"]
    assert r["nll_start"] == pytest.approx(t.read()["nll"], abs=2e-2)        # W = I / T, on tf32 operands
    W, b = out.W.cpu().numpy(), out.b.cpu().numpy()
    assert np.array_equal(np.array(r["W"], dtype=np.float32), W) and np.array_equal(np.array(r["b"], np.float32), b)
    J = R.objective_m(z, y, W, b, lam)
    assert abs(r["nll"] - J) <= R.bound_m(z, y, W, b, lam)[0]
    ref = R.fit_m(z, y, lam=lam, T=float(t.temperature))
    assert J <= ref["nll"] + 1e-3, (J, ref["nll"])
    v = mc.fit_scaling(bank).read()
    assert R.objective_m(z, y, W, b) < v["nll"] - 0.005, (R.objective_m(z, y, W, b), v["nll"])
    before = out.params.clone()
    bank._labels[3] = 10                                            # behind the host's back
    with pytest.raises(ValueError, match=r"a label is outside \[0, 10\)"):
        mc.fit_scaling(bank, "matrix", out=out).read()
    assert torch.equal(out.params, before)


def test_fit_matches_float64_restatement(dev):
    """The device fit follows scaling_ref.fit: never worse than its start, the same objective to within the kernel's
    bound at both results, and the same bits on every run."""
    from pytorch_bayesiancnn_b200 import mc
    z, y, _, _ = planted(3000, 4, 10, 11)
    bank = _bank_of(dev, z, y)
    out = mc.LogitScaling(dev, 10)
    fit = mc.fit_scaling(bank, out=out)
    assert fit.scaling is out
    r = fit.read()
    assert r == mc.fit_scaling(bank).read()
    assert r["nll"] <= r["nll_start"] and r["iters"] == 300
    assert r["a"] == out.a.tolist() and r["b"] == out.b.tolist()
    ref = R.fit(z, y)
    J = R.objective(z, y, r["a"], r["b"])
    assert abs(r["nll"] - J) <= R.bound(z, y, r["a"], r["b"])[0]
    assert abs(J - ref["nll"]) <= 1e-4, (J, ref["nll"])
    assert r["nll_start"] == pytest.approx(TR.nll(z, y, 1.0), abs=TR.bound(z, y, 1.0) + 1e-6)


def test_fit_beats_temperature_on_planted_per_class_problem(dev):
    from pytorch_bayesiancnn_b200 import mc
    z, y, _, _ = planted(5000, 4, 10, 7, b_scale=1.5)
    bank = _bank_of(dev, z, y)
    t = mc.fit_temperature(bank)
    tr = t.read()
    r = mc.fit_scaling(bank, init_temperature=t.temperature).read()
    assert r["nll_start"] == pytest.approx(tr["nll"], abs=1e-5)      # a = 1 / T: the temperature's predictive
    assert r["nll"] < tr["nll"] - 0.01, (r["nll"], tr["nll"])
    lJ = R.lbfgs(z, y)[2]
    assert r["nll"] - lJ <= 1e-4 + R.bound(z, y, r["a"], r["b"])[0], (r["nll"], lJ)


def test_no_fit_leaves_parameters(dev):
    """An empty bank, one that dropped images, a label the host never saw go bad and non-finite logits: the scaling
    keeps its parameters and read() raises with the reason."""
    from pytorch_bayesiancnn_b200 import EngineError, mc
    S, C = 2, 10
    sc = _scaling(dev, C, 4)
    before = sc.params.clone()
    bank = mc.LogitBank(dev, 64, S, C)
    with pytest.raises(ValueError, match="no fit -- the bank is empty"):
        mc.fit_scaling(bank, iters=5, out=sc).read()
    assert torch.equal(sc.params, before)
    z = torch.randn(S, 100, C, device=dev)
    y = torch.randint(0, C, (100,), device=dev)
    bank.append(z, y)
    with pytest.raises(ValueError, match="no fit -- the bank dropped 36 images"):
        mc.fit_scaling(bank, iters=5, out=sc).read()
    assert torch.equal(sc.params, before)
    good = mc.LogitBank(dev, 100, S, C)
    good.append(z, y)
    good._labels[5] = -1                                            # behind the host's back
    with pytest.raises(ValueError, match="1 images were logged without a label"):
        mc.fit_scaling(good, iters=5, out=sc).read()
    good._labels[5] = C
    with pytest.raises(ValueError, match=r"a label is outside \[0, 10\)"):
        mc.fit_scaling(good, iters=5, out=sc).read()
    good._labels[5] = y[5]
    good._logits[7, 1, 3] = float("nan")
    with pytest.raises(ValueError, match="no finite NLL"):
        mc.fit_scaling(good, iters=5, out=sc).read()
    assert torch.equal(sc.params, before)
    good._logits[7, 1, 3] = 0.0
    r = mc.fit_scaling(good, iters=5, out=sc).read()
    assert r["nll"] <= r["nll_start"] and not torch.equal(sc.params, before)
    unl = mc.LogitBank(dev, 10, S, C)
    unl.append(z[:, :10].contiguous())
    with pytest.raises(ValueError, match="without labels"):
        mc.fit_scaling(unl)
    with pytest.raises(EngineError, match="LogitScaling of 10"):
        mc.fit_scaling(good, out=mc.LogitScaling(dev, 11))


def test_calibrate_scaling_end_to_end(dev):
    """An over-confident BBBLeNet with a class it predicts too often: the scaling started from the fitted temperature is
    no worse than it on the calibration bank, the NLL it reports is the float64 NLL of the bank at the parameters it
    wrote, within the pass's bound, and evaluate() with it runs the scaled predictive."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    last = [m for m in net.children() if hasattr(m, "W_mu")][-1]
    with torch.no_grad():
        last.W_mu.mul_(5.0)
        last.bias_mu[3] += 4.0
    g = torch.Generator().manual_seed(0)
    proto = torch.randn(10, 1, 32, 32, generator=g)

    def batches(n, seed):
        gg = torch.Generator().manual_seed(seed)
        out = []
        for _ in range(n):
            y = torch.randint(0, 10, (128,), generator=gg)
            x = proto[y] + 2.0 * torch.randn(128, 1, 32, 32, generator=gg)
            out.append((x, y))
        return out
    cal, test = batches(6, 1), batches(6, 2)
    res = mc.calibrate_scaling(net, cal, 4, init="temperature", seed=5)
    assert res["fit"]["nll"] <= res["temperature_fit"]["nll"] + 1e-6
    assert res["fit"]["nll"] < res["temperature_fit"]["nll_at_one"]
    assert len(net._temperature_banks["calibration"]) == 768
    got = net._temperature_banks["calibration"].read()
    z, y = got["logits"].cpu().numpy(), got["labels"].cpu().numpy()
    sc = res["scaling"]
    a, b = sc.a.cpu().numpy(), sc.b.cpu().numpy()
    assert res["fit"]["a"] == a.tolist() and res["fit"]["b"] == b.tolist()
    assert abs(res["fit"]["nll"] - R.objective(z, y, a, b)) <= R.bound(z, y, a, b)[0]
    # the engines evaluate keeps for the scaling run the scaled predictive (the same noise as the unscaled call)
    before = mc.evaluate(net, test, 4, 1.0, seed=9)
    scaled = mc.evaluate(net, test, 4, 1.0, seed=9, scaling=sc)
    assert scaled["nll"] != before["nll"]

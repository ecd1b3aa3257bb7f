"""Temperature scaling on the GPU: the logit bank (bbb_mc_logit_log) and the temper (bbb_mc_temper) bit for bit, the
tempered Monte-Carlo step in every mode against the untempered engine, float64 (tests/mc_head_ref.py) and itself, the
NLL kernel (bbb_temperature_nll) against float64 (tests/temperature_ref.py) within its derived bound, the device search,
and calibrate_temperature end to end."""
import math

import numpy as np
import pytest
import torch

from tests import mc_head_ref as H
from tests import temperature_ref as R
from tests.test_gpu_mc import _net

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


# --------------------------------------------------------------------------- #
# the two copy kernels
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize("n,offset", [(1, 0), (3, 1), (10, 0), (4099, 3), (512 * 100 * 10 + 7, 2), (1 << 20, 1)])
def test_temper_is_torch_division(dev, n, offset):
    from pytorch_bayesiancnn_b200 import _lib as L
    from pytorch_bayesiancnn_b200 import functional as Fn
    g = torch.Generator().manual_seed(n)
    base = (torch.randn(n + offset, generator=g) * torch.logspace(-3, 3, n + offset)).to(dev)
    for T in (1.0, 0.37, 2.5, 1e-3, 1e3):
        t = torch.tensor([T], dtype=torch.float32, device=dev)
        z = base.clone()
        view = z[offset:]                                          # a start that is not 16-byte aligned
        L.check(L.lib().bbb_mc_temper(Fn._ptr(view), n, Fn._ptr(t), Fn._stream(dev)), "bbb_mc_temper")
        want = base[offset:] / t                                   # a device tensor: true division
        torch.cuda.synchronize()
        assert torch.equal(view.view(torch.int32), want.view(torch.int32)), T
        assert torch.equal(z[:offset], base[:offset])


def test_logit_bank_append_overflow_and_reset(dev):
    from pytorch_bayesiancnn_b200 import EngineError, mc
    S, C = 3, 7
    bank = mc.LogitBank(dev, 100, S, C)
    chunks = [torch.randn(S, b, C, device=dev) for b in (30, 7, 50, 40)]
    labels = [torch.randint(0, C, (b,), device=dev) for b in (30, 7, 50, 40)]
    for z, y in zip(chunks, labels):
        bank.append(z, y)
    torch.cuda.synchronize()
    assert len(bank) == 100 and bank.dropped == 27
    with pytest.raises(EngineError, match="27 images did not fit"):
        bank.read()
    full = torch.cat(chunks, 1)[:, :100].permute(1, 0, 2)
    assert torch.equal(bank._logits, full) and torch.equal(bank._labels, torch.cat(labels)[:100])
    T = torch.full((1,), 1.7, dtype=torch.float32, device=dev)
    with pytest.raises(ValueError, match="no fit -- the bank dropped 27 images"):
        mc.fit_temperature(bank, out=T).read()                     # a bank that dropped images has no fit
    assert float(T) == pytest.approx(1.7)                          # and engines reading T keep its last value
    bank.reset()
    bank.append(chunks[1])                                         # no labels: -1, and the fit refuses the bank
    torch.cuda.synchronize()
    got = bank.read()
    assert torch.equal(got["logits"], chunks[1].permute(1, 0, 2)) and bool((got["labels"] == -1).all())
    with pytest.raises(ValueError, match="without labels"):
        mc.fit_temperature(bank)
    with pytest.raises(EngineError, match="expected contiguous float32 logits"):
        bank.append(torch.randn(S + 1, 4, C, device=dev))


# --------------------------------------------------------------------------- #
# the tempered step
# --------------------------------------------------------------------------- #
def _case(key, inputs, variant, dev, steps=3, B=128):
    net, _ = _net(key, 10, inputs, variant, dev, "auto")
    g = torch.Generator().manual_seed(5)
    xs = [torch.randn(B, inputs, 32, 32, generator=g).to(dev) for _ in range(steps)]
    ys = [torch.randint(0, 10, (B,), generator=g).to(dev) for _ in range(steps)]
    return net, xs, ys


def _run(eng, ys, steps):
    outs = []
    for i in range(steps):
        o = eng(labels=ys[i], slot=i)
        if not eng.overlap:
            outs.append({k: v.clone() for k, v in o.items()})
    eng.wait()
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("key,inputs,variant", [("alexnet", 3, "lrt"), ("lenet", 1, "lrt"), ("alexnet", 3, "bbb")])
def test_tempered_step_every_mode(dev, key, inputs, variant):
    """The bank holds the raw per-step logits in every mode; T = 1 gives the untempered bits; T = 2.5 gives the bits of
    the serial tempered engine in every mode, within the float64 bounds of the head on bank / T; a ProbBank behind the
    temper is ProbBank.append(bank / T)."""
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
    ref_plain = mc.MCForward(net, xs[0], S, **kw)
    plain_out = _run(ref_plain, ys, steps)
    # T = 1: every output is the untempered engine's
    one = mc.MCForward(net, xs[0], S, temperature=1.0, **kw)
    assert one.kernels_per_step == ref_plain.kernels_per_step + 1
    for a, b in zip(_run(one, ys, steps), plain_out):
        for k in b:
            assert torch.equal(a[k], b[k]), ("T=1", k)
    T = 2.5
    t = torch.tensor([T], dtype=torch.float32, device=dev)
    serial = mc.MCForward(net, xs[0], S, temperature=t, **kw)
    if variant == "lrt":
        assert (serial.fold_steps is not None) if key == "alexnet" else (serial.layer_fold is not None)
    want = _run(serial, ys, steps)
    tempered = (raw_bank / t)
    for i, o in enumerate(want):
        z = tempered[i * B:(i + 1) * B].permute(1, 0, 2).contiguous()
        ref = H.head(z.cpu(), ys[i].cpu(), [0.0])
        bnd = H.bounds(z.cpu(), ys[i].cpu(), [0.0], S, 1, ref=ref)
        for k, rk in (("log_outputs", "lo"), ("pred", "pred"), ("epistemic", "epi"), ("aleatoric", "ale"),
                      ("entropy", "ent"), ("expected_entropy", "ee"), ("mutual_info", "mi")):
            err = (o[k].double().cpu() - ref[rk]).abs()
            assert bool((err <= bnd[rk]).all()), (k, float((err / bnd[rk]).max()))
        assert torch.equal(o["kl"], plain_out[i]["kl"])
        assert float(o["head"][1]) != float(plain_out[i]["head"][1])
    modes = {"eager": dict(graph=False), "serial": {}, "overlap": dict(overlap=True),
             "inflight": dict(overlap=True, inflight=4)}
    for name, extra in modes.items():
        bank = mc.LogitBank(dev, steps * B, S, 10)
        pb = mc.ProbBank(dev, steps * B, S, 10)
        eng = mc.MCForward(net, xs[0], S, temperature=t, logit_bank=bank, prob_bank=pb, **kw, **extra)
        if name == "eager":
            plain_e = mc.MCForward(net, xs[0], S, graph=False, **kw)
            zs = []
            for i in range(steps):
                o = eng(xs[i], ys[i])
                plain_e(xs[i], ys[i])
                zs.append(plain_e.logits_all[0].clone())
                torch.cuda.synchronize()
                assert torch.equal(eng.logits_all[0], plain_e.logits_all[0] / t), name
            got = bank.read()
            assert torch.equal(got["logits"], torch.cat(zs, 1).permute(1, 0, 2)), name
            assert torch.equal(got["labels"], torch.cat(ys)), name
            continue
        assert len(bank) == 0 and len(pb) == 0, name               # the warm-up steps are not logged
        for i in range(steps):
            eng(labels=ys[i], slot=i)
        eng.wait()
        torch.cuda.synchronize()
        for k in eng.out:
            assert torch.equal(eng.out[k], want[-1][k]), (name, k)
        got = bank.read()
        assert torch.equal(got["logits"], raw_bank), name
        assert torch.equal(got["labels"], torch.cat(ys)), name
        ref_pb = mc.ProbBank(dev, steps * B, S, 10)
        ref_pb.append(tempered.permute(1, 0, 2).contiguous())
        torch.cuda.synchronize()
        assert torch.equal(pb.read()["probs"], ref_pb.read()["probs"]), name


def test_in_place_temperature_is_read(dev):
    from pytorch_bayesiancnn_b200 import mc
    net, xs, ys = _case("lenet", 1, "lrt", dev, steps=1)
    t = torch.tensor([1.0], dtype=torch.float32, device=dev)
    kw = dict(with_labels=True, seed=3, static_inputs=xs)
    eng = mc.MCForward(net, xs[0], 4, temperature=t, **kw)
    ref2 = mc.MCForward(net, xs[0], 4, temperature=2.0, **kw)
    a = {k: v.clone() for k, v in eng(labels=ys[0]).items()}
    a2 = {k: v.clone() for k, v in ref2(labels=ys[0]).items()}
    t.fill_(2.0)                                                   # read by the captured graph's next replay
    b = eng(labels=ys[0])
    c = ref2(labels=ys[0])                                         # the same replay index: the same noise
    torch.cuda.synchronize()
    assert not torch.equal(a["log_outputs"], a2["log_outputs"])
    assert torch.equal(b["log_outputs"], c["log_outputs"]) and torch.equal(b["head"], c["head"])
    g = torch.Generator().manual_seed(8)
    batches = [(torch.rand(b_, 1, 32, 32, generator=g), torch.randint(0, 10, (b_,), generator=g)) for b_ in (64, 40)]
    t.fill_(1.0)
    m1 = mc.evaluate(net, batches, 4, 1.0, seed=21, temperature=t)
    m_plain = mc.evaluate(net, batches, 4, 1.0, seed=21)
    assert m1["nll"] == m_plain["nll"]
    # the engines evaluate keeps for the tensor read a value written in place; a second call draws the noise of the
    # second call of any other key
    t.fill_(3.0)
    m3 = mc.evaluate(net, batches, 4, 1.0, seed=21, temperature=t)
    mc.evaluate(net, batches, 4, 1.0, seed=21, temperature=3.0)
    m3f = mc.evaluate(net, batches, 4, 1.0, seed=21, temperature=3.0)
    m_plain2 = mc.evaluate(net, batches, 4, 1.0, seed=21)
    assert m3["nll"] != m_plain2["nll"] and m3["nll"] == m3f["nll"] and m3["ece"] == m3f["ece"]


def test_refusals(dev, monkeypatch):
    from pytorch_bayesiancnn_b200 import EngineError, mc
    net, xs, _ = _case("lenet", 1, "lrt", dev, steps=1, B=16)
    with pytest.raises(EngineError, match="MCTrainStep does not temper"):
        mc.MCTrainStep(net, xs[0], 2, 1000.0, temperature=2.0)
    with pytest.raises(EngineError, match="MCTrainStep does not fill a logit_bank"):
        mc.MCTrainStep(net, xs[0], 2, 1000.0, logit_bank=mc.LogitBank(dev, 8, 2, 10))
    with pytest.raises(ValueError, match="normalized"):
        mc.MCForward(net, xs[0], 2, normalized=True, temperature=2.0)
    with pytest.raises(EngineError, match="one-element float32"):
        mc.MCForward(net, xs[0], 2, temperature=torch.ones(2, device=dev))
    with pytest.raises(EngineError, match="logit_bank holds"):
        mc.MCForward(net, xs[0], 2, logit_bank=mc.LogitBank(dev, 8, 3, 10))
    with monkeypatch.context() as mp_:
        mp_.setattr(mc, "_dist_info", lambda group: (None, 2, 0))
        with pytest.raises(EngineError, match="one rank"):
            mc.MCForward(net, xs[0], 2, logit_bank=mc.LogitBank(dev, 8, 2, 10))


def test_expert_temperatures(dev):
    """Each expert of an ExpertStep tempers with its own temperature: its out is that of the tempered engine alone."""
    from pytorch_bayesiancnn_b200 import mc
    a, xs, _ = _case("lenet", 1, "lrt", dev, steps=1, B=64)
    b = _net("lenet", 10, 1, "lrt", dev, "auto")[0]
    with torch.no_grad():
        for p in b.parameters():
            p.mul_(1.01)
    step = mc.ExpertStep([a, b], xs[0], 3, seed=4, static_inputs=xs, temperatures=[0.5, 2.0])
    res = step()
    step.wait()
    for net, T, o in zip((a, b), (0.5, 2.0), res["experts"]):
        alone = mc.MCForward(net, xs[0], 3, want_uncertainty=True, seed=4, static_inputs=xs, overlap=True,
                             temperature=T)
        alone()
        alone.wait()
        torch.cuda.synchronize()
        for k in ("log_outputs", "pred", "epistemic"):
            assert torch.equal(o[k], alone.out[k]), k
    with pytest.raises(ValueError, match="one per expert"):
        mc.ExpertStep([a, b], xs[0], 3, temperatures=[1.0])


# --------------------------------------------------------------------------- #
# the NLL kernel and the search
# --------------------------------------------------------------------------- #
def _bank_of(dev, z, y):
    from pytorch_bayesiancnn_b200 import mc
    n, S, C = z.shape
    bank = mc.LogitBank(dev, n, S, C)
    bank.append(torch.as_tensor(z).permute(1, 0, 2).contiguous().to(dev), torch.as_tensor(y).to(dev))
    return bank


def _nll_kernel(dev, bank, taus):
    from pytorch_bayesiancnn_b200 import _lib as L
    from pytorch_bayesiancnn_b200 import functional as Fn
    lib = L.lib()
    tau = torch.tensor(taus, dtype=torch.float64, device=dev)
    out = torch.full((len(taus),), float("nan"), dtype=torch.float64, device=dev)
    nbytes = int(lib.bbb_temperature_workspace_bytes(bank.capacity, len(taus)))
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    L.check(lib.bbb_temperature_nll(Fn._ptr(bank._logits), Fn._ptr(bank._labels), Fn._ptr(bank._cursor),
                                    bank.capacity, bank.num_ens, bank.num_classes, Fn._ptr(tau), len(taus), 0, 0,
                                    Fn._ptr(out), None, None, None, Fn._ptr(ws), nbytes, Fn._stream(dev)),
            "bbb_temperature_nll")
    return out


@pytest.mark.parametrize("n,S,C,scale", [(1, 1, 2, 1.0), (37, 2, 10, 5.0), (1000, 25, 10, 1.0), (3001, 1, 10, 1e3),
                                         (130, 100, 10, 1e-3), (9, 256, 100, 3.0), (3, 25, 1000, 10.0),
                                         (2500, 2, 2, 1.0), (33, 100, 1000, 1.0)])
def test_nll_kernel_against_float64(dev, n, S, C, scale):
    rng = np.random.default_rng(n * 7 + S + C)
    z = (rng.standard_normal((n, S, C)) * scale).astype(np.float32)
    y = rng.integers(0, C, n)
    bank = _bank_of(dev, z, y)
    taus = [math.log(0.05), -1.0, 0.0, 0.9162907318741551, math.log(20.0)]
    got = _nll_kernel(dev, bank, taus).cpu().tolist()
    again = _nll_kernel(dev, bank, taus).cpu().tolist()
    assert got == again                                            # the same bits every run
    for tau, v in zip(taus, got):
        T = math.exp(tau)
        ref, b = R.nll(z, y, T), R.bound(z, y, T)
        assert abs(v - ref) <= b, (tau, v, ref, b)


def test_nll_kernel_bits_do_not_depend_on_capacity(dev):
    """Images past the cursor add nothing: a larger bank (a larger grid) gives the same bits."""
    from pytorch_bayesiancnn_b200 import mc
    rng = np.random.default_rng(1)
    z = rng.standard_normal((500, 10, 10)).astype(np.float32)
    y = rng.integers(0, 10, 500)
    small = _bank_of(dev, z, y)
    big = mc.LogitBank(dev, 5000, 10, 10)
    big.append(torch.as_tensor(z).permute(1, 0, 2).contiguous().to(dev), torch.as_tensor(y).to(dev))
    taus = [-0.5, 0.0, 0.5]
    assert _nll_kernel(dev, small, taus).tolist() == _nll_kernel(dev, big, taus).tolist()


def _planted(n, S, C, T0, seed):
    rng = np.random.default_rng(seed)
    z = (rng.standard_normal((n, S, C)) * 3 + rng.standard_normal((n, 1, C)) * 2).astype(np.float32)
    x = z.astype(np.float64) / T0
    x -= x.max(2, keepdims=True)
    p = np.exp(x)
    p = (p / p.sum(2, keepdims=True)).mean(1)
    cum = np.cumsum(p, 1)
    y = np.minimum((rng.random((n, 1)) * cum[:, -1:] > cum).sum(1), C - 1)
    return z, y


@pytest.mark.parametrize("T0,t_min,t_max,bound_hit", [(2.0, 0.05, 20.0, False), (0.5, 0.05, 20.0, False),
                                                      (4.0, 0.2, 1.5, True)])
def test_fit_temperature_search(dev, T0, t_min, t_max, bound_hit):
    from pytorch_bayesiancnn_b200 import mc
    z, y = _planted(3000, 4, 10, T0, int(T0 * 100))
    bank = _bank_of(dev, z, y)
    out = torch.zeros(1, dtype=torch.float32, device=dev)
    fit = mc.fit_temperature(bank, t_min, t_max, 16, 3, out=out, trace=True)
    assert fit.temperature is out
    r = fit.read()
    again = mc.fit_temperature(bank, t_min, t_max, 16, 3, trace=True).read()
    assert r == again                                              # the same bits every run
    assert r["at_bound"] == bound_hit
    assert float(out) == r["temperature"]
    # the device's rounds follow the planner on its own NLLs
    tr = r["trace"]
    assert tr[0]["tau"][:16] == mc.temperature_grid(t_min, t_max, 16) and tr[0]["tau"][16] == 0.0
    for a, b in zip(tr, tr[1:]):
        assert b["tau"] == mc.temperature_grid(t_min, t_max, 16, prev=a["tau"][:16], argmin=R.first_argmin(a["nll"][:16]))
    # every evaluated NLL is float64's within the bound, and the result is the best of the last round (or T = 1)
    for rnd in tr:
        for tau, v in zip(rnd["tau"], rnd["nll"]):
            assert abs(v - R.nll(z, y, math.exp(tau))) <= R.bound(z, y, math.exp(tau))
    assert r["nll"] == min(min(tr[-1]["nll"][:16]), r["nll_at_one"])
    assert r["nll"] <= r["nll_at_one"]
    # the fitted T is as good in float64 as the float64 search's, up to the kernel's error at both points
    ref = R.search(z, y, t_min, t_max, 16, 3)
    T = r["temperature"]
    assert R.nll(z, y, T) <= ref["nll"] + R.bound(z, y, T) + R.bound(z, y, ref["temperature"]) + 1e-9
    if not bound_hit:
        assert abs(math.log(T) - math.log(T0)) < 0.2


def test_calibrate_temperature_end_to_end(dev):
    """An overconfident BBBLeNet (classifier means x 5): the fit raises T above 1, and the held-out NLL and ECE with it
    are no worse than without (an illustration: asserted for direction only)."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    last = [m for m in net.children() if hasattr(m, "W_mu")][-1]
    with torch.no_grad():
        last.W_mu.mul_(5.0)
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
    res = mc.calibrate_temperature(net, cal, 4, seed=5)
    T = res["temperature"]
    assert res["fit"]["temperature"] > 1.0 and res["fit"]["nll"] <= res["fit"]["nll_at_one"]
    assert len(net._temperature_banks["calibration"]) == 768
    before = mc.evaluate(net, test, 4, 1.0, seed=9)
    after = mc.evaluate(net, test, 4, 1.0, seed=9, temperature=T)
    assert after["nll"] <= before["nll"] and after["ece"] <= before["ece"]


def test_unlabelled_bank_is_refused(dev):
    """A captured step with_labels=False logs label -1 on every replay, also after reset(): the host refuses the bank;
    a label the host never saw go bad is refused by the device, with its reason, and T keeps its value."""
    from pytorch_bayesiancnn_b200 import mc
    net, xs, ys = _case("lenet", 1, "lrt", dev, steps=2, B=64)
    bank = mc.LogitBank(dev, 256, 2, 10)
    eng = mc.MCForward(net, xs[0], 2, seed=3, static_inputs=xs, logit_bank=bank)
    bank.reset()
    eng(slot=0)
    torch.cuda.synchronize()
    assert len(bank) == 64 and bool((bank.read()["labels"] == -1).all())
    with pytest.raises(ValueError, match="without labels"):
        mc.fit_temperature(bank)
    good = mc.LogitBank(dev, 64, 2, 10)
    good.append(bank.read()["logits"].permute(1, 0, 2).contiguous(), ys[0])
    good._labels[5] = -1                                           # behind the host's back
    T = torch.full((1,), 0.8, dtype=torch.float32, device=dev)
    with pytest.raises(ValueError, match="1 images were logged without a label"):
        mc.fit_temperature(good, out=T).read()
    assert float(T) == pytest.approx(0.8)
    good._labels[5] = 10
    with pytest.raises(ValueError, match=r"a label is outside \[0, 10\)"):
        mc.fit_temperature(good, out=T).read()
    good._labels[5] = ys[0][5]
    r = mc.fit_temperature(good, out=T).read()
    assert float(T) == r["temperature"] and r["nll"] <= r["nll_at_one"]

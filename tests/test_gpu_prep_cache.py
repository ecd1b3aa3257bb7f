"""Operand tiles, bias rows and KL of the LRT layers prepared once per parameter version (mc.MCForward(cache_prep=True),
fused.PrepCache): every output equals, bit for bit, the engine that prepares them in every step (cache_prep=False), on
every engine layout and across in-place updates of the parameters and the prior -- with steps in flight as well."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _net(dev, variant="lrt", key="alexnet", inputs=3):
    from pytorch_bayesiancnn_b200.models import get_model
    net = get_model(key, inputs, 10, None, variant, "softplus")
    with torch.no_grad():
        g = torch.Generator().manual_seed(123)
        for name, p in net.named_parameters():
            p.copy_(torch.empty(p.shape).normal_(-5.0 if name.endswith("rho") else 0.0, 0.1, generator=g))
    return net.to(dev).train()


def _pair(net, x, num_ens, **kw):
    """(cached, uncached) engines of the same net, seed and noise blocks."""
    from pytorch_bayesiancnn_b200 import mc
    a = mc.MCForward(net, x, num_ens, seed=77, cache_prep=True, **kw)
    b = mc.MCForward(net, x, num_ens, seed=77, cache_prep=False, **kw)
    return a, b


def _step(eng, x=None, labels=None):
    """One step; a copy of its outputs, taken on the stream they are complete on (no host synchronisation)."""
    out = eng(x, labels)
    with torch.cuda.stream(eng.result_stream or torch.cuda.current_stream()):
        return {k: v.clone() for k, v in out.items()}


def _same(ra, rb, what):
    torch.cuda.synchronize()
    assert ra.keys() == rb.keys()
    for k in ra:
        assert torch.equal(ra[k], rb[k]), (what, k)


@pytest.mark.parametrize("layout", ["headline", "serial", "fold10", "sample_loop3", "uncertainty_labels"])
def test_cached_equals_uncached(dev, layout):
    """Steps of the cached and the uncached engine, interleaved, are bit-identical; the cached chain has no prep."""
    net = _net(dev)
    x = torch.randn(256, 3, 32, 32, device=dev)
    labels = None
    kw = {"headline": dict(num_ens=1, overlap=True, inflight=4),
          "serial": dict(num_ens=1),
          "fold10": dict(num_ens=10, overlap=True, inflight=2),
          "sample_loop3": dict(num_ens=3, fold=False),
          "uncertainty_labels": dict(num_ens=4, want_uncertainty=True, want_information=True, with_labels=True,
                                     train_size=50.0, beta=0.3, overlap=True, inflight=3)}[layout]
    if kw.get("with_labels"):
        labels = torch.randint(0, 10, (256,), device=dev)
    a, b = _pair(net, x, kw.pop("num_ens"), **kw)
    assert a._prep is not None and b._prep is None
    if layout == "fold10":
        assert a.fold_steps is not None
    for i in range(6):
        xi = torch.randn_like(x) if i % 2 else None
        _same(_step(a, xi, labels), _step(b, xi, labels), (layout, i))
    assert a.prep_replays == 0 and a.prep_kernels == 6
    assert a.kernels_per_step < b.kernels_per_step


def test_headline_kernel_counts(dev):
    """The headline step (BBBAlexNet LRT, one sample, four in flight) replays 8 engine kernels -- noise_advance, six GEMM
    kernels, the exchange -- and the six preps run once per parameter version."""
    from pytorch_bayesiancnn_b200 import _lib as L, mc
    net = _net(dev)
    x = torch.randn(512, 3, 32, 32, device=dev)
    a, b = _pair(net, x, 1, overlap=True, inflight=4)
    assert a.kernels_per_step == 8 and b.kernels_per_step == 14
    n0 = L.launch_count()
    for _ in range(5):
        a()
    assert L.launch_count() == n0                         # graph replays only
    assert a.prep_replays == 0
    with torch.no_grad():
        net.conv1.W_mu.mul_(1.01)
    for _ in range(5):
        a()
    a.wait()
    assert a.prep_replays == 1 and a.prep_kernels == 6
    # BBB layers draw their weights in every step: nothing is cached and the counts stay
    bn = _net(dev, "bbb")
    c = mc.MCForward(bn, x, 1, seed=5, overlap=True, inflight=4)
    d = mc.MCForward(bn, x, 1, seed=5, overlap=True, inflight=4, cache_prep=False)
    assert c._prep is None and c.kernels_per_step == d.kernels_per_step
    torch.cuda.synchronize()


def _adam(net):
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    g = torch.Generator(device=net.conv1.W_mu.device).manual_seed(3)

    def step():
        for p in net.parameters():
            p.grad = torch.randn(p.shape, device=p.device, generator=g)
        opt.step()
    return step


def _copy(net):
    def step():
        with torch.no_grad():
            for p in net.parameters():
                p.copy_(p * 0.99 + 0.001)
    return step


@pytest.mark.parametrize("update", ["adam", "copy", "set_prior_in_place", "kl_convention"])
@pytest.mark.parametrize("inflight", [1, 4])
def test_in_place_update_is_read_by_the_next_step(dev, update, inflight):
    """An update between steps is read by the very next step, as by the uncached engine given the same sequence."""
    from pytorch_bayesiancnn_b200.modules import _BayesLayer
    net = _net(dev)
    layers = [m for m in net.modules() if isinstance(m, _BayesLayer)]
    if update == "set_prior_in_place":
        for m in layers:
            m.set_prior(m.W_mu.detach() * 0.5, 0.2, 0.0, 0.3)
    x = torch.randn(256, 3, 32, 32, device=dev)
    kw = dict(overlap=True, inflight=inflight) if inflight > 1 else {}
    a, b = _pair(net, x, 1, **kw)
    if update == "adam":
        upd = _adam(net)
    elif update == "copy":
        upd = _copy(net)
    elif update == "set_prior_in_place":
        def upd():
            for m in layers:
                m.set_prior(m.W_mu.detach() * 0.7, torch.full_like(m.W_mu, 0.15), 0.1, 0.25)
    else:
        def upd():
            for m in layers:
                m.kl_convention = "textbook" if m.kl_convention == "reference" else "reference"
    ra0 = _step(a)
    _same(ra0, _step(b), "before")
    kls = [ra0["kl"]]
    for i in range(3):
        upd()
        ra = _step(a)
        _same(ra, _step(b), (update, i))
        kls.append(ra["kl"])
        ra = _step(a)
        _same(ra, _step(b), (update, i, "again"))
    if update != "kl_convention":                      # the KL settings are baked into both engines' graphs
        assert not torch.equal(kls[0], kls[1])
        assert a.prep_replays == 3
    torch.cuda.synchronize()


def test_new_prior_is_refused_as_before(dev):
    """A prior set anew (new buffers) or a mixture prior set after capture is refused by both engines."""
    from pytorch_bayesiancnn_b200 import _lib as L
    net = _net(dev)
    x = torch.randn(128, 3, 32, 32, device=dev)
    a, b = _pair(net, x, 1, overlap=True, inflight=2)
    _same(_step(a), _step(b), "before")
    net.conv1.set_prior(0.0, 0.5)
    for eng in (a, b):
        with pytest.raises(L.EngineError):
            eng()
    net2 = _net(dev)
    a, b = _pair(net2, x, 1)
    net2.conv2.set_mixture_prior(0.5, 1.0, 0.01)
    for eng in (a, b):
        with pytest.raises(L.EngineError):
            eng()


@pytest.mark.parametrize("fold", [True, False])
def test_mixture_prior_keeps_its_draw_in_the_step(dev, fold):
    """A mixture-prior layer's tiles are cached, its Monte-Carlo KL is drawn in every step: cached == uncached."""
    from pytorch_bayesiancnn_b200.modules import mixture_prior
    net = mixture_prior(_net(dev), 0.5, 1.0, 0.02)
    x = torch.randn(128, 3, 32, 32, device=dev)
    a, b = _pair(net, x, 3, fold=fold, overlap=True, inflight=2)
    assert a._prep is not None
    # one engine after the other: the draws' scratch is private per (layer, workspace slot), which the two in-flight
    # engines of one net share (Fn.workspace_slot)
    ra = [_step(a) for _ in range(4)]
    a.wait()
    torch.cuda.synchronize()
    rb = [_step(b) for _ in range(4)]
    for i in range(4):
        _same(ra[i], rb[i], ("mixture", fold, i))
    assert not torch.equal(ra[0]["kl"], ra[1]["kl"])   # a fresh draw per step
    assert a.kernels_per_step < b.kernels_per_step


def test_update_with_steps_in_flight(dev):
    """Four steps enqueued, an update, four more: each step equals a serial uncached run of the same sequence -- the
    re-prep waits for the steps still reading the old tiles and KL, and the later steps wait for it."""
    from pytorch_bayesiancnn_b200 import mc
    net = _net(dev)
    xs = [torch.randn(512, 3, 32, 32, device=dev) for _ in range(2)]
    a = mc.MCForward(net, xs[0], 1, seed=21, static_inputs=xs, overlap=True, inflight=4, cache_prep=True)
    s = mc.MCForward(net, xs[0], 1, seed=21, static_inputs=xs, cache_prep=False)
    upd = _copy(net)
    saved = [p.detach().clone() for p in net.parameters()]
    got = [_step_slot(a, i % 2) for i in range(4)]
    upd()
    got += [_step_slot(a, i % 2) for i in range(4, 8)]
    a.wait()
    torch.cuda.synchronize()
    with torch.no_grad():                               # the serial reference replays the same sequence from the start
        for p, v in zip(net.parameters(), saved):
            p.copy_(v)
    ref = []
    for i in range(8):
        if i == 4:
            upd()
        ref.append(_step_slot(s, i % 2))
    torch.cuda.synchronize()
    for i, (ra, rb) in enumerate(zip(got, ref)):
        for k in ra:
            assert torch.equal(ra[k], rb[k]), (i, k)
    assert a.prep_replays == 1


def _step_slot(eng, slot):
    out = eng(slot=slot)
    with torch.cuda.stream(eng.result_stream or torch.cuda.current_stream()):
        return {k: v.clone() for k, v in out.items()}


def test_evaluate_re_preps_once_per_epoch(dev):
    """mc.evaluate keeps its engines on the net: after an optimizer step the next epoch's first step re-preps, once."""
    from pytorch_bayesiancnn_b200 import mc
    net = _net(dev)
    loader = [(torch.randn(64, 3, 32, 32), torch.randint(0, 10, (64,))) for _ in range(5)]
    upd = _adam(net)
    mc.evaluate(net, loader, 2, 100.0, seed=4)
    engines = [e["eng"] for ev in net.__dict__["_mc_eval"].values() for e in ev["engines"].values()]
    assert engines and all(e._prep is not None and e.prep_replays == 0 for e in engines)
    upd()
    mc.evaluate(net, loader, 2, 100.0, seed=4)
    assert all(e.prep_replays == 1 for e in engines)
    mc.evaluate(net, loader, 2, 100.0, seed=4)
    assert all(e.prep_replays == 1 for e in engines)

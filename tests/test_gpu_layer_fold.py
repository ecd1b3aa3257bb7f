"""Monte-Carlo samples of BBBLeNet / BBB3Conv3FC folded into passes of the per-layer tensor-core kernel: each row draws
from its own sample's Philox stream (LRT) or multiplies by its own sample's weight draw (BBB), and the aten activations
and pools between the layers treat every image on its own.  A folded step must equal the sample loop bit for bit."""
import numpy as np
import pytest
import torch

from tests.test_gpu_mc import MC_NS, _engine_eps, _net
from tests.util import scale_err

pytestmark = pytest.mark.gpu
KEYS = ("log_outputs", "kl", "pred", "epistemic", "aleatoric", "entropy")
NETS = [("lenet", "lrt"), ("lenet", "bbb"), ("3conv3fc", "lrt"), ("3conv3fc", "bbb")]


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def _pair(net, x, S, seed, **kw):
    from pytorch_bayesiancnn_b200 import mc
    a = mc.MCForward(net, x, S, want_uncertainty=True, seed=seed, fold=True, **kw)
    b = mc.MCForward(net, x, S, want_uncertainty=True, seed=seed, fold=False, **kw)
    return a, b


def _assert_identical(a, b):
    oa = {k: v.clone() for k, v in a(a.x).items()}
    ob = b(b.x)
    torch.cuda.synchronize()
    for k in range(a.logits.shape[0]):
        assert torch.equal(a.logits[k], b.logits[k]), k
    for k in KEYS:
        assert torch.equal(oa[k], ob[k]), k
    assert torch.equal(a.kl_one, b.kl_one)


@pytest.mark.parametrize("key,variant", NETS)
def test_layer_fold_equals_sample_loop(dev, key, variant):
    net, _ = _net(key, 10, 1, variant, dev, "auto")
    x = torch.randn(256, 1, 32, 32, device=dev)
    a, b = _pair(net, x, 5, 11)
    assert a.fold_steps is None and a.layer_fold is not None and b.layer_fold is None
    assert a.layer_fold[0] * a.layer_fold[1] >= 5
    _assert_identical(a, b)
    assert a.kernels_per_step < b.kernels_per_step, (a.kernels_per_step, b.kernels_per_step)


def test_layer_fold_ragged_batch(dev):
    """B = 200: LRT folds (its rows need no tile alignment); BBB does not (a 128-row tile would hold two samples)."""
    x = torch.randn(200, 1, 32, 32, device=dev)
    net, _ = _net("3conv3fc", 10, 1, "lrt", dev, "auto")
    a, b = _pair(net, x, 4, 13)
    assert a.layer_fold is not None
    _assert_identical(a, b)
    assert a.kernels_per_step < b.kernels_per_step
    net, _ = _net("lenet", 10, 1, "bbb", dev, "auto")
    a, b = _pair(net, x, 4, 13)
    assert a.layer_fold is None and a.fold_steps is None and a.kernels_per_step == b.kernels_per_step
    _assert_identical(a, b)
    assert np.isfinite(a.out["log_outputs"].cpu().numpy()).all()


@pytest.mark.parametrize("variant", ["lrt", "bbb"])
def test_layer_fold_stride_of_emulated_ranks(dev, variant):
    """Rank 1 of 3 folds its samples 1 and 4: row block k == net(x) as sample 1 + 3k, bit for bit; the KL is unfolded."""
    from pytorch_bayesiancnn_b200 import functional as Fn
    B, world, rank, seed = 256, 3, 1, 5
    net, _ = _net("lenet", 10, 1, variant, dev, "auto")
    x = torch.randn(B, 1, 32, 32, device=dev)
    with torch.no_grad(), Fn.mc_sample(rank, seed), Fn.layer_fold(B, world << 40):
        logits, kl = net(x.repeat(2, 1, 1, 1))
    for k in range(2):
        with torch.no_grad(), Fn.mc_sample(rank + k * world, seed):
            ref, ref_kl = net(x)
        assert torch.equal(logits[k * B:(k + 1) * B], ref), k
        assert torch.equal(kl, ref_kl)
    assert not torch.equal(logits[:B], logits[B:])


@pytest.mark.parametrize("key,variant", [("3conv3fc", "lrt"), ("lenet", "bbb")])
def test_layer_fold_sample_matches_oracle(dev, key, variant):
    """The row block of folded sample j == the oracle's forward on the eps the engine draws for sample j (bf16 bar)."""
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import functional as Fn
    from oracle import bbb_oracle as O
    B, seed, j = 128, 23, 2
    net, params = _net(key, 10, 1, variant, dev, "auto")
    x = torch.rand(B, 1, 32, 32, generator=torch.Generator().manual_seed(9))
    with torch.no_grad(), Fn.mc_sample(0, seed), Fn.layer_fold(B, 1 << 40):
        logits, kl = net(x.to(dev).repeat(3, 1, 1, 1))
    eps = _engine_eps(bbb, key, 10, 1, variant, B, seed, MC_NS | (j << 40), dev)
    ref, ref_kl = O.net_forward(key, params, x, eps, variant, "softplus", 0.0, 0.1, 10)
    e = scale_err(logits[j * B:(j + 1) * B], ref)
    assert e < 1e-2, e
    assert abs(float(kl) - float(ref_kl)) <= 1e-5 * abs(float(ref_kl))


@pytest.mark.parametrize("variant", ["lrt", "bbb"])
def test_layer_fold_graph_replay_draws_fresh_noise(dev, variant):
    """Captured folded step: the second replay draws new noise and equals the eager sample loop at replay base 2^20."""
    from pytorch_bayesiancnn_b200 import functional as Fn, mc
    from pytorch_bayesiancnn_b200.graph import _STRIDE
    net, _ = _net("lenet", 10, 1, variant, dev, "auto")
    x = torch.randn(128, 1, 32, 32, device=dev)
    eng = mc.MCForward(net, x, 3, want_uncertainty=True, seed=31)
    assert eng.layer_fold is not None
    first = {k: v.clone() for k, v in eng(x).items()}
    out = eng(x)
    torch.cuda.synchronize()
    assert not torch.equal(first["log_outputs"], out["log_outputs"])
    assert torch.equal(first["kl"], out["kl"])
    base = torch.full((1,), _STRIDE, dtype=torch.int64, device=dev)
    for j in range(3):
        with Fn.stream_base(base), Fn.mc_sample(j, 31), torch.no_grad():
            lg, kl = net(x)
        assert torch.equal(eng.logits[j], lg), j
    assert torch.equal(eng.kl_one, kl)
    assert eng.timeouts() == 0


@pytest.mark.parametrize("variant", ["lrt", "bbb"])
def test_layer_fold_overlapped_inflight_equals_serial(dev, variant):
    """overlap=True, inflight=2 with a layer fold in two groups: bit-identical to the serial folded engine, step for step."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("3conv3fc", 10, 1, variant, dev, "auto")
    x = torch.randn(128, 1, 32, 32, device=dev)
    labs = [torch.randint(0, 10, (128,), device=dev) for _ in range(3)]
    kw = dict(want_uncertainty=True, with_labels=True, train_size=10.0, beta=0.2, seed=3, fold_group=3)
    a = mc.MCForward(net, x, 5, **kw)
    c = mc.MCForward(net, x, 5, overlap=True, inflight=2, **kw)
    assert a.layer_fold == (3, 2) and c.layer_fold == (3, 2) and c.inflight == 2
    for n in (1, 2):
        for i in range(n):
            oa = a(x, labs[i])
        ra = {k: v.clone() for k, v in oa.items()}
        for i in range(n):
            oc = c(x, labs[i])
        c.wait()
        torch.cuda.synchronize()
        for k in ra:
            assert torch.equal(ra[k], oc[k]), (n, k)
    assert a.timeouts() == 0 and c.timeouts() == 0


def test_c5_layer_fold_equals_sample_loop_within_budget(dev):
    """C5 on one GPU (BBB3Conv3FC, 1x32x32, B = 2048, 100 samples, LRT, uncertainty): folded in groups == fold=False
    exactly; one folded step's activations stay within the byte budget on top of the engine's own buffers."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("3conv3fc", 10, 1, "lrt", dev, "auto")
    x = torch.rand(2048, 1, 32, 32, device=dev)
    a, b = _pair(net, x, 100, 99)
    G, n_groups = a.layer_fold
    assert 1 < G < 100 and n_groups == -(-100 // G)
    _assert_identical(a, b)
    assert a.kernels_per_step < b.kernels_per_step
    del a, b
    e = mc.MCForward(net, x, 100, want_uncertainty=True, seed=99, graph=False)
    assert e.layer_fold == (G, n_groups)
    e()                                        # first call: the layers' workspaces
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(dev)
    torch.cuda.reset_peak_memory_stats(dev)
    e()
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated(dev) - base
    print("C5 layer fold G", G, "groups", n_groups, "peak activation bytes", extra, "budget", mc.LAYER_FOLD_BUDGET)
    assert extra <= mc.LAYER_FOLD_BUDGET + (1 << 20), extra      # + the per-call KL scalars and logits


def test_layer_fold_refuses_autograd_and_external_eps(dev):
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    net, _ = _net("lenet", 10, 1, "lrt", dev, "auto")
    x = torch.randn(256, 1, 32, 32, device=dev)
    with pytest.raises(L.EngineError, match="forward-only"), Fn.layer_fold(128, 1 << 40):
        net(x)                                                        # parameters require grad
    eps = [torch.zeros(256, 6, 28, 28)]
    with pytest.raises(L.EngineError, match="no external eps"), torch.no_grad(), Fn.layer_fold(128, 1 << 40), \
            bbb.external_eps(eps):
        net(x)
    assert not Fn.layer_fold_active()

"""Monte-Carlo samples of a BBB net (weight-space sampling) folded into one pass of the fused chain: each 128-row tile
multiplies by its own sample's weight draw.  A folded run must equal the sample loop, sample by sample."""
import numpy as np
import pytest
import torch

from tests.test_gpu_mc import MC_NS, _engine_eps, _net
from tests.util import scale_err

pytestmark = pytest.mark.gpu
KEYS = ("log_outputs", "kl", "pred", "epistemic", "aleatoric", "entropy")


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    return torch.device("cuda:0")


def test_bbb_fold_equals_sample_loop(dev):
    """Same bars as the LRT folding test: logits, combine and uncertainty outputs of S = 5 folded samples == 5 passes."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("alexnet", 10, 3, "bbb", dev, "auto")
    x = torch.randn(256, 3, 32, 32, device=dev)
    a = mc.MCForward(net, x, 5, want_uncertainty=True, seed=11, fold=True)
    b = mc.MCForward(net, x, 5, want_uncertainty=True, seed=11, fold=False)
    assert a.fold_steps is not None and b.fold_steps is None
    oa, ob = a(x), b(x)
    torch.cuda.synchronize()
    assert (a.logits - b.logits).abs().max() <= 1e-6 * b.logits.abs().max()
    for k in KEYS:
        assert (oa[k] - ob[k]).abs().max() <= 1e-5 * max(1.0, float(ob[k].abs().max())), k
    assert a.kernels_per_step < b.kernels_per_step, (a.kernels_per_step, b.kernels_per_step)


def _fold_run(steps, x, rows, world, rank, seed):
    """What MCForward runs on rank `rank` of `world`: its samples rank, rank + world, ... folded into one pass."""
    from pytorch_bayesiancnn_b200 import fused, functional as Fn
    with torch.no_grad(), Fn.mc_sample(rank, seed):
        return fused._run(steps, x, True, None, False, None, fold=(rows, world << 40))


def test_bbb_fold_stride_of_emulated_ranks(dev):
    """Rank 1 of 3 folds its samples 1 and 4: row block k == net(x) as sample 1 + 3k, and the KL is the unfolded one."""
    from pytorch_bayesiancnn_b200 import fused, functional as Fn
    B, world, rank, seed = 256, 3, 1, 5
    net, _ = _net("alexnet", 10, 3, "bbb", dev, "auto")
    x = torch.randn(B, 3, 32, 32, device=dev)
    steps = fused.plan(list(net.children()), (2 * B, 3, 32, 32), (B, world << 40))
    assert steps is not None
    logits, kl = _fold_run(steps, x, B, world, rank, seed)
    torch.cuda.synchronize()
    for k in range(2):
        with torch.no_grad(), Fn.mc_sample(rank + k * world, seed):
            ref, ref_kl = net(x)
        blk = logits[k * B:(k + 1) * B]
        assert (blk - ref).abs().max() <= 1e-6 * ref.abs().max(), k
        assert torch.equal(kl, ref_kl)
    assert not torch.equal(logits[:B], logits[B:])                       # two different weight draws


def test_bbb_fold_sample_matches_oracle(dev):
    """The row block of folded sample j == the oracle's forward on the eps the engine draws for sample j (bf16 bar)."""
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import fused
    from oracle import bbb_oracle as O
    B, seed = 128, 23
    net, params = _net("alexnet", 10, 3, "bbb", dev, "auto")
    x = torch.rand(B, 3, 32, 32, generator=torch.Generator().manual_seed(9))
    steps = fused.plan(list(net.children()), (3 * B, 3, 32, 32), (B, 1 << 40))
    logits, kl = _fold_run(steps, x.to(dev), B, 1, 0, seed)
    j = 2
    eps = _engine_eps(bbb, "alexnet", 10, 3, "bbb", B, seed, MC_NS | (j << 40), dev)
    ref, ref_kl = O.net_forward("alexnet", params, x, eps, "bbb", "softplus", 0.0, 0.1, 10)
    e = scale_err(logits[j * B:(j + 1) * B], ref)
    assert e < 1e-2, e
    assert abs(float(kl) - float(ref_kl)) <= 1e-5 * abs(float(ref_kl))


def test_bbb_fold_graph_replay_draws_fresh_noise(dev):
    """Captured folded step: the second replay draws new weights and equals the eager sample loop at replay base 2^20."""
    from pytorch_bayesiancnn_b200 import functional as Fn, mc
    from pytorch_bayesiancnn_b200.graph import _STRIDE
    from oracle import bbb_oracle as O
    net, _ = _net("alexnet", 10, 3, "bbb", dev, "auto")
    x = torch.randn(128, 3, 32, 32, device=dev)
    eng = mc.MCForward(net, x, 3, want_uncertainty=True, seed=31)
    assert eng.fold_steps is not None
    first = {k: v.clone() for k, v in eng(x).items()}
    out = eng(x)
    torch.cuda.synchronize()
    assert not torch.equal(first["log_outputs"], out["log_outputs"])
    assert torch.equal(first["kl"], out["kl"])
    base = torch.full((1,), _STRIDE, dtype=torch.int64, device=dev)
    logits = []
    for j in range(3):
        with Fn.stream_base(base), Fn.mc_sample(j, 31), torch.no_grad():
            lg, kl = net(x)
        logits.append(lg.cpu())
    ref = O.mc_combine(logits)
    assert (out["log_outputs"].cpu() - ref).abs().max() < 1e-4
    assert abs(float(out["kl"]) - float(kl)) <= 1e-6 * abs(float(kl))
    assert eng.timeouts() == 0


def test_bbb_fold_overlapped_inflight_equals_serial(dev):
    """overlap=True, inflight=2 with a BBB fold: bit-identical to the serial folded engine, step for step."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("alexnet", 10, 3, "bbb", dev, "auto")
    x = torch.randn(128, 3, 32, 32, device=dev)
    labs = [torch.randint(0, 10, (128,), device=dev) for _ in range(3)]
    kw = dict(want_uncertainty=True, with_labels=True, train_size=10.0, beta=0.2, seed=3)
    a = mc.MCForward(net, x, 3, **kw)
    c = mc.MCForward(net, x, 3, overlap=True, inflight=2, **kw)
    assert a.fold_steps is not None and c.fold_steps is not None and c.inflight == 2
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


def test_bbb_fold_falls_back_to_the_sample_loop(dev):
    """B = 200 is not a whole number of 128-row tiles: no fold, and the results are the sample loop's."""
    from pytorch_bayesiancnn_b200 import mc
    net, _ = _net("alexnet", 10, 3, "bbb", dev, "auto")
    x = torch.randn(200, 3, 32, 32, device=dev)
    a = mc.MCForward(net, x, 4, want_uncertainty=True, seed=17, fold=True)
    b = mc.MCForward(net, x, 4, want_uncertainty=True, seed=17, fold=False)
    assert a.fold_steps is None and a.kernels_per_step == b.kernels_per_step
    oa = {k: v.clone() for k, v in a(x).items()}
    ob = b(x)
    torch.cuda.synchronize()
    for k in KEYS:
        assert torch.equal(oa[k], ob[k]), k
    assert np.isfinite(oa["log_outputs"].cpu().numpy()).all()

"""BatchBALD without a GPU: the float64 reference (tests/batchbald_ref.py) against brute-force enumeration, the host
plan of the greedy rounds, the bank's padding and size, and the argument checks of the selection entry points."""
import numpy as np
import pytest
import torch

from tests import batchbald_ref as R


def _probs(N, S, C, seed=0):
    rng = np.random.default_rng(seed)
    lo = rng.normal(size=(N, S, C)) * 2.0
    p = np.exp(lo - lo.max(2, keepdims=True))
    return p / p.sum(2, keepdims=True)


def test_exact_estimator_equals_brute_force():
    """C = 3, S = 5, N = 20, k <= 5: sum_m omega_m h_m(i) + const == H(y_A, y_i) for every candidate and every A of the
    greedy path, and round 0 is the mutual information."""
    probs = _probs(20, 5, 3, seed=1)
    chosen, _ = R.greedy_exact(probs, 5)
    eh = R.expected_entropy(probs)
    for n in range(5):
        A = chosen[:n]
        pt, omega, const, configs = R.exact_configs(probs, A)
        assert configs.shape == (3 ** n, n) and abs(omega.sum() - 1.0) < 1e-12
        h = R.h_m(probs, pt)
        for i in range(20):
            if i in A:
                continue
            assert abs(h[i] @ omega + const - R.joint_entropy_brute(probs, A + [i])) < 1e-12, (n, i)
        if n == 0:
            pbar = probs.mean(1)
            mi = -(pbar * np.log(pbar)).sum(1) - eh
            a, _ = R.scores(probs, pt, omega, const, A)
            assert np.allclose(a, mi, rtol=0, atol=1e-14)


def test_sampled_estimator_identity_on_all_configurations():
    """The sampled estimator's identity: over configurations drawn from the exact joint it converges to the exact
    H(y_A, y_i); with the configurations listed with multiplicity proportional to their weight it is exact."""
    probs = _probs(12, 4, 3, seed=2)
    A = [0, 5]
    pt, omega, const, configs = R.exact_configs(probs, A)
    rng = np.random.default_rng(0)
    draw = rng.choice(len(omega), size=200000, p=omega / omega.sum())
    pts, om, cs = R.sampled_configs(probs, A, configs[draw])
    h = R.h_m(probs, pts)
    for i in (1, 7, 11):
        exact = R.joint_entropy_brute(probs, A + [i])
        assert abs(h[i] @ om + cs - exact) < 2e-2, i
        # the columns of the sampled configurations are the exact ones
        assert np.allclose(pts, pt[draw], atol=1e-14)


def test_greedy_score_never_decreases():
    probs = _probs(30, 6, 4, seed=3)
    _, got = R.greedy_exact(probs, 4)
    assert all(b >= a - 1e-12 for a, b in zip(got, got[1:])), got


@pytest.mark.parametrize("C,k,num_configs", [(10, 6, 10000), (3, 8, 100), (2, 3, 1), (100, 3, 1000)])
def test_plan_switches_to_sampling_past_num_configs(C, k, num_configs):
    from pytorch_bayesiancnn_b200 import mc
    plan = mc.batchbald_plan(C, k, num_configs)
    assert len(plan) == k
    for n, (M, exact) in enumerate(plan):
        assert exact == (C ** n <= num_configs)
        assert M == (C ** n if exact else num_configs)
    assert plan[0] == (1, True)


@pytest.mark.parametrize("S,C,pads", [(1, 2, (8, 2)), (8, 3, (8, 4)), (100, 10, (104, 16)), (256, 128, (256, 128)),
                                      (20, 100, (24, 128)), (9, 16, (16, 16))])
def test_bank_padding_and_size(S, C, pads):
    from pytorch_bayesiancnn_b200 import mc
    assert mc.bank_pads(S, C) == pads
    bank = mc.ProbBank("cpu", 5, S, C)
    assert (bank.S_pad, bank.C_pad) == pads
    assert tuple(bank._probs.shape) == (5, pads[1], pads[0]) and bank._probs.dtype == torch.float32
    assert bool((bank._probs == 0).all()) and tuple(bank._ee.shape) == (5,) and bank._ee.dtype == torch.float64
    assert len(bank) == 0 and bank.dropped == 0
    # the MNIST-scale pool of the benchmark: 60 000 x 16 x 104 fp32 words
    assert 60000 * mc.bank_pads(100, 10)[1] * mc.bank_pads(100, 10)[0] * 4 == 399_360_000


def test_argument_checks():
    from pytorch_bayesiancnn_b200 import EngineError, mc
    with pytest.raises(ValueError, match="num_classes"):
        mc.ProbBank("cpu", 4, 10, 129)
    with pytest.raises(ValueError, match="num_classes"):
        mc.ProbBank("cpu", 4, 10, 1)
    with pytest.raises(ValueError, match="num_ens"):
        mc.ProbBank("cpu", 4, 257, 10)
    with pytest.raises(ValueError, match="capacity"):
        mc.ProbBank("cpu", -1, 10, 10)
    bank = mc.ProbBank("cpu", 4, 10, 10)
    bank._cursor[0] = 3                                   # three entries held
    for sel in (lambda: mc.batchbald(bank, 4), lambda: mc.bald(bank, 4), lambda: mc.batchbald(bank, 0)):
        with pytest.raises(ValueError, match="k must be"):
            sel()
    with pytest.raises(ValueError, match="num_configs"):
        mc.batchbald(bank, 2, num_configs=0)
    for S, C in ((11, 10), (10, 11)):
        with pytest.raises(EngineError, match="prob_bank holds 10 samples x 10 classes"):
            bank._require(S, C, "MCForward")
    bank._require(10, 10, "MCForward")
    with pytest.raises(ValueError, match="method"):
        mc.acquire(torch.nn.Linear(2, 2), [], 1, 2, method="maxent")


def test_selection_refuses_a_bank_that_dropped_images():
    from pytorch_bayesiancnn_b200 import EngineError, mc
    bank = mc.ProbBank("cpu", 4, 10, 10)
    bank._cursor[0], bank._cursor[1] = 6, 2               # six appended into four entries
    for sel in (lambda: mc.batchbald(bank, 2), lambda: mc.bald(bank, 2)):
        with pytest.raises(EngineError, match="2 images did not fit"):
            sel()


def test_draw_from_one_distribution_takes_one_cumulative_sum():
    """The first sampled round draws M configurations of one joint over M_prev * C outcomes: [M] indices from one
    cumulative sum of M_prev * C words (not M rows of it), with zero-weight outcomes never drawn; row-wise draws take
    one index per row."""
    from pytorch_bayesiancnn_b200 import mc
    g = torch.Generator().manual_seed(0)
    w = torch.rand(100000, dtype=torch.float64, generator=g)
    w[::2] = 0.0
    idx = mc._draw(w, torch.Generator().manual_seed(1), 10000)
    assert idx.shape == (10000,) and idx.dtype == torch.int64
    assert bool((idx % 2 == 1).all()) and int(idx.min()) >= 0 and int(idx.max()) < w.numel()
    p = torch.tensor([0.1, 0.0, 0.6, 0.3], dtype=torch.float64)
    freq = torch.bincount(mc._draw(p, torch.Generator().manual_seed(2), 200000), minlength=4).double() / 200000
    assert torch.allclose(freq, p, atol=5e-3)
    rows = torch.tensor([[0.0, 1.0, 0.0], [0.0, 0.0, 2.0]], dtype=torch.float64)
    assert mc._draw(rows, torch.Generator().manual_seed(3)).tolist() == [1, 2]

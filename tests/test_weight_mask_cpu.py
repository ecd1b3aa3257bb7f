"""Pruning masks without a GPU: prune_by_snr's ranking and counts, set_weight_mask's refusals, the state_dict round trip,
the captured-engine guard's view of masks, and the float64 reference (tests/mask_ref.py) against hand-computed cases."""
import math

import pytest
import torch

from tests import mask_ref as MR


def _net(seed=0):
    import pytorch_bayesiancnn_b200 as bbb
    torch.manual_seed(seed)

    class Net(bbb.ModuleWrapper):
        def __init__(self):
            super().__init__()
            self.conv = bbb.BBBLRTConv2d(2, 3, 2)
            self.fc = bbb.BBBLRTLinear(4, 5)
    return Net()


def _layers(net):
    return [m for m in net.modules() if hasattr(m, "W_mu")]


def test_snr_is_abs_mu_over_softplus_rho():
    import pytorch_bayesiancnn_b200 as bbb
    net = _net()
    for m in _layers(net):
        ref = m.W_mu.detach().double().abs() / torch.log1p(torch.exp(m.W_rho.detach().double()))
        assert torch.allclose(bbb.snr(m).double(), ref, rtol=1e-6)
        assert bbb.snr(m).dtype == torch.float32


def test_prune_by_snr_counts_and_global_ranking():
    import pytorch_bayesiancnn_b200 as bbb
    net = _net(1)
    snrs = torch.cat([bbb.snr(m).reshape(-1) for m in _layers(net)])
    N = snrs.numel()
    assert N == 3 * 2 * 2 * 2 + 5 * 4
    out = bbb.prune_by_snr(net, 0.5)
    n = math.floor(0.5 * N)
    assert out["pruned"] == n and out["total"] == N
    assert set(out["per_layer"]) == {"conv", "fc"}
    assert sum(p for p, _ in out["per_layer"].values()) == n
    assert [t for _, t in out["per_layer"].values()] == [24, 20]
    kept = torch.cat([m.W_mask.reshape(-1) for m in _layers(net)])
    assert int((~kept).sum()) == n
    # one global threshold: every pruned SNR <= every kept SNR, the threshold the largest pruned one
    assert float(snrs[~kept].max()) <= float(snrs[kept].min())
    assert out["threshold"] == float(snrs[~kept].max())
    for m in _layers(net):
        assert m.W_mask.dtype == torch.bool and m.W_mask.shape == m.W_mu.shape
        assert m.mask_tensors()[1] is None                      # biases are not ranked without biases=True


def test_prune_by_snr_fraction_edges_and_refusals():
    import pytorch_bayesiancnn_b200 as bbb
    net = _net(2)
    out = bbb.prune_by_snr(net, 0.0)
    assert out["pruned"] == 0 and out["threshold"] is None
    assert all(bool(m.W_mask.all()) for m in _layers(net))
    out = bbb.prune_by_snr(net, 1.0)
    assert out["pruned"] == out["total"]
    assert all(not bool(m.W_mask.any()) for m in _layers(net))
    for bad in (-0.1, 1.5, float("nan")):
        with pytest.raises(ValueError, match="fraction"):
            bbb.prune_by_snr(net, bad)


def test_prune_by_snr_ties_follow_layer_order_then_flat_index():
    import pytorch_bayesiancnn_b200 as bbb
    net = _net(3)
    with torch.no_grad():
        for m in _layers(net):
            m.W_mu.fill_(1.0)
            m.W_rho.fill_(0.0)                                  # every SNR equal
    out = bbb.prune_by_snr(net, 30.5 / 44)
    conv, fc = _layers(net)
    assert out["pruned"] == 30
    assert not bool(conv.W_mask.any())                          # all 24 of the first layer
    assert (~fc.W_mask).reshape(-1).tolist() == [True] * 6 + [False] * 14   # then the first 6 of the second, in order


def test_prune_by_snr_again_is_monotone_and_counts_pruned_first():
    import pytorch_bayesiancnn_b200 as bbb
    net = _net(4)
    bbb.prune_by_snr(net, 0.5)
    first = [m.W_mask.clone() for m in _layers(net)]
    # make some pruned weights look strong: they stay pruned and count towards the total
    with torch.no_grad():
        for m in _layers(net):
            m.W_mu.masked_fill_(~m.W_mask, 100.0)
    out = bbb.prune_by_snr(net, 0.75)
    assert out["pruned"] == math.floor(0.75 * out["total"])
    for m, f in zip(_layers(net), first):
        assert not bool((m.W_mask & ~f).any())                  # nothing pruned before is kept now
    # a smaller fraction than already pruned leaves the masks as they are
    before = [m.W_mask.clone() for m in _layers(net)]
    out = bbb.prune_by_snr(net, 0.25)
    assert out["pruned"] == sum(int((~b).sum()) for b in before)
    for m, b in zip(_layers(net), before):
        assert torch.equal(m.W_mask, b)


def test_prune_by_snr_with_biases():
    import pytorch_bayesiancnn_b200 as bbb
    net = _net(5)
    out = bbb.prune_by_snr(net, 0.5, biases=True)
    assert out["total"] == 24 + 3 + 20 + 5
    assert out["per_layer"]["conv"][1] == 27 and out["per_layer"]["fc"][1] == 25
    pruned = sum(int((~m.W_mask).sum()) + int((~m.bias_mask).sum()) for m in _layers(net))
    assert pruned == out["pruned"] == 26


def test_set_weight_mask_refusals():
    import pytorch_bayesiancnn_b200 as bbb
    m = bbb.BBBLRTLinear(4, 3)
    with pytest.raises(ValueError, match="bool"):
        m.set_weight_mask(torch.ones(3, 4))
    with pytest.raises(ValueError, match="shape"):
        m.set_weight_mask(torch.ones(4, 3, dtype=torch.bool))
    with pytest.raises(ValueError, match="shape"):
        m.set_weight_mask(torch.ones(3, 4, dtype=torch.bool), torch.ones(4, dtype=torch.bool))
    with pytest.raises(ValueError, match="device"):
        m.set_weight_mask(torch.ones(3, 4, dtype=torch.bool, device="meta"))
    nb = bbb.BBBLRTLinear(4, 3, bias=False)
    with pytest.raises(ValueError, match="no bias"):
        nb.set_weight_mask(torch.ones(3, 4, dtype=torch.bool), torch.ones(3, dtype=torch.bool))
    # a mixture prior and a mask exclude each other, in either order
    m.set_mixture_prior()
    with pytest.raises(ValueError, match="mixture"):
        m.set_weight_mask(torch.ones(3, 4, dtype=torch.bool))
    m.clear_prior()
    m.set_weight_mask(torch.ones(3, 4, dtype=torch.bool))
    with pytest.raises(ValueError, match="mask"):
        m.set_mixture_prior()


def test_masks_are_buffers_set_in_place_and_round_trip_the_state_dict():
    import pytorch_bayesiancnn_b200 as bbb
    m = bbb.BBBConv2d(2, 3, 2)
    if m.W_mu.is_cuda:
        m = m.cpu()
    keys = set(m.state_dict())
    assert "W_mask" not in keys and m.mask_tensors() is None
    wm = torch.rand(m.W_mu.shape) > 0.5
    bm = torch.tensor([True, False, True])
    m.set_weight_mask(wm, bm)
    assert set(m.state_dict()) == keys | {"W_mask", "bias_mask"}
    ptr = m.W_mask.data_ptr()
    m.set_weight_mask(~wm, bm)                                  # same shapes: copied in place
    assert m.W_mask.data_ptr() == ptr and torch.equal(m.W_mask, ~wm)
    fresh = bbb.BBBConv2d(2, 3, 2).cpu()
    fresh.load_state_dict(m.state_dict())
    assert torch.equal(fresh.W_mask, ~wm) and torch.equal(fresh.bias_mask, bm)
    plain = bbb.BBBConv2d(2, 3, 2).cpu()
    plain.load_state_dict(bbb.BBBConv2d(2, 3, 2).cpu().state_dict())   # a checkpoint without masks loads as before
    assert plain.mask_tensors() is None
    m.set_weight_mask(wm)                                       # no bias mask: every bias kept again
    assert m.mask_tensors()[1] is None and "bias_mask" not in m.state_dict()
    m.clear_weight_mask()
    assert m.mask_tensors() is None and set(m.state_dict()) == keys


def test_guard_sees_masks_set_cleared_and_reallocated_but_not_in_place_updates():
    from pytorch_bayesiancnn_b200.modules import PriorGuard
    net = _net(6)
    conv, fc = _layers(net)
    g = PriorGuard(net)
    assert g.ok()
    conv.set_weight_mask(torch.ones(conv.W_mu.shape, dtype=torch.bool))
    assert not g.ok()
    g = PriorGuard(net)
    conv.set_weight_mask(torch.zeros(conv.W_mu.shape, dtype=torch.bool))      # in place
    assert g.ok()
    conv.clear_weight_mask()
    assert not g.ok()


def test_mask_ref_against_hand_computed_cases():
    # linear 2 -> 1, weights (mu, rho) = (0.5, 0), (NaN, 100): the second pruned; bias kept
    W_mu, W_rho = torch.tensor([[0.5, float("nan")]]), torch.tensor([[0.0, 100.0]])
    b_mu, b_rho = torch.tensor([0.25]), torch.tensor([-1.0])
    wm = torch.tensor([[True, False]])
    x = torch.tensor([[2.0, 3.0]])
    eps_w, eps_b = torch.tensor([[1.0, -7.0]]), torch.tensor([0.5])
    s0, sb = math.log1p(math.exp(0.0)), math.log1p(math.exp(-1.0))
    ref, _, _ = MR.layer_ref("bbb", x, W_mu, W_rho, b_mu, b_rho, wm, None, (eps_w, eps_b), None)
    assert abs(float(ref) - (2.0 * (0.5 + s0) + 0.25 + 0.5 * sb)) < 1e-12
    eps = torch.tensor([[2.0]])
    ref, _, sd = MR.layer_ref("lrt", x, W_mu, W_rho, b_mu, b_rho, wm, None, eps, None)
    sd_hand = math.sqrt(1e-16 + 4.0 * s0 ** 2 + sb ** 2)
    assert abs(float(sd) - sd_hand) < 1e-12
    assert abs(float(ref) - (2.0 * 0.5 + 0.25 + 2.0 * sd_hand)) < 1e-12
    pm, ps = 0.0, 0.1
    term = lambda mu, s: 0.5 * (2.0 * math.log(s / ps) - 1.0 + (ps / s) ** 2 + ((mu - pm) / s) ** 2)
    kl = float(MR.kl_ref(W_mu, W_rho, b_mu, b_rho, wm, None, pm, ps))
    assert abs(kl - (term(0.5, s0) + term(0.25, sb))) < 1e-9
    kl = float(MR.kl_ref(W_mu, W_rho, b_mu, b_rho, wm, torch.tensor([False]), pm, ps))
    assert abs(kl - term(0.5, s0)) < 1e-9
    assert float(MR.kl_ref(W_mu, W_rho, None, None, torch.zeros(1, 2, dtype=torch.bool), None, pm, ps)) == 0.0
    tb = lambda mu, s: math.log(ps / s) + (s * s + mu * mu) / (2 * ps * ps) - 0.5
    kl = float(MR.kl_ref(W_mu, W_rho, None, None, wm, None, pm, ps, "textbook"))
    assert abs(kl - tb(0.5, s0)) < 1e-9

"""Host side of the operand tiles prepared once per parameter version (fused.PrepCache, mc.MCForward(cache_prep=True)):
which chains are cached, and which updates move the version key the engine compares before every step."""
import types

import pytest
import torch


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()


def _net(variant):
    from pytorch_bayesiancnn_b200.models import get_model
    return get_model("alexnet", 3, 10, None, variant, "softplus")


def _steps(net, batch=64):
    from pytorch_bayesiancnn_b200 import fused
    return fused.plan(list(net.children()), (batch, 3, 32, 32))


def test_only_lrt_chains_are_cached(built):
    from pytorch_bayesiancnn_b200 import fused
    lrt, bbb = _steps(_net("lrt")), _steps(_net("bbb"))
    assert lrt is not None and bbb is not None
    assert fused.PrepCache.eligible(lrt)
    assert not fused.PrepCache.eligible(bbb)
    assert not fused.PrepCache.eligible(None)


def test_cache_covers_its_own_layers_only(built):
    from pytorch_bayesiancnn_b200 import fused
    net = _net("lrt")
    cache = fused.PrepCache(_steps(net), None, torch.device("cpu"))
    assert cache.covers(_steps(net)) and cache.covers(_steps(net, 128))
    assert not cache.covers(_steps(_net("lrt")))
    assert not cache.covers(_steps(net)[:-1])
    assert cache.kl.shape == (6,) and cache.ws == [None] * 6


def _key_of(net):
    """The version key of an engine whose prep cache holds `net`'s chain (mc.MCForward._prep_version)."""
    from pytorch_bayesiancnn_b200 import fused, mc
    eng = types.SimpleNamespace(_prep=fused.PrepCache(_steps(net), None, torch.device("cpu")), _prep_watch=None)
    return lambda: mc.MCForward._prep_version(eng)


@pytest.mark.parametrize("update", ["adam", "copy", "load_state_dict", "set_prior_in_place"])
def test_autograd_visible_updates_move_the_key(built, update):
    net = _net("lrt")
    if update == "set_prior_in_place":
        net.conv3.set_prior(0.0, 0.5)
    key = _key_of(net)
    k0 = key()
    assert key() == k0                                   # reading it changes nothing
    if update == "adam":
        opt = torch.optim.Adam(net.parameters(), lr=1e-3)
        for p in net.parameters():
            p.grad = torch.ones_like(p)
        opt.step()
    elif update == "copy":
        with torch.no_grad():
            net.classifier.bias_rho.copy_(net.classifier.bias_rho + 1.0)
    elif update == "load_state_dict":
        net.load_state_dict({k: v.clone() for k, v in net.state_dict().items()})
    else:
        net.conv3.set_prior(0.1, 0.4)
    k1 = key()
    assert k1 != k0
    assert key() == k1


def test_graph_step_refuses_missing_handles(built):
    """bbb_mc_graph_step checks its handles before any runtime call: a missing graph or event is BBB_E_INVALID."""
    from pytorch_bayesiancnn_b200 import _lib as L
    lib = L.lib()
    assert lib.bbb_mc_graph_step(None, None, None, None, None, None, 1, None, 1, 1) != 0
    assert b"NULL graph or event" in lib.bbb_last_error()
    assert lib.bbb_mc_graph_step(None, 2, None, None, None, 1, 1, None, 1, 1) != 0      # other stream, no in_ready


def test_writes_through_data_do_not_move_the_key(built):
    """The documented contract: a write through p.data is not seen (the layer KL cache has the same contract)."""
    net = _net("lrt")
    key = _key_of(net)
    k0 = key()
    net.conv1.W_mu.data.add_(1.0)
    assert key() == k0

"""The scale-mixture prior without a GPU: the float64 restatement of the Monte-Carlo KL (tests/kl_mc_ref.py) against
autograd, the textbook Gaussian KL (pi = 1) and numerical integration; the host surface of the layers (validation,
state_dict, one prior per layer, the guard of captured engines) and the argument checks of the C entry points."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
from scipy import integrate

from tests import kl_mc_ref as K


@pytest.fixture(scope="module")
def bbb():
    import __graft_entry__ as g
    g.build()
    import pytorch_bayesiancnn_b200 as pkg
    return pkg


def _rand(n, seed):
    g = torch.Generator().manual_seed(seed)
    return (0.3 * torch.randn(n, generator=g, dtype=torch.float64),
            -3.0 + torch.randn(n, generator=g, dtype=torch.float64),
            torch.randn(n, generator=g, dtype=torch.float64))


@pytest.mark.parametrize("pi,s1,s2", [(0.5, 1.0, math.exp(-6)), (0.25, 0.5, math.exp(-8)), (1.0, 0.3, 1.0)])
def test_closed_form_gradients_equal_autograd(pi, s1, s2):
    mu, rho, eps = _rand(257, 1)
    mu.requires_grad_(True)
    rho.requires_grad_(True)
    K.kl_terms(mu, rho, eps, pi, s1, s2).sum().backward()
    gm, gr = K.kl_mc_grads(mu.detach(), rho.detach(), eps, pi, s1, s2)
    torch.testing.assert_close(gm, mu.grad, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(gr, rho.grad, rtol=1e-10, atol=1e-12)


def test_pi_one_converges_to_the_gaussian_kl():
    n = 1 << 16
    eps = torch.randn(n, generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    for mu, sigma, ps in [(0.0, 0.05, 0.1), (0.3, 0.02, 1.0), (-0.2, 0.5, 0.3)]:
        rho = math.log(math.expm1(sigma))
        t = K.kl_terms(torch.full((n,), mu), torch.full((n,), rho, dtype=torch.float64), eps, 1.0, ps, 1.0)
        se = float(t.std()) / math.sqrt(n)
        assert abs(float(t.mean()) - K.gaussian_kl(mu, sigma, ps)) <= 4 * se + 1e-12


@pytest.mark.parametrize("s2", [math.exp(-6), math.exp(-7), math.exp(-8)])
@pytest.mark.parametrize("mu,sigma,pi,s1", [(0.0, 0.05, 0.5, 1.0), (0.1, 0.007, 0.25, 1.0), (-0.02, 0.001, 0.75, 0.5),
                                            (0.0005, 0.0003, 0.5, 1.0)])
def test_mean_over_draws_matches_quadrature(mu, sigma, pi, s1, s2):
    """E_q[log q - log p] by scipy.integrate.quad, per element."""
    def f(w):
        log_q = -math.log(sigma) - (w - mu) ** 2 / (2 * sigma ** 2)
        log_p = float(K.log_prior(torch.tensor(w, dtype=torch.float64), pi, s1, s2))
        return math.exp(log_q) / math.sqrt(2 * math.pi) * (log_q - log_p)
    lo, hi = mu - 12 * sigma, mu + 12 * sigma
    pts = sorted({p for p in (mu, 0.0, -4 * s2, 4 * s2) if lo < p < hi})
    want, err = integrate.quad(f, lo, hi, points=pts, limit=400)
    assert err < 1e-6 * max(1.0, abs(want))
    n = 1 << 16
    eps = torch.randn(n, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    rho = math.log(math.expm1(sigma))
    t = K.kl_terms(torch.full((n,), mu, dtype=torch.float64), torch.full((n,), rho, dtype=torch.float64), eps, pi, s1, s2)
    assert abs(float(t.mean()) - want) <= 4 * float(t.std()) / math.sqrt(n) + 1e-9


def test_draw_index_rule(bbb):
    from pytorch_bayesiancnn_b200 import functional as Fn
    for n_w in (1, 7, 2400):
        assert [Fn.kl_draw_index(n_w, n) for n in range(3)] == [0, 1, 2] == [K.draw_index(n_w, n) for n in range(3)]
        assert [Fn.kl_draw_index(n_w, n, bias=True) for n in range(3)] == [n_w, n_w + 1, n_w + 2]
        assert Fn.kl_draw_index(n_w, 5, bias=True) == K.draw_index(n_w, 5, bias=True)


def test_abi_struct_layout(bbb):
    from pytorch_bayesiancnn_b200 import _lib as L
    assert C.sizeof(L.MixturePrior) == 12
    assert [(n, getattr(L.MixturePrior, n).offset) for n, _ in L.MixturePrior._fields_] == [("pi", 0), ("sigma1", 4), ("sigma2", 8)]
    for name in ("bbb_kl_mc_forward", "bbb_kl_mc_backward", "bbb_kl_mc_workspace_bytes"):
        assert name in L.SYMBOLS and hasattr(L.lib(), name)


def test_entry_points_refuse_bad_arguments(bbb):
    """Return codes only: every refusal happens before a launch, so no GPU is needed (the pointers are never read)."""
    from pytorch_bayesiancnn_b200 import _lib as L
    lib, p = L.lib(), C.c_void_p(256)
    need = lib.bbb_kl_mc_workspace_bytes(3)
    assert need >= 3 * 4 + 3 * 8 and lib.bbb_kl_mc_workspace_bytes(16) > need

    def fwd(prior, n_draws=1, ws_bytes=1 << 24, w=p):
        return lib.bbb_kl_mc_forward(w, p, 4, None, None, 0, C.byref(L.MixturePrior(*prior)) if prior else None, 0, 0, None,
                                     n_draws, 0, p, p, ws_bytes, None)

    def bwd(prior, n_draws=1):
        return lib.bbb_kl_mc_backward(p, p, 4, 0, C.byref(L.MixturePrior(*prior)) if prior else None, 0, 0, None, n_draws,
                                      0, p, p, p, None)
    inf, nan = float("inf"), float("nan")
    for bad in [(0.0, 1, 1), (-0.1, 1, 1), (1.5, 1, 1), (nan, 1, 1), (0.5, 0, 1), (0.5, 1, 0), (0.5, -1, 1), (0.5, inf, 1),
                (0.5, 1, nan), (0.5, 1, 1e-30), None]:
        assert fwd(bad) == -1 and bwd(bad) == -1, bad
    ok = (0.5, 1.0, math.exp(-6))
    assert fwd(ok, n_draws=0) == -1 and bwd(ok, n_draws=0) == -1 and fwd(ok, n_draws=-3) == -1
    assert fwd(ok, n_draws=3, ws_bytes=need - 1) == -3
    assert fwd(ok, w=None) == -1
    assert b"workspace" in lib.bbb_last_error() or b"NULL" in lib.bbb_last_error()


@pytest.mark.parametrize("cls,args", [("BBBLinear", (5, 3)), ("BBBLRTLinear", (5, 3)), ("BBBConv2d", (2, 3, 3)),
                                      ("BBBLRTConv2d", (2, 3, 3))])
def test_layer_surface(bbb, cls, args):
    from pytorch_bayesiancnn_b200 import modules as M
    layer = getattr(bbb, cls)(*args)
    keys = list(layer.state_dict())
    assert keys == ["W_mu", "W_rho", "bias_mu", "bias_rho"] and layer.mixture_values() is None
    for bad in [dict(pi=0.0), dict(pi=1.01), dict(pi=float("nan")), dict(sigma1=0.0), dict(sigma2=-1.0),
                dict(sigma2=float("inf")), dict(sigma2=1e-30)]:
        with pytest.raises(ValueError):
            layer.set_mixture_prior(**bad)
    assert list(layer.state_dict()) == keys and layer.mixture_values() is None      # a refused call changes nothing
    v0 = layer._versions()
    layer.set_mixture_prior()
    want = tuple(np.float32(v).item() for v in (0.5, 1.0, math.exp(-6)))
    assert layer.mixture_values() == want and layer._versions() != v0 and layer._cfg(True)["mixture"] == want
    assert list(layer.state_dict()) == keys + ["mixture_prior"]
    assert layer.mixture_prior.dtype == torch.float32 and layer.mixture_prior.tolist() == list(want)
    assert M.has_mixture(layer) and M.prior_signature(layer) == (("mixture",) + want,)
    # a layer has one prior: each setter replaces the other, clear_prior goes back to the scalar prior
    layer.set_prior(0.0, 0.2)
    assert layer.mixture_values() is None and "mixture_prior" not in layer.state_dict() and layer.prior_tensors() is not None
    layer.set_mixture_prior(0.25, 2.0, 0.01)
    assert layer.prior_tensors() is None and "W_prior_mu" not in layer.state_dict()
    assert layer.mixture_values() == tuple(np.float32(v).item() for v in (0.25, 2.0, 0.01))
    # state_dict round trip into a fresh layer; a checkpoint without a mixture does not load into a layer that has one
    fresh = getattr(bbb, cls)(*args)
    fresh.load_state_dict(layer.state_dict())
    assert fresh.mixture_values() == layer.mixture_values() and torch.equal(fresh.mixture_prior, layer.mixture_prior)
    sd = {k: v.clone() for k, v in layer.state_dict().items()}
    sd["mixture_prior"][0] = 2.0
    with pytest.raises(RuntimeError, match="pi must be"):
        getattr(bbb, cls)(*args).load_state_dict(sd)
    layer.clear_prior()
    assert layer.mixture_values() is None and list(layer.state_dict()) == keys and not M.has_mixture(layer)
    with pytest.raises(RuntimeError):
        fresh.load_state_dict(layer.state_dict())
    assert layer.double().float().mixture_values() is None


def test_net_helper_and_guard(bbb):
    from pytorch_bayesiancnn_b200 import modules as M
    from pytorch_bayesiancnn_b200.models import BBBLeNet
    from tests.util import DEF_PRIORS
    net = BBBLeNet(10, 3, DEF_PRIORS, "lrt", "softplus")
    guard = M.PriorGuard(net)
    assert bbb.mixture_prior(net, 0.5, 1.0, math.exp(-7)) is net
    layers = [m for m in net.modules() if isinstance(m, M._BayesLayer)]
    assert len(layers) == 5 and all(m.mixture_values() == layers[0].mixture_values() for m in layers)
    assert not guard.ok()                                  # the prior kind changed: a captured engine must not replay
    guard = M.PriorGuard(net)
    bbb.mixture_prior(net, 0.5, 1.0, math.exp(-7))
    assert guard.ok()                                      # the same values again: what a graph holds is still right
    layers[2].set_mixture_prior(0.5, 1.0, math.exp(-6))
    assert not guard.ok()                                  # the values are kernel arguments of the captured launches
    with pytest.raises(bbb.EngineError, match="prior"):
        guard.check("engine")
    guard = M.PriorGuard(net)
    layers[0].clear_prior()                                # mixed nets are allowed; the guard sees the change
    assert not guard.ok() and M.has_mixture(net)
    moved = net.to(torch.float64).to(torch.float32)
    assert [m.mixture_values() for m in moved.modules() if isinstance(m, M._BayesLayer)][1] == layers[1].mixture_values()

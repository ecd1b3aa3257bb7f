"""Per-weight Gaussian priors (set_prior / posterior_as_prior, the bbb_prior C ABI) -- the host side, no GPU needed:
setting, checking and storing the prior, state_dict compatibility, KL-cache and captured-engine invalidation, the
ctypes mirror of the header and the argument refusals of the five *_prior entry points."""
import ctypes as C
import os
import re

import pytest
import torch

from tests.conftest import ROOT


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    return g.LIB


def _layers():
    import pytorch_bayesiancnn_b200 as bbb
    return [bbb.BBBConv2d(3, 8, 5, priors=None), bbb.BBBLRTLinear(7, 3, bias=False), bbb.BBBLRTConv2d(4, 6, 3)]


def test_set_prior_broadcasts_numbers_and_tensors():
    for m in _layers():
        ws = m.W_mu.shape
        row = torch.linspace(-1, 1, ws[-1])
        m.set_prior(mu=row, sigma=0.5)
        assert m.W_prior_mu.shape == ws and m.W_prior_mu.dtype == torch.float32 and m.W_prior_mu.is_contiguous()
        assert torch.equal(m.W_prior_mu.cpu(), row.expand(ws)) and bool((m.W_prior_sigma == 0.5).all())
        assert m.W_prior_mu.device == m.W_mu.device
        if m.use_bias:
            # a bias part left as None takes the layer's scalars
            assert bool((m.bias_prior_mu == float(m.prior_mu)).all()) and bool((m.bias_prior_sigma == float(m.prior_sigma)).all())
        else:
            assert m.prior_tensors()[2:] == (None, None)
        m.set_prior()                                      # all None: the scalars as tensors
        assert bool((m.W_prior_mu == float(m.prior_mu)).all()) and bool((m.W_prior_sigma == float(m.prior_sigma)).all())


def test_set_prior_refusals():
    m = _layers()[0]
    with pytest.raises(ValueError, match="broadcast"):
        m.set_prior(mu=torch.zeros(3, 3))
    with pytest.raises(ValueError, match="broadcast"):
        m.set_prior(bias_mu=torch.zeros(9))
    for bad in (0.0, -0.1, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="> 0"):
            m.set_prior(sigma=bad)
    s = torch.full(m.W_mu.shape, 0.2)
    s[0, 0, 0, 0] = float("nan")
    with pytest.raises(ValueError, match="W_prior_sigma"):
        m.set_prior(sigma=s)
    with pytest.raises(ValueError, match="bias_prior_sigma"):
        m.set_prior(bias_sigma=torch.zeros(8))
    with pytest.raises(ValueError, match="finite"):
        m.set_prior(mu=float("nan"))
    with pytest.raises(ValueError, match="no bias"):
        _layers()[1].set_prior(bias_mu=0.0)
    assert m.prior_tensors() is None                       # nothing was stored by a refused call


def test_set_prior_again_copies_in_place():
    m = _layers()[0]
    m.set_prior(mu=0.3, sigma=0.2, bias_mu=0.1, bias_sigma=0.4)
    ptrs = [t.data_ptr() for t in m.prior_tensors()]
    v0 = m._versions()
    m.set_prior(mu=torch.randn(m.W_mu.shape), sigma=0.7, bias_sigma=torch.full((8,), 0.9))
    assert [t.data_ptr() for t in m.prior_tensors()] == ptrs
    assert bool((m.W_prior_sigma == 0.7).all()) and bool((m.bias_prior_sigma == 0.9).all())
    assert bool((m.bias_prior_mu == 0.0).all())            # left as None: the scalar again, not the previous value
    assert m._versions() != v0
    m.clear_prior()
    assert m.prior_tensors() is None and "W_prior_mu" not in m.state_dict()


def test_versions_change_with_the_prior():
    m = _layers()[2]
    v0 = m._versions()
    m.set_prior(sigma=0.2)
    v1 = m._versions()
    assert v1 != v0
    m.set_prior(sigma=0.2)                                 # the same values, copied in place: a new version all the same
    assert m._versions() != v1
    m.clear_prior()
    assert m._versions() == v0


def test_state_dict_keys_and_round_trip():
    import pytorch_bayesiancnn_b200 as bbb
    m = bbb.BBBConv2d(3, 8, 5)
    assert list(m.state_dict().keys()) == ["W_mu", "W_rho", "bias_mu", "bias_rho"]
    n = bbb.BBBLRTLinear(7, 3, bias=False)
    assert list(n.state_dict().keys()) == ["W_mu", "W_rho"]
    m.set_prior(mu=torch.randn(8, 3, 5, 5), sigma=torch.rand(8, 3, 5, 5) + 0.1, bias_mu=torch.randn(8), bias_sigma=0.3)
    sd = m.state_dict()
    assert list(sd.keys()) == ["W_mu", "W_rho", "bias_mu", "bias_rho", "W_prior_mu", "W_prior_sigma", "bias_prior_mu",
                               "bias_prior_sigma"]
    fresh = bbb.BBBConv2d(3, 8, 5)
    fresh.load_state_dict(sd)
    for a, b in zip(fresh.prior_tensors(), m.prior_tensors()):
        assert torch.equal(a, b)
    # a checkpoint without a prior still loads into a fresh layer (drop-in compatibility)
    plain = bbb.BBBConv2d(3, 8, 5)
    plain.load_state_dict({k: v for k, v in sd.items() if "prior" not in k})
    assert plain.prior_tensors() is None


def test_posterior_as_prior_values():
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200.models import BBBLeNet
    from tests.util import CFG_PRIORS
    net = BBBLeNet(10, 3, CFG_PRIORS, "lrt", "softplus")
    assert bbb.posterior_as_prior(net) is net
    layers = [m for m in net.modules() if hasattr(m, "W_mu")]
    assert len(layers) == 5
    for m in layers:
        assert torch.equal(m.W_prior_mu, m.W_mu.detach())
        assert torch.equal(m.W_prior_sigma, torch.log1p(torch.exp(m.W_rho.detach())))
        assert torch.equal(m.bias_prior_mu, m.bias_mu.detach())
        assert torch.equal(m.bias_prior_sigma, torch.log1p(torch.exp(m.bias_rho.detach())))
        assert m.W_prior_mu.data_ptr() != m.W_mu.data_ptr()          # a copy, not a view of the parameter
    with torch.no_grad():
        layers[0].W_mu.add_(1.0)
    assert not torch.equal(layers[0].W_prior_mu, layers[0].W_mu)


def test_checkpoint_prior_of_another_shape_is_refused():
    import pytorch_bayesiancnn_b200 as bbb
    m = bbb.BBBConv2d(3, 8, 5)
    m.set_prior(sigma=0.3)
    sd = m.state_dict()
    for key, bad in (("W_prior_mu", torch.zeros(8, 3, 5)), ("bias_prior_sigma", torch.ones(9))):
        fresh = bbb.BBBConv2d(3, 8, 5)
        with pytest.raises(RuntimeError, match="size mismatch"):
            fresh.load_state_dict({**sd, key: bad})
    # a bias prior in the checkpoint of a bias-free layer is an unexpected key, not a buffer
    n = bbb.BBBLRTLinear(7, 3, bias=False)
    with pytest.raises(RuntimeError, match="Unexpected"):
        n.load_state_dict({**n.state_dict(), "W_prior_mu": torch.zeros(3, 7), "W_prior_sigma": torch.ones(3, 7),
                           "bias_prior_mu": torch.zeros(3)})


def test_prior_guard_follows_the_identity_of_the_buffers():
    """What a captured engine baked in (modules.PriorGuard): an in-place set_prior keeps it valid; a first set_prior,
    clear_prior, a re-allocation or a move does not -- and the guard keeps the buffers it saw alive."""
    from pytorch_bayesiancnn_b200.models import BBBLeNet
    from pytorch_bayesiancnn_b200.modules import PriorGuard, prior_signature
    from tests.util import CFG_PRIORS
    net = BBBLeNet(10, 3, CFG_PRIORS, "lrt", "softplus")
    layers = [m for m in net.modules() if hasattr(m, "W_mu")]
    g0 = PriorGuard(net)
    assert g0.ok() and prior_signature(net) == (None,) * 5
    layers[2].set_prior(sigma=0.2)                          # scalar -> tensor
    assert not g0.ok()
    g1 = PriorGuard(net)
    old = layers[2].W_prior_sigma
    layers[2].set_prior(sigma=0.3)                          # in place
    assert g1.ok() and layers[2].W_prior_sigma is old
    layers[2].clear_prior()                                 # tensor -> scalar: the guard still holds the old buffers
    assert not g1.ok() and any(t is old for t in g1.keep)
    layers[2].set_prior(sigma=0.3)
    g2 = PriorGuard(net)
    layers[2].set_prior(mu=torch.zeros(1))                  # the same shapes: in place again
    assert g2.ok()
    net.double()                                            # moves / re-allocates every buffer
    assert not g2.ok()


def test_prior_struct_mirrors_the_header(built):
    from pytorch_bayesiancnn_b200 import _lib as L
    hdr = open(os.path.join(ROOT, "include", "bbb_b200.h")).read()
    body = re.search(r"typedef struct bbb_prior \{(.*?)\} bbb_prior;", hdr, flags=re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = re.findall(r"const float\*\s*(\w+)", body)
    assert fields == ["w_mu", "w_sigma", "b_mu", "b_sigma"]
    assert [f for f, _ in L.Prior._fields_] == fields
    assert C.sizeof(L.Prior) == 4 * C.sizeof(C.c_void_p)
    lib = L.lib()
    for name in ("bbb_conv2d_forward_prior", "bbb_linear_forward_prior", "bbb_layer_forward_fused_prior",
                 "bbb_kl_forward_prior", "bbb_kl_backward_prior"):
        assert name in L.SYMBOLS and getattr(lib, name).argtypes[-1] is C.POINTER(L.Prior), name
        assert re.search(name + r"\(.*?const bbb_prior\* prior\);", hdr, flags=re.S), name


def _desc(bias=True):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    return Fn.make_desc((4, 3, 8, 8), (6, 3, 3, 3), ((1, 1), (1, 1), (1, 1)), L.VARIANT_LRT, True, bias, 0.0, 0.1,
                        L.MATH_BF16_TC)


FAKE = 0x10000          # a non-NULL pointer no call dereferences: every call below is refused on the host


def _msg():
    from pytorch_bayesiancnn_b200 import _lib as L
    return L.lib().bbb_last_error().decode()


def test_prior_entry_point_refusals(built):
    from pytorch_bayesiancnn_b200 import _lib as L
    lib = L.lib()
    f = C.c_void_p(FAKE)
    nul = L.Prior(None, None, None, None)
    w_only = L.Prior(FAKE, FAKE, None, None)
    no_sigma = L.Prior(FAKE, None, FAKE, FAKE)

    def conv(desc, prior):
        return lib.bbb_conv2d_forward_prior(C.byref(desc), f, f, f, f, f, f, f, None, None, None, 0, 0, None, f,
                                            C.c_size_t(1 << 30), None, prior)

    def fused(desc, prior):
        return lib.bbb_layer_forward_fused_prior(C.byref(desc), f, None, L.LAYOUT_NCHW_F32, 0, 1, f, f, f, f, f, None,
                                                 L.LAYOUT_NCHW_F32, 0, f, None, None, 0, 0, None, f,
                                                 C.c_size_t(1 << 30), None, prior)

    for call in (conv, fused):
        for prior, what in ((nul, "w_mu"), (no_sigma, "w_mu"), (w_only, "b_mu")):
            assert call(_desc(), C.byref(prior)) == -1                  # BBB_E_INVALID
            assert what in _msg(), (call.__name__, _msg())
    lin = _desc()
    assert lib.bbb_linear_forward_prior(C.byref(lin), f, f, f, f, f, f, f, None, None, None, 0, 0, None, f,
                                        C.c_size_t(1 << 30), None, C.byref(nul)) == -1
    # the stand-alone KL: weight pointers required, bias pointers when n_b > 0
    kf = lambda prior, n_b: lib.bbb_kl_forward_prior(f, f, 10, f if n_b else None, f if n_b else None, n_b, 0.0, 0.1, 0,
                                                      f, f, C.c_size_t(1 << 20), None, prior)
    assert kf(C.byref(nul), 0) == -1 and "w_mu" in _msg()
    assert kf(C.byref(w_only), 4) == -1 and "b_mu" in _msg()
    kb = lambda prior: lib.bbb_kl_backward_prior(f, f, 10, 0.0, 0.1, 0, f, f, f, None, prior)
    assert kb(C.byref(nul)) == -1 and "w_mu" in _msg()
    assert kb(C.byref(no_sigma)) == -1 and "w_mu" in _msg()
    # the scalar path of the new entry points keeps the old checks (prior_sigma > 0 without a tensor prior)
    assert lib.bbb_kl_forward_prior(f, f, 10, None, None, 0, 0.0, 0.0, 0, f, f, C.c_size_t(1 << 20), None, None) == -1
    assert "prior_sigma" in _msg()

"""Expected entropy and mutual information of the Monte-Carlo step without a GPU: the float64 reference against a
literal per-image loop, the generic torch.distributed path (2-rank gloo) against one process, and the host-side checks
of the C ABI (bbb_mc_exchange_info, BBB_MC_INFO)."""
import ctypes
import math
import os
import re
import socket
import tempfile

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from tests.conftest import ROOT
from tests.info_ref import information
from tests.util import CFG_PRIORS


def _per_image_loop(logits_per_sample, normalized):
    """get_uncertainty_per_image (uncertainty_estimation.py:37-58) style: one image at a time, numpy float64."""
    L = np.stack([np.asarray(l, dtype=np.float64) for l in logits_per_sample])          # [T, B, C]
    T, B, Cc = L.shape
    ee, mi = np.zeros(B), np.zeros(B)
    for b in range(B):
        net_out = L[:, b, :]
        if normalized:
            sp = np.where(net_out > 20, net_out, np.log1p(np.exp(np.minimum(net_out, 20))))
            p_hat = sp / sp.sum(1, keepdims=True)
        else:
            e = np.exp(net_out - net_out.max(1, keepdims=True))
            p_hat = e / e.sum(1, keepdims=True)
        p_bar = p_hat.mean(0)
        hs = []
        for t in range(T):
            hs.append(-sum(p * math.log(p) for p in p_hat[t] if p > 0))
        ee[b] = sum(hs) / T
        mi[b] = -sum(p * math.log(p) for p in p_bar if p > 0) - ee[b]
    return ee, mi


@pytest.mark.parametrize("normalized", [False, True])
def test_information_matches_per_image_loop(normalized):
    g = torch.Generator().manual_seed(1)
    logits = torch.randn(7, 9, 10, generator=g) * 3
    logits[:, 0, :] = torch.tensor([-200.0] * 9 + [0.0])         # softmax underflows to exactly 0 in 9 classes
    ee, mi = information(list(logits), normalized=normalized)
    ree, rmi = _per_image_loop(list(logits), normalized)
    assert ee.dtype == torch.float64 and mi.dtype == torch.float64
    assert np.abs(ee.numpy() - ree).max() < 1e-12 and np.abs(mi.numpy() - rmi).max() < 1e-12


@pytest.mark.parametrize("normalized", [False, True])
def test_mutual_info_zero_for_identical_samples_and_never_negative(normalized):
    g = torch.Generator().manual_seed(2)
    one = torch.randn(16, 100, generator=g) * 5
    one[3] = torch.tensor([-200.0] * 99 + [0.0])
    ee, mi = information([one] * 6, normalized=normalized)
    assert torch.isfinite(ee).all() and torch.isfinite(mi).all()
    assert mi.abs().max() < 1e-12
    logits = torch.randn(6, 16, 100, generator=g) * 5
    logits[:, 3, :] = torch.tensor([-200.0] * 99 + [0.0])
    ee, mi = information(list(logits), normalized=normalized)
    assert torch.isfinite(ee).all() and torch.isfinite(mi).all()
    assert (mi >= -1e-12).all()
    # total = expected + information, with the oracle's H[p_bar]
    from oracle import bbb_oracle as O
    ent = O.uncertainty(list(logits), normalized=normalized)[3]
    assert (ent - (ee + mi)).abs().max() < 1e-12


# --------------------------------------------------------------------------- #
# generic path: 2 ranks (gloo) == one process
# --------------------------------------------------------------------------- #
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _forward_fn():
    from oracle import bbb_oracle as O
    params = O.init_params("lenet", 10, 3, CFG_PRIORS, seed=5)
    shapes = O.eps_shapes("lenet", 10, 3, "lrt", 6)

    def fn(x, j):
        eps = O.draw_eps_like_reference(shapes, seed=1000 + j)      # noise keyed by the GLOBAL sample id
        return O.net_forward("lenet", params, x, eps, "lrt", "softplus", 0.0, 0.1, 10)
    return fn


def _worker(rank, world, port, num_ens, out_path):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"; os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.set_num_threads(1)
    from pytorch_bayesiancnn_b200 import mc
    x = torch.randn(6, 3, 32, 32, generator=torch.Generator().manual_seed(0))
    out, kl, unc = mc.mc_forward(_forward_fn(), x, num_ens, want_uncertainty=True, information=True)
    torch.save((out, kl, unc), out_path + f".{rank}")
    dist.destroy_process_group()


@pytest.mark.parametrize("num_ens", [1, 5])
def test_sharded_information_equals_single_process(num_ens):
    from pytorch_bayesiancnn_b200 import mc
    torch.set_num_threads(1)
    x = torch.randn(6, 3, 32, 32, generator=torch.Generator().manual_seed(0))
    fn = _forward_fn()
    logits = [fn(x, j)[0] for j in range(num_ens)]
    ree, rmi = information(logits)
    single = mc.mc_forward(fn, x, num_ens, want_uncertainty=True, information=True)
    assert len(single[2]) == 6
    base = mc.mc_forward(fn, x, num_ens, want_uncertainty=True)
    assert len(base[2]) == 4 and all(torch.equal(a, b) for a, b in zip(base[2], single[2][:4]))
    assert torch.equal(base[0], single[0])
    ee1, mi1 = single[2][4], single[2][5]
    assert ee1.shape == (6,) and torch.allclose(ee1.double(), ree, atol=1e-5) and torch.allclose(mi1.double(), rmi, atol=1e-5)
    assert torch.equal(mi1, single[2][3] - ee1)
    ctx = mp.get_context("spawn")
    port = _free_port()
    out_path = os.path.join(tempfile.mkdtemp(), "info")
    procs = [ctx.Process(target=_worker, args=(r, 2, port, num_ens, out_path)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=300)
        assert p.exitcode == 0
    res = [torch.load(out_path + f".{r}") for r in range(2)]
    for r in range(2):
        out, kl, unc = res[r]
        assert len(unc) == 6
        assert torch.allclose(out, single[0], atol=1e-5)
        for a, b in zip(unc, single[2]):
            assert torch.allclose(a, b, atol=1e-5)
        assert torch.allclose(unc[4].double(), ree, atol=1e-5) and torch.allclose(unc[5].double(), rmi, atol=1e-5)
    for a, b in zip(res[0][2], res[1][2]):
        assert torch.equal(a, b)                                    # every rank holds the same result


def test_information_needs_uncertainty():
    from pytorch_bayesiancnn_b200 import EngineError, mc
    x = torch.randn(6, 3, 32, 32)
    with pytest.raises(EngineError, match="want_uncertainty"):
        mc.mc_forward(_forward_fn(), x, 2, information=True)
    with pytest.raises(EngineError, match="want_uncertainty"):
        mc.MCForward(None, x, 2, want_information=True)


# --------------------------------------------------------------------------- #
# C ABI, host side only: every check runs before a launch
# --------------------------------------------------------------------------- #
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from pytorch_bayesiancnn_b200 import _lib
    return _lib.lib()


def test_info_flag_matches_header(lib):
    from pytorch_bayesiancnn_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "bbb_b200.h")).read()
    assert int(re.search(r"BBB_MC_INFO\s*=\s*(-?\d+)", hdr).group(1)) == _lib.MC_INFO == 4
    assert _lib.MC_INFO & (_lib.MC_MOMENTS | _lib.MC_NORMALIZED) == 0


def test_buffer_bytes_grow_only_with_info(lib):
    from pytorch_bayesiancnn_b200 import _lib as L
    for B, Cc, world in ((5, 10, 1), (2048, 10, 8), (1024, 100, 8), (700, 10, 4)):
        for norm in (0, L.MC_NORMALIZED):
            mom = L.MC_MOMENTS | norm
            # the parent layout: 2 slots x world x (planes * B * C + 2) words behind a 4096-byte control block
            assert lib.bbb_mc_buffer_bytes(B, Cc, norm, world) == 4096 + 2 * world * (2 * B * Cc + 2) * 8
            assert lib.bbb_mc_buffer_bytes(B, Cc, mom, world) == 4096 + 2 * world * (5 * B * Cc + 2) * 8
            # INFO: one more [B] plane per rank and slot
            assert lib.bbb_mc_buffer_bytes(B, Cc, mom | L.MC_INFO, world) == \
                lib.bbb_mc_buffer_bytes(B, Cc, mom, world) + 2 * world * B * 8
            assert lib.bbb_mc_buffer_bytes(B, Cc, norm | L.MC_INFO, world) == 0     # INFO needs MOMENTS


def _call_info(lib, flags, ee=None, mi=None):
    peers = (ctypes.c_void_p * 1)(0x1000)
    return lib.bbb_mc_exchange_info(None, 0, 1, 4, 10, None, 0, flags, None, ctypes.c_float(1.0), ctypes.c_float(0.0),
                                    0, 1, peers, 0x2000, 0x3000, None, None, None, None, None, None, None, 0, ee, mi, None)


def test_exchange_info_refusals_without_gpu(lib):
    from pytorch_bayesiancnn_b200 import _lib as L
    assert _call_info(lib, L.MC_INFO) == -1                                  # INFO without MOMENTS
    assert b"BBB_MC_MOMENTS" in lib.bbb_last_error()
    assert _call_info(lib, L.MC_INFO | L.MC_NORMALIZED, 0x4000, 0x5000) == -1
    for ee, mi in ((0x4000, None), (None, 0x5000), (0x4000, 0x5000)):     # new outputs without INFO
        assert _call_info(lib, L.MC_MOMENTS, ee, mi) == -1
        assert b"BBB_MC_INFO" in lib.bbb_last_error()

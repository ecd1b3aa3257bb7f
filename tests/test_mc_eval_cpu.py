"""Held-out evaluation of the Monte-Carlo step without a GPU: the float64 restatement of validate_model and of the
calibration figures against a literal per-image loop, read_metrics on a hand-built accumulator, and the host-side
checks of the C ABI (bbb_mc_exchange_metrics, bbb_mc_metrics_bytes, BBB_MC_CAL_BINS)."""
import ctypes
import math
import os
import re

import pytest
import torch

from tests import eval_ref as E
from tests.conftest import ROOT


def _batch(seed, B=37, Cc=10):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(B, Cc, generator=g, dtype=torch.float64) * 3
    logits[0] = torch.tensor([-200.0] * (Cc - 1) + [0.0], dtype=torch.float64)    # probabilities that underflow
    logits[1] = 0.0                                                                 # every class tied: argmax 0
    lo = torch.log_softmax(logits, 1)
    return lo, torch.randint(0, Cc, (B,), generator=g)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_batch_sums_match_per_image_loop(seed):
    lo, y = _batch(seed)
    s, r = E.batch_sums(lo, y), E.per_image_loop(lo, y)
    assert s["images"] == lo.shape[0]
    for k in ("nll", "correct", "brier"):
        assert math.isclose(s[k], r[k], rel_tol=1e-12), k
    for k in ("bin_count", "bin_conf", "bin_correct"):
        assert torch.allclose(s[k], torch.tensor(r[k], dtype=torch.float64), rtol=1e-12, atol=0), k
    assert int(s["bin_count"].sum()) == lo.shape[0]


def test_bins_are_right_closed_and_cover_the_unit_interval():
    mid = torch.tensor([(m + 0.5) / 15 for m in range(15)], dtype=torch.float64)
    assert E.bin_of(mid).tolist() == list(range(15))
    assert E.bin_of(torch.tensor([0.0, 1.0, 0.5 / 15 + 1e-3], dtype=torch.float64)).tolist() == [0, 14, 0]
    assert E.bin_of(torch.tensor([1.0 / 10], dtype=torch.float64)).item() == 1    # uniform over 10 classes


@pytest.mark.parametrize("beta_type", [0.1, "Blundell", "Soenderby", "Standard"])
def test_validate_matches_literal_loop(beta_type):
    from pytorch_bayesiancnn_b200 import mc
    batches = [_batch(10 + i, B=16 if i < 4 else 5) for i in range(5)]             # a ragged last batch
    los, ys = [b[0] for b in batches], [b[1] for b in batches]
    klsums = [1234.5] * 5
    loss, acc = E.validate(los, ys, klsums, 50000.0, beta_type, epoch=3, num_epochs=20)
    n, ref_loss, accs = len(batches), 0.0, []
    for i, (lo, y) in enumerate(zip(los, ys)):
        r = E.per_image_loop(lo, y)
        beta = mc.get_beta(i - 1, n, beta_type, 3, 20)
        assert beta == E.get_beta(i - 1, n, beta_type, 3, 20)
        ref_loss += r["nll"] / len(y) * 50000.0 + beta * klsums[i]
        accs.append(r["correct"] / len(y))
    assert math.isclose(loss, ref_loss / n, rel_tol=1e-12) and math.isclose(acc, sum(accs) / n, rel_tol=1e-12)
    # the accumulator's form of the loss: (train_size * sum nll_i + (sum beta_i) * klsum) / n
    nll_steps = sum(E.per_image_loop(lo, y)["nll"] / len(y) for lo, y in zip(los, ys))
    beta_sum = sum(mc.get_beta(i - 1, n, beta_type, 3, 20) for i in range(n))
    assert math.isclose(loss, (50000.0 * nll_steps + beta_sum * 1234.5) / n, rel_tol=1e-12)


def _hand_built(sums_list, klsum):
    """The accumulator words (include/bbb_b200.h, bbb_mc_exchange_metrics) of the given steps."""
    a = torch.zeros(64 + 64 * 48, dtype=torch.float64)
    for s in sums_list:
        B = s["images"]
        a[0] += 1; a[1] += B; a[2] += s["nll"] / B; a[3] += s["correct"] / B; a[4] += klsum
        a[5] += s["nll"]; a[6] += s["correct"]; a[7] += s["brier"]
        a[8:23] += s["bin_count"]; a[23:38] += s["bin_conf"]; a[38:53] += s["bin_correct"]
    return a


def test_read_metrics_on_hand_built_accumulator():
    from pytorch_bayesiancnn_b200 import mc
    sums = [E.batch_sums(*_batch(20 + i, B=16 if i < 3 else 7)) for i in range(4)]
    m = mc.read_metrics(_hand_built(sums, 99.5))
    ref = E.summarize(sums)
    assert m["steps"] == 4 and m["images"] == ref["images"] == 3 * 16 + 7
    assert math.isclose(m["klsum"], 99.5)
    for k in ("nll", "accuracy", "brier", "ece"):
        assert math.isclose(m[k], ref[k], rel_tol=1e-12), k
    assert m["bin_count"] == ref["bin_count"]
    for k in ("bin_confidence", "bin_accuracy"):
        for a, b in zip(m[k], ref[k]):
            assert (math.isnan(a) and math.isnan(b)) or math.isclose(a, b, rel_tol=1e-12), k
    assert any(math.isnan(v) for v in m["bin_confidence"])                      # empty bins are nan
    assert math.isclose(m["sum_acc_step"], sum(s["correct"] / s["images"] for s in sums), rel_tol=1e-12)
    empty = mc.read_metrics(torch.zeros(64 + 64 * 48, dtype=torch.float64))
    assert empty["steps"] == 0 and math.isnan(empty["nll"]) and math.isnan(empty["ece"])


# --------------------------------------------------------------------------- #
# C ABI, host side only: every check runs before a launch
# --------------------------------------------------------------------------- #
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from pytorch_bayesiancnn_b200 import _lib
    return _lib.lib()


def test_cal_bins_match_header_and_reference(lib):
    from pytorch_bayesiancnn_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "bbb_b200.h")).read()
    assert int(re.search(r"BBB_MC_CAL_BINS\s*=\s*(\d+)", hdr).group(1)) == _lib.MC_CAL_BINS == E.BINS == 15


def test_metrics_bytes(lib):
    # 64 accumulator words, then per-CTA partials of 3 + 3 * 15 = 48 words for up to 64 CTAs
    assert lib.bbb_mc_metrics_bytes() == (64 + 64 * 48) * 8


def _call(lib, labels, metrics, flags=0):
    peers = (ctypes.c_void_p * 1)(0x1000)
    return lib.bbb_mc_exchange_metrics(None, 0, 1, 4, 10, None, 0, flags, labels, ctypes.c_float(1.0),
                                       ctypes.c_float(0.0), 0, 1, peers, 0x2000, 0x3000, None, None, None, None, None,
                                       None, None, 0, None, None, 1, metrics, None)


def test_exchange_metrics_refusals_without_gpu(lib):
    from pytorch_bayesiancnn_b200 import _lib as L
    assert _call(lib, 0x4000, None) == -1
    assert b"metrics" in lib.bbb_last_error()
    assert _call(lib, None, 0x5000) == -1
    assert b"labels" in lib.bbb_last_error()
    assert _call(lib, None, None) == -1
    # the checks of bbb_mc_exchange_sharded still apply
    assert _call(lib, 0x4000, 0x5000, flags=L.MC_INFO) == -1
    assert b"BBB_MC_MOMENTS" in lib.bbb_last_error()

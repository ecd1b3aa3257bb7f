"""The per-layer Bayesian forward (bbb_conv2d_forward / bbb_linear_forward: weight_prep_kernel + gemm_tc_kernel in bf16
and tf32, fwd_simt_kernel in fp32) at every geometry of tests/forward_ref.CASES, against the float64 reference there.

For every case, variant and math mode the case is accepted on, calling the C ABI the way BayesLayerFn.forward does:
  - tight tier: the mean path (sample = 0) on the rounded operands within 1e-4 M; LRT: the variance plane on inputs
    with exact squares gives act_std^2 - 1e-16 = c_n sum x^2, one c_n per channel to 1e-4, and c_n the operand rounding
    of sigma_n^2 to 1e-4 (forward_ref.var_plane_err);
  - loose tier: the sampled layer within C (M + |ref|), act_std within 2u sd -- LRT with act_std requested (IEEE
    sqrtf) and without (sqrt.approx on the tensor cores);
  - every output element written and finite, the guard of sentinels behind y and act_std untouched;
  - the KL against oracle.kl_loss / kl_textbook in float64 to 1e-5 relative;
  - the path: bbb_launch_count moves by 2 on the tensor cores, 1 on fp32, 0 where the case is refused; auto runs the
    row's resolved mode bit for bit;
  - in-kernel Philox noise bit-identical to the same call fed philox_normal as external eps; two runs bit-identical;
  - folds: row block j of a folded call bit-identical to an unfolded call on stream stream_id + j * stride, and within
    the loose tier of float64 on sample j's noise.
Large cases (B >= 2048, folds) compare a fixed subset of images (forward_ref.check_images) with float64.
Run with -s to see the worst normalised error (<= 1 passes) per (math, tier)."""
import collections
import ctypes as C
import sys

import numpy as np
import pytest
import torch

from oracle import bbb_oracle as O
from tests import forward_ref as R

pytestmark = pytest.mark.gpu
GUARD = 1024
SENTINEL = 12345.678
_worst = collections.defaultdict(float)


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    yield torch.device("cuda:0")
    if _worst:
        lines = [f"  {fam:30s} worst normalised error = {v:.3e}" for fam, v in sorted(_worst.items())]
        sys.__stdout__.write("\n[layer forward geometry]\n" + "\n".join(lines) + "\n")


def _record(fam, e):
    _worst[fam] = max(_worst[fam], e)
    return e


Out = collections.namedtuple("Out", "rc y std kl launches")


def _guarded(shape, dev):
    n = int(np.prod(shape))
    buf = torch.full((n + GUARD,), float("nan"), dtype=torch.float32, device=dev)
    buf[n:] = SENTINEL
    return buf, buf[:n].view(shape)


def _check_written(buf, shape, what):
    n = int(np.prod(shape))
    assert bool((buf[n:] == SENTINEL).all()), f"{what}: the guard behind the output was written"
    assert bool(torch.isfinite(buf[:n]).all()), f"{what}: an unwritten (NaN) or non-finite element"


def _call(cs, variant, math, inp, sample, eps=None, seed=0, stream=0, base=None, want_std=False, fold=None,
          first_image=0, x=None):
    """One layer call on the engine, as BayesLayerFn.forward makes it.  Returns Out; rc != 0 leaves y etc. None."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    dev = inp[0].device
    x = inp[0] if x is None else x
    _, W_mu, W_rho, b_mu, b_rho = inp
    B = x.shape[0]
    conv = R.conv_of(cs)
    d = Fn.make_desc(tuple(x.shape), tuple(W_mu.shape), conv, L.VARIANT_LRT if variant == "lrt" else L.VARIANT_BBB,
                     sample, b_mu is not None, 0.0, 0.1, L.MATH_BY_NAME[math], L.KL_BY_NAME[cs.kl],
                     L.ACT_BY_NAME[cs.act], fold=None if fold is None else (fold, R.FOLD_STRIDE),
                     first_image=first_image)
    yshape = R.y_shape(cs, B)
    ybuf, y = _guarded(yshape, dev)
    sbuf, std = _guarded(yshape, dev) if want_std else (None, None)
    kl = torch.full((), float("nan"), dtype=torch.float32, device=dev)
    eps_a = eps_b = None
    if eps is not None:
        eps_a, eps_b = (eps[0].contiguous(), eps[1]) if variant == "bbb" else (eps.contiguous(), None)
    ws = Fn.workspace(dev, d)
    fn = L.lib().bbb_linear_forward if conv is None else L.lib().bbb_conv2d_forward
    n0 = L.launch_count()
    rc = fn(C.byref(d), Fn._ptr(x), Fn._ptr(W_mu), Fn._ptr(W_rho), Fn._ptr(b_mu), Fn._ptr(b_rho), Fn._ptr(y),
            Fn._ptr(kl), Fn._ptr(std), Fn._ptr(eps_a), Fn._ptr(eps_b), C.c_uint64(seed), C.c_uint64(stream),
            Fn._ptr(base), Fn._ptr(ws), C.c_size_t(ws.numel()), Fn._stream(dev))
    launches = L.launch_count() - n0
    if rc != 0:
        return Out(rc, None, None, None, launches)
    torch.cuda.synchronize()
    _check_written(ybuf, yshape, f"{cs.name} {variant} {math} y")
    if want_std:
        _check_written(sbuf, yshape, f"{cs.name} {variant} {math} act_std")
    assert launches == (1 if math == "fp32" or (math == "auto" and R.resolves(cs) == "fp32") else 2), launches
    return Out(rc, y, std, kl, launches)


def _philox_eps(cs, variant, seed, stream, B, first_image, has_bias, dev):
    """The noise the kernels draw in-kernel, from philox_normal: BBB the flat OIHW weight index, then N*K + n for the
    bias; LRT the NHWC-flat activation index of image first_image + b, returned NCHW."""
    from pytorch_bayesiancnn_b200 import functional as Fn
    if variant == "bbb":
        ws = R.w_shape(cs)
        nw = int(np.prod(ws))
        return (Fn.philox_normal(nw, seed, stream, 0, device=dev).view(ws),
                Fn.philox_normal(ws[0], seed, stream, nw, device=dev) if has_bias else None)
    shp = R.y_shape(cs, B)
    per = int(np.prod(shp[1:]))
    z = Fn.philox_normal(B * per, seed, stream, first_image * per, device=dev)
    if len(shp) == 2:
        return z.view(shp)
    return z.view(shp[0], shp[2], shp[3], shp[1]).permute(0, 3, 1, 2).contiguous()


def _kl_check(cs, inp, kl, math):
    _, W_mu, W_rho, b_mu, b_rho = (None if t is None else t.double() for t in inp)
    f = O.kl_loss if cs.kl == "reference" else O.kl_textbook
    ref = float(f(W_mu, W_rho, b_mu, b_rho, 0.0, 0.1))
    e = abs(float(kl) - ref) / abs(ref)
    assert _record(f"{math} kl (rel)", e) <= 1e-5, (cs.name, math, float(kl), ref)


def _loose(cs, variant, math, got_y, got_std, inp, eps, imgs, fam, x=None):
    """got_y / got_std: the outputs at images `imgs`; eps: the call's noise (LRT: all images of the call)."""
    xs = (inp[0] if x is None else x)[imgs]
    e_sub = eps if variant == "bbb" else eps[imgs]
    ref, M, sd = R.layer_ref(variant, xs, *inp[1:], e_sub, R.conv_of(cs), True, cs.act)
    e = R.loose_err(got_y, ref, M, math)
    assert _record(f"{math} loose y{fam}", e) <= 1, (cs.name, variant, math, fam, e)
    if got_std is not None:
        e = R.std_err(got_std, sd, math)
        assert _record(f"{math} act_std", e) <= 1, (cs.name, variant, math, e)


def _maths(cs):
    return [m for m in R.MATHS if m not in cs.refuse]


PARAMS = [(cs, v) for cs in R.CASES for v in cs.variants]


@pytest.mark.parametrize("cs,variant", PARAMS, ids=[f"{cs.name}-{v}" for cs, v in PARAMS])
def test_layer_forward_matches_float64(dev, cs, variant):
    idx = R.CASES.index(cs)
    g = torch.Generator(device=dev).manual_seed(1000 * idx + (variant == "lrt"))
    x, W_mu, W_rho, b_mu, b_rho, _ = R.make_inputs(cs, variant, g, dev)
    inp = (x, W_mu, W_rho, b_mu, b_rho)
    imgs = R.check_images(cs, idx)
    conv = R.conv_of(cs)
    lrt = variant == "lrt"
    seed, stream = 17 + idx, 5 + 3 * idx
    fold = cs.fold[0] if cs.fold else None
    first = cs.fold[1] if cs.fold else 0
    for math in R.MATHS:
        if math in cs.refuse:
            out = _call(cs, variant, math, inp, True, seed=seed, stream=stream, fold=fold, first_image=first)
            assert out.rc != 0 and out.launches == 0, (cs.name, math, out.rc)
            continue
        # ---- tight tier, the mean path (unfolded: a fold needs a sampling call)
        out = _call(cs, variant, math, inp, False)
        ref, M = R.mean_ref(x[imgs], W_mu, b_mu, conv, math, cs.act)
        assert _record(f"{math} tight mean", R.tight_err(out.y[imgs], ref, M)) <= 1, (cs.name, variant, math)
        _kl_check(cs, inp, out.kl, math)
        del out
        # ---- the sampled layer: in-kernel Philox, twice, then the same noise as external eps
        a = _call(cs, variant, math, inp, True, seed=seed, stream=stream, want_std=lrt, fold=fold, first_image=first)
        b = _call(cs, variant, math, inp, True, seed=seed, stream=stream, want_std=lrt, fold=fold, first_image=first)
        assert torch.equal(a.y, b.y) and torch.equal(a.kl, b.kl), "two runs differ"
        if lrt:
            assert torch.equal(a.std, b.std), "two runs differ (act_std)"
        del b
        _kl_check(cs, inp, a.kl, math)
        if math == R.resolves(cs):
            au = _call(cs, variant, "auto", inp, True, seed=seed, stream=stream, want_std=lrt, fold=fold,
                       first_image=first)
            assert torch.equal(au.y, a.y), f"auto did not run {math}"
            del au
        if fold is None:
            eps = _philox_eps(cs, variant, seed, stream, cs.B, 0, cs.bias, dev)
            c = _call(cs, variant, math, inp, True, eps=eps, want_std=lrt)
            assert torch.equal(c.y, a.y), "in-kernel noise differs from philox_normal fed as eps"
            if lrt:
                assert torch.equal(c.std, a.std)
            del c
            _loose(cs, variant, math, a.y[imgs], a.std[imgs] if lrt else None, inp, eps, imgs, "")
            if lrt:     # act_std not requested: the tensor-core epilogue takes sqrt.approx
                d = _call(cs, variant, math, inp, True, eps=eps, want_std=False)
                _loose(cs, variant, math, d.y[imgs], None, inp, eps, imgs, " (no act_std)")
                del d
            del eps
        else:
            S = cs.B // fold
            for j in range(S):
                xj = x[j * fold:(j + 1) * fold]
                u = _call(cs, variant, math, inp, True, seed=seed, stream=stream + j * R.FOLD_STRIDE, want_std=lrt,
                          first_image=first, x=xj)
                blk = slice(j * fold, (j + 1) * fold)
                assert torch.equal(a.y[blk], u.y), f"fold row block {j} differs from its unfolded call"
                if lrt:
                    assert torch.equal(a.std[blk], u.std), f"fold row block {j} (act_std)"
                assert torch.equal(a.kl, u.kl), "the folded KL differs from an unfolded call's"
                sub = [i - j * fold for i in imgs if j * fold <= i < (j + 1) * fold]
                if sub:
                    eps = _philox_eps(cs, variant, seed, stream + j * R.FOLD_STRIDE, fold, first, cs.bias, dev)
                    _loose(cs, variant, math, u.y[sub], u.std[sub] if lrt else None, inp, eps, sub, " (fold)", x=xj)
                    del eps
                del u
        del a
        torch.cuda.empty_cache()
        # ---- tight tier, the LRT variance plane
        if lrt:
            gv = torch.Generator(device=dev).manual_seed(7 + idx)
            xv, Wm, Wr, _, _, _ = R.make_inputs(cs, variant, gv, dev, var_plane=True)
            v = _call(cs, variant, math, (xv, Wm, Wr, None, None), True, seed=seed, stream=stream, want_std=True)
            spread, c_err = R.var_plane_err(v.std[imgs], xv[imgs], Wr, conv, math)
            assert _record(f"{math} tight var spread", spread) <= 1, (cs.name, math, spread)
            assert _record(f"{math} var c_n", c_err) <= 1, (cs.name, math, c_err)
            del v, xv
            torch.cuda.empty_cache()


STREAM_BASE_CASES = ["lenet_conv1_b256", "alexnet_conv2_b512", "edge_lin_k100_n70", "3conv3fc_conv3_b256"]


@pytest.mark.parametrize("name", STREAM_BASE_CASES)
def test_philox_with_device_stream_base(dev, name):
    """With a device stream base b the kernels draw from stream stream_id + b: the same bits as a call on that stream,
    and as philox_normal of it fed as external eps."""
    cs = next(c for c in R.CASES if c.name == name)
    idx = R.CASES.index(cs)
    for variant in cs.variants:
        g = torch.Generator(device=dev).manual_seed(31 + idx)
        inp = R.make_inputs(cs, variant, g, dev)[:5]
        base_v = (3 << 33) + 11
        base = torch.tensor([base_v], dtype=torch.int64, device=dev)
        for math in _maths(cs):
            lrt = variant == "lrt"
            a = _call(cs, variant, math, inp, True, seed=99, stream=4, base=base, want_std=lrt)
            b = _call(cs, variant, math, inp, True, seed=99, stream=4 + base_v, want_std=lrt)
            eps = _philox_eps(cs, variant, 99, 4 + base_v, cs.B, 0, cs.bias, dev)
            c = _call(cs, variant, math, inp, True, eps=eps, want_std=lrt)
            assert torch.equal(a.y, b.y) and torch.equal(a.y, c.y), (name, variant, math)
            if lrt:
                assert torch.equal(a.std, b.std) and torch.equal(a.std, c.std)

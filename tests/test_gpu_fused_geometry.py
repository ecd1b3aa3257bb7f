"""The fused tensor-core chain layer by layer, at every geometry its planner accepts, against a float64 reference.

Each case of CASES is one bbb_layer_forward_fused call, made the way fused.run_step makes it, on external eps and a
tiled packed input built by tests/fused_ref.pack_tiled.  It checks:
  - every output element against tests/fused_ref.layer_ref within C_BF16 * (M + |ref|) (and the x^2 plane against
    ref^2 when the layer writes it);
  - every element of rows < B is written and finite, the padding rows of the last 128-row block keep their NaN fill,
    and fp32 outputs leave a guard of sentinel floats behind them untouched;
  - the KL against oracle.kl_loss to 1e-5 relative;
  - LRT: the in-kernel Philox noise is bit-identical to the same call fed philox_normal as external eps.
The `why` of a case names the branch it exists for; test_case_table_covers_every_branch checks that together they reach
every map, kernel, channel count, batch, tile width, prep and output layout listed there.  Whole nets (fused_ref.NETS)
then check the planner's wiring end to end, and the nets it must refuse run correctly unfused.
Run with -s to see the worst normalised error per case family."""
import collections
import sys

import pytest
import torch

from tests import fused_ref as R
from tests.fused_ref import CASES, GUARD, SENTINEL, _alloc_out, _layer, _out_hw, _prep, _step, _tile_bn
from tests.fused_ref import fused_call as _call
from tests.util import scale_err

def test_case_table_covers_every_branch():
    tap = [c for c in CASES if c.kind == "tap"]
    tg = tap + [c for c in CASES if c.kind == "linear"]
    assert {c.hw for c in tg} == {(1, 1), (2, 2), (4, 4), (8, 8), (4, 8)}
    assert {(c.k, c.s, c.p) for c in tap} == {(1, 1, 0), (3, 1, 0), (3, 1, 1), (5, 1, 2), (3, 2, 1)}
    assert {c.cin for c in tap} == {64, 128, 192, 256}
    assert {c.cout for c in tg if c.out == "packed"} >= {64, 128, 192, 320}
    assert {c.cout for c in tg if c.out == "f32"} >= {10, 72, 100}
    assert {(c.variant, c.act) for c in tg} == {(v, a) for v in ("bbb", "lrt") for a in ("none", "relu", "softplus")}
    assert {(c.variant, c.pool) for c in tap} == {(v, p) for v in ("bbb", "lrt") for p in (False, True)}
    assert {c.sq for c in tg if c.out == "packed"} == {False, True}
    assert {c.wide for c in tg} == {0, 1}
    assert {(c.pool, _tile_bn(c)) for c in tg if c.out == "packed"} == {(p, bn) for p in (False, True) for bn in (64, 128)}
    assert {c.B for c in tg} >= {1, 127, 128, 129, 300}
    # the bulk-copy store (unpooled packed, a full 128-row tile) and the direct store of a ragged last tile
    assert any(not c.pool and c.out == "packed" and c.B >= 128 and c.B % 128 for c in tg)
    assert {_prep(c) for c in tg} == {"tap_prep_conv_kernel", "tap_prep_kernel"}
    assert {c.prev_hw for c in tg if c.kind == "linear"} == {1, 4, 6, 8}
    gat = [c for c in CASES if c.kind == "gather"]
    assert {c.cin for c in gat} >= {1, 3, 16} and {c.hw for c in gat} >= {(8, 8), (4, 8)}
    assert {c.out for c in gat if c.pool} == {"packed", "f32"}
    s4 = [c for c in CASES if c.kind == "s4"]
    assert {c.cin for c in s4} == {1, 3, 4} and {(c.k, c.p) for c in s4} == {(11, 5), (7, 3)}
    assert {c.hw for c in s4} == {(32, 32), (48, 32), (64, 32)}      # 64x64 has OW = 16: the gather case above
    assert {c.B for c in s4} == {1, 15, 16, 17, 200}


# --------------------------------------------------------------------------------------------- per-layer GPU tests
_worst = collections.defaultdict(float)


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    yield torch.device("cuda:0")
    if _worst:
        lines = [f"  {fam:8s} worst |y - ref| / (C (M + |ref|)) = {v:.3f}" for fam, v in sorted(_worst.items())]
        sys.__stdout__.write("\n[fused geometry]\n" + "\n".join(lines) + "\n")


@pytest.mark.gpu
@pytest.mark.parametrize("cs", CASES, ids=[c.name for c in CASES])
def test_fused_layer_matches_float64_reference(dev, cs):
    from oracle import bbb_oracle as O
    from pytorch_bayesiancnn_b200 import _lib as L, philox_normal
    idx = CASES.index(cs)
    g = torch.Generator().manual_seed(1000 + idx)
    m = _layer(cs)
    with torch.no_grad():
        R.init_layer_params(m, m.W_mu[0].numel(), g)
    m = m.to(dev)
    st = _step(cs, m)
    if cs.kind in ("gather", "s4"):
        assert R.nchw_path(st) == cs.kind
    B, cout, (oh, ow) = cs.B, cs.cout, _out_hw(cs)

    # input: bf16-representable values; a packed input carries x^2 for an LRT layer, its padding rows are NaN
    if cs.kind == "linear":
        x = R.bf16(torch.randn(B, cs.cin, generator=g))                       # reference feature order c*HW + pix
        cols = x.view(B, cs.cin // cs.prev_hw, cs.prev_hw).transpose(1, 2).reshape(B, -1)
    else:
        x = R.bf16(torch.randn((B, cs.cin) + tuple(cs.hw), generator=g))
        cols = R.nchw_to_cols(x)
    if st.in_layout == L.LAYOUT_PACKED_BF16:
        xin = R.pack_tiled(cols, 2 if cs.variant == "lrt" else 1).to(dev)
        xin_sq = xin.view(-1)[8192:] if cs.variant == "lrt" else None
    else:
        xin, xin_sq = x.float().to(dev), None

    pre_shape = (B, cout) if cs.kind == "linear" else (B, cout, oh, ow)
    if cs.variant == "lrt":
        ea, eb = torch.randn(pre_shape, generator=g), None
    else:
        ea, eb = torch.randn(m.W_mu.shape, generator=g), torch.randn(cout, generator=g)
    conv = None if cs.kind == "linear" else ((cs.s, cs.s), (cs.p, cs.p))
    p = [t.detach().cpu() for t in (m.W_mu, m.W_rho, m.bias_mu, m.bias_rho)]
    ref, mag = R.layer_ref(x, *p, cs.variant, ea, eb, conv=conv, act=cs.act, pool=cs.pool)

    prev = L.lib().bbb_set_wide_tiles(cs.wide)
    try:
        y, y_sq, n = _alloc_out(cs, st, dev)
        kl = _call(st, xin, xin_sq, y, y_sq, ea.to(dev), None if eb is None else eb.to(dev))
        torch.cuda.synchronize()
        if cs.variant == "lrt":
            # in-kernel Philox vs the same stream drawn by philox_normal (NHWC-flat element index of the pre-pool output)
            seed, stream = 77, 500 + idx
            z = philox_normal(int(torch.Size(pre_shape).numel()), seed, stream, 0, device=dev)
            if cs.kind != "linear":
                z = z.view(B, oh, ow, cout).permute(0, 3, 1, 2)
            z = z.reshape(pre_shape).contiguous()
            y1, y1_sq, _ = _alloc_out(cs, st, dev)
            _call(st, xin, xin_sq, y1, y1_sq, None, None, seed, stream)
            y2, y2_sq, _ = _alloc_out(cs, st, dev)
            _call(st, xin, xin_sq, y2, y2_sq, z, None, seed, stream)
            torch.cuda.synchronize()
    finally:
        L.lib().bbb_set_wide_tiles(prev)

    fam = cs.kind
    if cs.out == "packed":
        F_ = st.out_chw[0] * st.out_chw[1] * st.out_chw[2]
        planes = 2 if cs.sq else 1
        refc = ref if cs.kind == "linear" else R.nchw_to_cols(ref)
        magc = mag if cs.kind == "linear" else R.nchw_to_cols(mag)
        yc = R.unpack_tiled(y, B, F_, planes)
        assert bool(torch.isfinite(yc).all()), "rows < B not all written / not finite"
        err = R.norm_err(yc, refc, magc)
        if cs.sq:
            ys = R.unpack_tiled(y, B, F_, planes, plane=1)
            assert bool(torch.isfinite(ys).all())
            err_sq = R.norm_err(ys, refc * refc, R.sq_mag(refc, magc))
            assert err_sq <= 1.0, f"x^2 plane: {err_sq:.3f}"
            _worst[fam + "^2"] = max(_worst[fam + "^2"], err_sq)
        pad = R.padding_bits(y, B, F_, planes)
        assert bool((pad == R.BF16_NAN_BITS).all()), "padding rows of the last row tile were written"
    else:
        out = y[:n].cpu().double().view(ref.shape)
        assert bool(torch.isfinite(out).all()), "outputs not all written / not finite"
        err = R.norm_err(out, ref, mag)
        assert bool((y[n:].cpu() == SENTINEL).all()), "the guard behind the fp32 output was written"
    _worst[fam] = max(_worst[fam], err)
    assert err <= 1.0, f"{cs.name}: normalised error {err:.3f}"

    kl_ref = float(O.kl_loss(*[t.double() for t in p], m.prior_mu, m.prior_sigma))
    assert abs(float(kl) - kl_ref) <= 1e-5 * abs(kl_ref), (float(kl), kl_ref)

    if cs.variant == "lrt":
        bits = torch.int16 if cs.out == "packed" else torch.int32
        assert torch.equal(y1.view(bits), y2.view(bits)), "in-kernel Philox noise differs from philox_normal"
        if cs.out == "packed":
            assert bool(torch.isfinite(R.unpack_tiled(y1, B, F_, planes)).all())


# --------------------------------------------------------------------------------------------- whole nets
@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["lrt", "bbb"])
@pytest.mark.parametrize("name", sorted(R.NETS) + sorted(R.REFUSED_NETS))
def test_whole_net_matches_float64_oracle(dev, name, variant):
    """The planner's wiring (layouts, pitches, prev_hw, y_sq selection) end to end: the fused chain (math='auto',
    no_grad) and the same net with fuse=False against an fp64 composition of the oracle's layers on identical eps.
    The nets the planner refuses must run unfused and still match."""
    import pytorch_bayesiancnn_b200 as bbb
    fusable = name in R.NETS
    shape, spec = R.NETS[name] if fusable else R.REFUSED_NETS[name]
    seed = sorted(list(R.NETS) + list(R.REFUSED_NETS)).index(name)
    net = R.make_net(spec, variant, seed=seed).to(dev)
    net.set_flag("math", "auto")
    x = R.bf16(torch.randn(shape, generator=torch.Generator().manual_seed(50 + seed))).float()
    eps = R.net_eps(net, shape, variant, seed=90 + seed)
    ref, kl_ref = R.net_ref(net, x, eps, variant)
    with torch.no_grad(), bbb.external_eps(eps):
        out, kl = net(x.to(dev))
    torch.cuda.synchronize()
    assert (net._fused_plans.get(tuple(shape)) is not None) == fusable
    assert tuple(out.shape) == tuple(ref.shape)
    assert bool(torch.isfinite(out).all())
    assert scale_err(out, ref) < 1e-2, scale_err(out, ref)
    assert abs(float(kl) - kl_ref) <= 1e-5 * abs(kl_ref)
    net.set_flag("fuse", False)
    with torch.no_grad(), bbb.external_eps(eps):
        out2, kl2 = net(x.to(dev))
    torch.cuda.synchronize()
    assert scale_err(out2, ref) < 1e-2, scale_err(out2, ref)
    assert abs(float(kl2) - kl_ref) <= 1e-5 * abs(kl_ref)

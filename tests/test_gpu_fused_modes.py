"""The fused tensor-core chain's call modes, layer by layer, at every geometry of tests/fused_ref.CASES.

tests/test_gpu_fused_geometry.py checks each case in one mode: phase 0, no fold, image 0, external eps.  The chain also
runs split into a PREP_ONLY and a SKIP_PREP call (fused.run_step, fused.PrepCache), folds Monte-Carlo samples into the
batch (mc.MCForward), starts at a row block's first image, reads its Philox stream from a device base (captured graphs),
draws BBB weights in-kernel, and takes a pruning mask and a tensor prior.  Each test here runs one of those modes at
every case that accepts it, with the geometry test's checks on every output (rows < B written and finite, padding rows
still NaN, fp32 guard sentinels untouched), and compares it bit for bit with the call that must give the same bits, or
with tests/fused_ref.layer_ref within its bar (norm_err <= 1).  Run with -s to see the worst normalised error per
(mode, kind)."""
import collections
import sys

import pytest
import torch

from tests import fused_ref as R
from tests import mask_ref as MR
from tests.fused_ref import CASES

pytestmark = pytest.mark.gpu

IDS = [c.name for c in CASES]
BBB_CASES = [c for c in CASES if c.variant == "bbb"]
FOLD_CASES = [c for c in CASES if R.folds(c)]
SEED = 0x5EED_0001
STREAM = (1 << 32) - 2          # just below 2^32: stream + base and stream + j * stride carry into the high word
STRIDE = (1 << 40) + 3          # bits above 2^32, as the engine's world << 40
BIAS_SIGMA = 1.0                # the BBB noise test's bias sigma
BASE = 5                        # device stream base: STREAM + BASE = 2^32 + 3
_worst = collections.defaultdict(float)


@pytest.fixture(scope="module")
def dev():
    import __graft_entry__ as g
    g.build()
    yield torch.device("cuda:0")
    if _worst:
        lines = [f"  {mode:12s} {kind:7s} worst {v:.3g}" for (mode, kind), v in sorted(_worst.items())]
        sys.__stdout__.write("\n[fused modes] y: |y - ref| / (C (M + |ref|)); kl: relative error\n"
                             + "\n".join(lines) + "\n")


class _Layer:
    """One case's layer on the device, its inputs and calls."""

    def __init__(self, cs, dev, bias_sigma=None):
        self.cs, self.dev = cs, dev
        self.idx = CASES.index(cs)
        self.g = torch.Generator().manual_seed(4000 + self.idx)
        m = R._layer(cs)
        with torch.no_grad():
            R.init_layer_params(m, m.W_mu[0].numel(), self.g, bias_sigma)
        self.m = m.to(dev)
        self.conv = None if cs.kind == "linear" else ((cs.s, cs.s), (cs.p, cs.p))
        self.oh, self.ow = R._out_hw(cs)
        self.lrt = cs.variant == "lrt"

    def step(self, B):
        return R._step(self.cs, self.m, B)

    def params(self):
        return [t.detach().cpu() for t in (self.m.W_mu, self.m.W_rho, self.m.bias_mu, self.m.bias_rho)]

    def x(self, rows):
        """float64 input of `rows` images, bf16-representable (linear: reference feature order c*HW + pix)."""
        cs = self.cs
        if cs.kind == "linear":
            return R.bf16(torch.randn(rows, cs.cin, generator=self.g))
        return R.bf16(torch.randn((rows, cs.cin) + tuple(cs.hw), generator=self.g))

    def xin(self, x):
        """(x, x_sq) device operands of a float64 input: tiled packed (+ its square for an LRT layer) or NCHW fp32."""
        cs = self.cs
        if cs.kind in ("gather", "s4"):
            return x.float().to(self.dev), None
        B = x.shape[0]
        cols = (x.view(B, cs.cin // cs.prev_hw, cs.prev_hw).transpose(1, 2).reshape(B, -1) if cs.kind == "linear"
                else R.nchw_to_cols(x))
        buf = R.pack_tiled(cols, 2 if self.lrt else 1).to(self.dev)
        return buf, (buf.view(-1)[8192:] if self.lrt else None)

    def run(self, B, xin, **kw):
        """One call on B rows; returns (y, kl)."""
        st = self.step(B)
        y, y_sq, _ = R._alloc_out(self.cs, st, self.dev, B)
        kl = R.fused_call(st, xin[0], xin[1], y, y_sq, **kw)
        return y, kl

    def bits(self, y, B):
        """[B, F * planes] int bits of the output rows, after the geometry test's checks of the whole buffer."""
        cs = self.cs
        cout, oh, ow = self.step(B).out_chw
        F_ = cout * oh * ow
        if cs.out == "packed":
            planes = 2 if cs.sq else 1
            flat = y.reshape(-1).cpu().view(torch.int16)
            v = [R.unpack_tiled(y, B, F_, planes, p) for p in range(planes)]
            assert all(bool(torch.isfinite(t).all()) for t in v), "rows < B not all written / not finite"
            assert bool((R.padding_bits(y, B, F_, planes) == R.BF16_NAN_BITS).all()), "padding rows were written"
            return torch.cat([flat[R.tiled_index(B, F_, planes, p)] for p in range(planes)], 1)
        n = B * F_
        yc = y.cpu()
        assert bool(torch.isfinite(yc[:n]).all()), "outputs not all written / not finite"
        assert bool((yc[n:] == R.SENTINEL).all()), "the guard behind the fp32 output was written"
        return yc[:n].view(torch.int32).view(B, F_)

    def values(self, y, B):
        """The output rows as float64 in the reference's shape (NCHW, or [B, N])."""
        cs = self.cs
        cout, oh, ow = self.step(B).out_chw
        if cs.out == "packed":
            v = R.unpack_tiled(y, B, cout * oh * ow, 2 if cs.sq else 1)
            return v if cs.kind == "linear" else R.cols_to_nchw(v, cout, oh, ow)
        return y[:B * cout * oh * ow].cpu().double().view((B, cout) if cs.kind == "linear" else (B, cout, oh, ow))

    def philox_eps(self, rows, seed, stream, first_image=0):
        """(eps_a, eps_b) of an in-kernel call, drawn by philox_normal: BBB weights at the flat OIHW index and the bias at
        N*K + n; LRT activations at the NHWC-flat index of the pre-pool output, from image `first_image` on."""
        from pytorch_bayesiancnn_b200 import philox_normal
        m, N = self.m, self.cs.cout
        if not self.lrt:
            nk = m.W_mu.numel()
            z = philox_normal(nk + N, seed, stream, 0, device=self.dev)
            return z[:nk].view(m.W_mu.shape), z[nk:]
        per = self.oh * self.ow * N
        z = philox_normal(rows * per, seed, stream, first_image * per, device=self.dev)
        if self.cs.kind == "linear":
            return z.view(rows, N), None
        return z.view(rows, self.oh, self.ow, N).permute(0, 3, 1, 2).contiguous(), None

    def check_ref(self, mode, y, B, x, ea, eb, params=None):
        """y within the float64 bar of layer_ref on the same eps (params: float64 (W_mu, W_rho, b_mu, b_rho))."""
        cs = self.cs
        p = self.params() if params is None else params
        ref, mag = R.layer_ref(x, *p, cs.variant, ea.cpu(), None if eb is None else eb.cpu(), conv=self.conv,
                               act=cs.act, pool=cs.pool)
        err = R.norm_err(self.values(y, B), ref, mag)
        _worst[(mode, cs.kind)] = max(_worst[(mode, cs.kind)], err)
        assert err <= 1.0, f"{mode}: normalised error {err:.3f}"

    def check_kl(self, mode, kl, ref):
        rel = abs(float(kl) - float(ref)) / abs(float(ref))
        _worst[(mode + " kl", self.cs.kind)] = max(_worst[(mode + " kl", self.cs.kind)], rel)
        assert rel <= 1e-5, (mode, float(kl), float(ref))

    def fold_rows(self):
        """(rows per sample, samples) of a fold: LRT 3 samples of the case's batch (ragged 128-row tiles straddle
        samples); BBB 2 samples of 128 or 256 rows (a row tile multiplies by one weight sample)."""
        if self.lrt:
            return self.cs.B, 3
        return (256 if self.cs.B > 128 else 128), 2

    def fold_input(self, rows, S):
        """(x of every row block, device input of the fold): the stride-4 kernel's NCHW input holds `rows` images."""
        if self.cs.kind == "s4":
            x = self.x(rows)
            return [x] * S, self.xin(x)
        x = self.x(rows * S)
        return [x[j * rows:(j + 1) * rows] for j in range(S)], self.xin(x)


def _same(a, b, what):
    assert torch.equal(a, b), f"{what}: {int((a != b).sum())} of {a.numel()} output words differ"


def _eq_kl(a, b, what):
    assert float(a) == float(b), (what, float(a), float(b))


# --------------------------------------------------------------------------------------------- in-kernel BBB noise
@pytest.mark.parametrize("cs", BBB_CASES, ids=[c.name for c in BBB_CASES])
def test_in_kernel_bbb_noise_is_philox_normal(dev, cs):
    """In-kernel BBB weight and bias noise = philox_normal fed as eps_a (flat OIHW index, the reference's order also
    where prev_hw > 1 permutes the packed features) and eps_b (element N*K + n), bit for bit; and within the float64
    bar, with a bias sigma of 1 so the bar sees the bias draw too (test_fused_modes_cpu)."""
    s = _Layer(cs, dev, bias_sigma=BIAS_SIGMA)
    x = s.x(cs.B)
    xin = s.xin(x)
    with R.wide_tiles(cs.wide):
        y1, kl1 = s.run(cs.B, xin, seed=SEED, stream=STREAM)
        ea, eb = s.philox_eps(cs.B, SEED, STREAM)
        y2, kl2 = s.run(cs.B, xin, eps_a=ea, eps_b=eb)
    _same(s.bits(y1, cs.B), s.bits(y2, cs.B), "in-kernel vs philox_normal eps")
    _eq_kl(kl1, kl2, "KL")
    s.check_ref("bbb noise", y1, cs.B, x, ea, eb)


# --------------------------------------------------------------------------------------------- device stream base
@pytest.mark.parametrize("cs", CASES, ids=IDS)
def test_device_stream_base(dev, cs):
    """stream_id + *stream_base (read on the device, carrying across 2^32) = that sum passed as stream_id, bit for bit;
    folded too."""
    s = _Layer(cs, dev)
    base = torch.tensor([BASE], dtype=torch.int64, device=dev)
    runs = [(cs.B, None, s.xin(s.x(cs.B)))]
    if R.folds(cs):
        rows, S = s.fold_rows()
        runs.append((rows * S, (rows, STRIDE), s.fold_input(rows, S)[1]))
    with R.wide_tiles(cs.wide):
        for B, fold, xin in runs:
            y1, kl1 = s.run(B, xin, seed=SEED, stream=STREAM, stream_base=base, fold=fold)
            y2, kl2 = s.run(B, xin, seed=SEED, stream=STREAM + BASE, fold=fold)
            _same(s.bits(y1, B), s.bits(y2, B), f"stream base, fold {fold}")
            _eq_kl(kl1, kl2, "KL")


# --------------------------------------------------------------------------------------------- split phases
@pytest.mark.parametrize("cs", CASES, ids=IDS)
def test_split_phases_equal_one_call(dev, cs):
    """PREP_ONLY then SKIP_PREP on one workspace = phase 0 (y, y_sq and KL), unfolded and folded."""
    from pytorch_bayesiancnn_b200 import _lib as L
    s = _Layer(cs, dev)
    runs = [(cs.B, None, s.xin(s.x(cs.B)))]
    if R.folds(cs):
        rows, S = s.fold_rows()
        runs.append((rows * S, (rows, STRIDE), s.fold_input(rows, S)[1]))
    with R.wide_tiles(cs.wide):
        for B, fold, xin in runs:
            st = s.step(B)
            y0, kl0 = s.run(B, xin, seed=SEED, stream=STREAM, fold=fold)
            ws = _fresh_ws(st, fold, dev)
            klp = R.fused_call(st, None, None, None, None, seed=SEED, stream=STREAM, phase=L.FUSED_PREP_ONLY, fold=fold,
                               ws=ws)
            y1, _ = s.run(B, xin, seed=SEED, stream=STREAM, phase=L.FUSED_SKIP_PREP, fold=fold, ws=ws)
            _same(s.bits(y1, B), s.bits(y0, B), f"PREP_ONLY + SKIP_PREP vs phase 0, fold {fold}")
            _eq_kl(klp, kl0, "KL of the PREP_ONLY call")


@pytest.mark.parametrize("cs", CASES, ids=IDS)
def test_prepared_operands_serve_many_calls(dev, cs):
    """One PREP_ONLY | NO_TIMELINE call, then three SKIP_PREP calls on other inputs, seeds and streams.  LRT (the
    PrepCache contract): each equals a fresh phase-0 call on its own seed and stream.  BBB: each reuses the one weight
    draw of the PREP_ONLY call's stream."""
    from pytorch_bayesiancnn_b200 import _lib as L
    s = _Layer(cs, dev)
    st = s.step(cs.B)
    ws = _fresh_ws(st, None, dev)
    with R.wide_tiles(cs.wide):
        R.fused_call(st, None, None, None, None, seed=SEED, stream=STREAM, phase=L.FUSED_PREP_ONLY | L.FUSED_NO_TIMELINE,
                     ws=ws)
        for i in range(3):
            xin = s.xin(s.x(cs.B))
            seed, stream = SEED + 1 + i, 1000 + 7 * i
            y1, _ = s.run(cs.B, xin, seed=seed, stream=stream, phase=L.FUSED_SKIP_PREP, ws=ws)
            ref_noise = dict(seed=seed, stream=stream) if s.lrt else dict(seed=SEED, stream=STREAM)
            y0, _ = s.run(cs.B, xin, **ref_noise)
            _same(s.bits(y1, cs.B), s.bits(y0, cs.B), f"SKIP_PREP call {i} on prepared operands")


def _fresh_ws(st, fold, dev):
    import ctypes as C
    from pytorch_bayesiancnn_b200 import _lib as L
    d = R.step_desc(st, 0, fold)
    return torch.zeros(int(L.lib().bbb_workspace_bytes(C.byref(d))), dtype=torch.uint8, device=dev)


# --------------------------------------------------------------------------------------------- MC-sample folds
@pytest.mark.parametrize("cs", FOLD_CASES, ids=[c.name for c in FOLD_CASES])
def test_fold_equals_one_call_per_sample(dev, cs):
    """Row block j of a folded call = the unfolded call on stream + j * stride, bit for bit (the stream crosses 2^32 and
    the stride has bits above it); the KL = the unfolded KL; block j within the float64 bar on philox_normal of sample
    j's stream."""
    s = _Layer(cs, dev)
    rows, S = s.fold_rows()
    xs, xin = s.fold_input(rows, S)
    with R.wide_tiles(cs.wide):
        yf, klf = s.run(rows * S, xin, seed=SEED, stream=STREAM, fold=(rows, STRIDE))
        bf = s.bits(yf, rows * S)
        for j in range(S):
            stream = (STREAM + j * STRIDE) & ((1 << 64) - 1)
            yj, klj = s.run(rows, s.xin(xs[j]), seed=SEED, stream=stream)
            _same(bf[j * rows:(j + 1) * rows], s.bits(yj, rows), f"fold block {j}")
            _eq_kl(klf, klj, "folded KL")
            ea, eb = s.philox_eps(rows, SEED, stream)
            s.check_ref("fold", yj, rows, xs[j], ea, eb)


@pytest.mark.parametrize("cs", CASES, ids=IDS)
def test_fold_refusals_launch_nothing(dev, cs):
    """Refused folds, each with 0 launches: the gather path; BBB rows % 128 != 0; external eps; a BBB fold given the
    unfolded workspace (BBB_E_WORKSPACE)."""
    from pytorch_bayesiancnn_b200 import _lib as L
    s = _Layer(cs, dev)
    refusals = []                                     # (what, batch, fold, eps, ws, expected code)
    ea = torch.zeros(1, device=dev)
    if not R.folds(cs):
        refusals.append(("gather fold", cs.B * 2, (cs.B, STRIDE), None, None, -2))
    else:
        rows, S = s.fold_rows()
        refusals.append(("external eps", rows * S, (rows, STRIDE), ea, None, -2))
        if not s.lrt:
            refusals.append(("rows % 128", 128, (64, STRIDE), None, None, -2))
            refusals.append(("unfolded workspace", rows * S, (rows, STRIDE), None, _fresh_ws(s.step(rows), None, dev), -3))
    for what, B, fold, eps, ws, code in refusals:
        st = s.step(B)
        xin = s.xin(s.x(B if cs.kind != "s4" else fold[0]))
        y, y_sq, _ = R._alloc_out(cs, st, dev, B)
        n0 = L.launch_count()
        rc, _ = R.fused_call_rc(st, xin[0], xin[1], y, y_sq, eps_a=eps, seed=SEED, stream=STREAM, fold=fold, ws=ws)
        assert rc == code, (what, rc, L.lib().bbb_last_error())
        assert L.launch_count() == n0, f"{what}: a refused call launched kernels"


# --------------------------------------------------------------------------------------------- first image
@pytest.mark.parametrize("cs", CASES, ids=IDS)
def test_first_image(dev, cs):
    """LRT: first image 3 = external eps taken from philox_normal at offset 3 * OH*OW*Cout, bit for bit.  BBB: the
    weight noise does not depend on rows, so it equals the first-image-0 call."""
    s = _Layer(cs, dev)
    xin = s.xin(s.x(cs.B))
    with R.wide_tiles(cs.wide):
        y1, kl1 = s.run(cs.B, xin, seed=SEED, stream=STREAM, first_image=3)
        if s.lrt:
            ea, _ = s.philox_eps(cs.B, SEED, STREAM, first_image=3)
            y2, kl2 = s.run(cs.B, xin, eps_a=ea)
        else:
            y2, kl2 = s.run(cs.B, xin, seed=SEED, stream=STREAM)
    _same(s.bits(y1, cs.B), s.bits(y2, cs.B), "first image 3")
    _eq_kl(kl1, kl2, "KL")


LAST_IMAGE_CASES = [c for c in CASES if c.name in ("s_c3_k11_32x32_b17_lrt", "t8x8_c64_k3p1_pool_lrt", "l_prev4_n100_lrt")]


@pytest.mark.parametrize("cs", LAST_IMAGE_CASES, ids=[c.name for c in LAST_IMAGE_CASES])
def test_largest_first_image(dev, cs):
    """The largest first image the engine accepts (int32 element counts, the 23-bit field) draws philox_normal at that
    offset, bit for bit."""
    s = _Layer(cs, dev)
    fi = R.first_image_max(cs, cs.B)
    xin = s.xin(s.x(cs.B))
    with R.wide_tiles(cs.wide):
        y1, _ = s.run(cs.B, xin, seed=SEED, stream=STREAM, first_image=fi)
        ea, _ = s.philox_eps(cs.B, SEED, STREAM, first_image=fi)
        y2, _ = s.run(cs.B, xin, eps_a=ea)
    _same(s.bits(y1, cs.B), s.bits(y2, cs.B), f"first image {fi}")


# --------------------------------------------------------------------------------------------- pruning masks
def _random_masks(s, frac, bias):
    m = s.m
    wm = torch.rand(m.W_mu.shape, generator=s.g) >= frac
    bm = (torch.rand(m.bias_mu.shape, generator=s.g) >= frac) if bias else None
    return wm.to(s.dev), None if bm is None else bm.to(s.dev)


def _set_params(m, p):
    with torch.no_grad():
        for t, v in zip((m.W_mu, m.W_rho, m.bias_mu, m.bias_rho), p):
            t.copy_(v)


@pytest.mark.parametrize("cs", CASES, ids=IDS)
def test_weight_mask(dev, cs):
    """All-ones masks = no mask, bit for bit.  50 % (with a bias mask, NaN planted in pruned mu / rho) and 95 % (weights
    only, inf planted): y within the bar of layer_ref on mask_ref.masked_params, the KL within 1e-5 of mask_ref.kl_ref
    (both conventions), and y = the unmasked call on zeroed parameters (mu = 0, rho = -inf), bit for bit -- folded BBB
    calls too.  A fully pruned layer (weights and biases) has KL exactly 0."""
    s = _Layer(cs, dev)
    m = s.m
    p0 = [t.detach().clone() for t in (m.W_mu, m.W_rho, m.bias_mu, m.bias_rho)]
    x = s.x(cs.B)
    xin = s.xin(x)
    calls = [(cs.B, None, xin)]
    if R.folds(cs) and not s.lrt:
        rows, S = s.fold_rows()
        calls.append((rows * S, (rows, STRIDE), s.fold_input(rows, S)[1]))
    noise = dict(seed=SEED, stream=STREAM)
    with R.wide_tiles(cs.wide):
        plain = [s.run(B, xi, fold=f, **noise) for B, f, xi in calls]
        m.set_weight_mask(torch.ones_like(m.W_mu, dtype=torch.bool), torch.ones_like(m.bias_mu, dtype=torch.bool))
        for (B, f, xi), (y0, kl0) in zip(calls, plain):
            y1, kl1 = s.run(B, xi, fold=f, **noise)
            _same(s.bits(y1, B), s.bits(y0, B), f"all-ones mask, fold {f}")
            _eq_kl(kl1, kl0, "all-ones mask KL")
        for frac, bias, plant, conv in ((0.5, True, float("nan"), "reference"), (0.95, False, float("inf"), "textbook")):
            wm, bm = _random_masks(s, frac, bias)
            m.kl_convention = conv
            m.set_weight_mask(wm, bm)
            with torch.no_grad():
                m.W_mu.masked_fill_(~wm, plant)
                m.W_rho.masked_fill_(~wm, plant)
                if bm is not None:
                    m.bias_mu.masked_fill_(~bm, plant)
                    m.bias_rho.masked_fill_(~bm, plant)
            mp = MR.masked_params(*[t.cpu() for t in p0], wm.cpu(), None if bm is None else bm.cpu())
            kl_ref = MR.kl_ref(*p0, wm, bm, m.prior_mu, m.prior_sigma, conv)
            # external eps: the float64 bar and the KL
            if s.lrt:
                ea, eb = torch.randn((cs.B, cs.cout) + ((s.oh, s.ow) if cs.kind != "linear" else ()), generator=s.g), None
            else:
                ea, eb = torch.randn(m.W_mu.shape, generator=s.g), torch.randn(cs.cout, generator=s.g)
            y, kl = s.run(cs.B, xin, eps_a=ea.to(dev), eps_b=None if eb is None else eb.to(dev))
            s.bits(y, cs.B)
            s.check_ref("mask", y, cs.B, x, ea, eb, params=mp)
            s.check_kl("mask", kl, kl_ref)
            # in-kernel noise: the masked calls, then the unmasked calls on zeroed parameters
            masked = [s.run(B, xi, fold=f, **noise) for B, f, xi in calls]
            for (B, f, xi), (y1, kl1) in zip(calls, masked):
                s.check_kl("mask", kl1, kl_ref)
            m.clear_weight_mask()
            _set_params(m, [t.float() for t in mp])
            for (B, f, xi), (y1, _) in zip(calls, masked):
                y2, _ = s.run(B, xi, fold=f, **noise)
                _same(s.bits(y1, B), s.bits(y2, B), f"{frac:.0%} mask vs zeroed parameters, fold {f}")
            _set_params(m, p0)
        m.kl_convention = "reference"
        m.set_weight_mask(torch.zeros_like(m.W_mu, dtype=torch.bool), torch.zeros_like(m.bias_mu, dtype=torch.bool))
        for B, f, xi in calls:
            y, kl = s.run(B, xi, fold=f, **noise)
            s.bits(y, B)
            assert float(kl) == 0.0, float(kl)


# --------------------------------------------------------------------------------------------- tensor priors
@pytest.mark.parametrize("cs", CASES, ids=IDS)
def test_tensor_prior(dev, cs):
    """A tensor prior filled with the scalar prior = the scalar call (y and KL), bit for bit.  A random prior
    (mu_p = W_mu + N(0, 0.05), sigma_p = softplus(W_rho + N(0, 0.5))) in both KL conventions, and with a 50 % mask:
    KL within 1e-5 of mask_ref.kl_ref(prior=...), y bit for bit the scalar-prior call -- folded BBB calls too."""
    s = _Layer(cs, dev)
    m = s.m
    xin = s.xin(s.x(cs.B))
    calls = [(cs.B, None, xin)]
    if R.folds(cs) and not s.lrt:
        rows, S = s.fold_rows()
        calls.append((rows * S, (rows, STRIDE), s.fold_input(rows, S)[1]))
    noise = dict(seed=SEED, stream=STREAM)
    p = s.params()
    sp = lambda t: torch.nn.functional.softplus(t)
    pri = (p[0] + 0.05 * torch.randn(p[0].shape, generator=s.g), sp(p[1] + 0.5 * torch.randn(p[1].shape, generator=s.g)),
           p[2] + 0.05 * torch.randn(p[2].shape, generator=s.g), sp(p[3] + 0.5 * torch.randn(p[3].shape, generator=s.g)))
    wm, _ = _random_masks(s, 0.5, False)
    ones = torch.ones_like(m.W_mu, dtype=torch.bool)
    with R.wide_tiles(cs.wide):
        scalar = {}
        for conv in ("reference", "textbook"):
            m.kl_convention = conv
            scalar[conv] = [s.run(B, xi, fold=f, **noise) for B, f, xi in calls]
        m.set_weight_mask(wm)
        scalar_mk = [s.run(B, xi, fold=f, **noise) for B, f, xi in calls]
        m.clear_weight_mask()
        m.kl_convention = "reference"
        m.set_prior(torch.full_like(m.W_mu, m.prior_mu), torch.full_like(m.W_mu, m.prior_sigma),
                    torch.full_like(m.bias_mu, m.prior_mu), torch.full_like(m.bias_mu, m.prior_sigma))
        for (B, f, xi), (y0, kl0) in zip(calls, scalar["reference"]):
            y1, kl1 = s.run(B, xi, fold=f, **noise)
            _same(s.bits(y1, B), s.bits(y0, B), f"constant tensor prior, fold {f}")
            _eq_kl(kl1, kl0, "constant tensor prior KL")
        m.set_prior(*[t.to(dev) for t in pri])
        for conv, mask in (("reference", None), ("textbook", None), ("textbook", wm)):
            m.kl_convention = conv
            if mask is not None:
                m.set_weight_mask(mask)
            kl_ref = MR.kl_ref(*p, (ones if mask is None else mask).cpu(), None, m.prior_mu, m.prior_sigma, conv,
                               prior=pri)
            base = scalar[conv] if mask is None else scalar_mk
            for (B, f, xi), (y0, _) in zip(calls, base):
                y1, kl1 = s.run(B, xi, fold=f, **noise)
                _same(s.bits(y1, B), s.bits(y0, B), f"random tensor prior ({conv}, mask {mask is not None}), fold {f}")
                s.check_kl("prior" + ("+mask" if mask is not None else ""), kl1, kl_ref)

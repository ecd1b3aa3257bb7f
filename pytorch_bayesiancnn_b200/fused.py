"""Fused execution of a ModuleWrapper's children (SURVEY.md 8f row f2).

The reference's model files interleave the Bayesian layers with ``nn.Softplus`` /
``nn.ReLU``, ``nn.MaxPool2d(2, 2)`` and ``FlattenLayer`` children
(BayesianAlexNet.py:34-53).  ``ModuleWrapper.forward`` (layers/misc.py:16-18) just
calls them in order; here the same child list is pattern-matched into runs of
``[Bayesian layer, activation?, 2x2 max-pool?, flatten*]`` and each run becomes ONE
``bbb_layer_forward_fused`` call (weight-prep kernel + tensor-core GEMM kernel whose
epilogue applies the activation and the pool and writes the packed bf16 format the
next layer's TMA loads).  The model files stay unmodified; anything that does not
match (other pools, other modules, autograd needed) falls back to the plain
child-by-child path.
"""
from __future__ import annotations

import ctypes as C
import os

import torch
from torch import nn

from . import _lib as L
from . import functional as Fn


class _Step:
    __slots__ = ("layer", "act", "pool", "conv", "in_shape", "in_layout", "prev_hw", "out_layout", "out_chw",
                 "eps_shape", "linear", "batch")


def _act_code(m):
    if isinstance(m, nn.Softplus) and m.beta == 1 and m.threshold == 20:
        return L.ACT_SOFTPLUS
    if isinstance(m, nn.ReLU):
        return L.ACT_RELU
    return None


def _is_pool22(m):
    def two(v):
        return v == 2 or v == (2, 2)
    return (isinstance(m, nn.MaxPool2d) and two(m.kernel_size) and two(m.stride) and m.padding in (0, (0, 0))
            and m.dilation in (1, (1, 1)) and not m.ceil_mode and not m.return_indices)


def plan(children, x_shape, fold=None):
    """Return the list of fused steps for this child list and input shape, or None.
    ``fold`` = (rows per MC sample, Philox stream stride): x_shape[0] is then the FOLDED batch (samples x rows)."""
    from .modules import _BayesLayer, FlattenLayer
    if len(x_shape) != 4:
        return None
    batch, c, h, w = x_shape
    state = ("nchw", c, h, w)
    steps = []
    i, n = 0, len(children)
    while i < n:
        m = children[i]
        if not isinstance(m, _BayesLayer) or m.math not in ("bf16", "auto"):
            return None
        st = _Step()
        st.layer = m
        st.batch = batch
        st.conv = m._conv_geometry()
        st.linear = st.conv is None
        lay, c, h, w = state
        if st.linear:
            if lay != "packed" or m.in_features != c * h * w:
                return None
            st.prev_hw = h * w
            st.in_shape = (c * h * w, 1, 1)
            cout, oh, ow = m.out_features, 1, 1
        else:
            if m.in_channels != c:
                return None
            (sh, sw), (ph, pw), (dh, dw) = st.conv
            if (dh, dw) != (1, 1):
                return None
            kh, kw = m.kernel_size
            oh, ow = (h + 2 * ph - kh) // sh + 1, (w + 2 * pw - kw) // sw + 1
            if oh < 1 or ow < 1:
                return None
            if lay == "packed" and (h * w > 64 or c % 64):
                return None
            st.prev_hw = 1
            st.in_shape = (c, h, w)
            cout = m.out_channels
        st.in_layout = L.LAYOUT_NCHW_F32 if lay == "nchw" else L.LAYOUT_PACKED_BF16
        st.eps_shape = (cout, oh, ow)
        i += 1
        st.act = L.ACT_NONE
        if i < n and _act_code(children[i]) is not None:
            st.act = _act_code(children[i])
            i += 1
        st.pool = False
        if i < n and isinstance(children[i], nn.MaxPool2d):
            if not _is_pool22(children[i]) or st.linear or oh % 2 or ow % 2:
                return None
            st.pool = True
            oh, ow = oh // 2, ow // 2
            i += 1
        while i < n and isinstance(children[i], FlattenLayer):
            if children[i].num_features != cout * oh * ow:
                return None            # the reference's view(-1, F) would fold the batch (SURVEY D2): not fused
            i += 1
        st.out_chw = (cout, oh, ow)
        state = ("packed", cout, oh, ow)
        steps.append(st)
    if not steps:
        return None
    last = steps[-1]
    last.out_layout = L.LAYOUT_ROWMAJOR_F32 if last.out_chw[1] * last.out_chw[2] == 1 else L.LAYOUT_NCHW_F32
    for st in steps[:-1]:
        st.out_layout = L.LAYOUT_PACKED_BF16
        if st.out_chw[0] % 64:                  # tiled packed format: whole 64-channel blocks per pixel
            return None
    # the engine has the last word (same checks bbb_layer_forward_fused makes, host-only): run() must not
    # discover an unsupported shape after noise was drawn and prep kernels were enqueued on side streams
    lib = L.lib()
    for st in steps:
        d = _step_desc(st, 0, fold)
        rc = lib.bbb_fused_supported(C.byref(d), st.in_layout, _in_pitch(st), st.prev_hw, st.out_layout, _out_pitch(st))
        if rc == -2:                            # BBB_E_UNSUPPORTED: not fusable, the caller runs child by child
            return None
        L.check(rc, "bbb_fused_supported")
    return steps


def _in_pitch(st):
    cin, h, w = st.in_shape
    return 0 if st.in_layout == L.LAYOUT_NCHW_F32 else cin * h * w


def _out_pitch(st):
    cout, oh, ow = st.out_chw
    return cout * oh * ow if st.out_layout == L.LAYOUT_PACKED_BF16 else 0


def _step_desc(st, phase, fold=None):
    m = st.layer
    cin, h, w = st.in_shape
    x_shape = (st.batch, cin) if st.linear else (st.batch, cin, h, w)
    # ModuleWrapper calls children with sample=True (SURVEY D6)
    d = Fn.make_desc(x_shape, tuple(m.W_mu.shape), st.conv, m._variant, True, m.use_bias, m.prior_mu, m.prior_sigma,
                     L.MATH_BF16_TC, L.KL_BY_NAME[m.kl_convention], st.act, fold=fold,
                     first_image=Fn.current_first_image())
    d.pool_k = d.pool_s = 2 if st.pool else 0
    d.reserved[0] |= phase
    return d


_side_streams: dict = {}
_direct = {"out": None, "terms": False}
_cached = {"prep": None}


class PrepCache:
    """The parameter-only half of a planned chain -- bf16 operand tiles, bias rows and the Gaussian KL of every layer --
    in workspaces of its own, prepared ahead of the steps that read them (mc.MCForward: once per parameter version).

    Only a chain of LRT layers is cached: an LRT prep is a pure function of the parameters and the prior (the LRT noise is
    drawn on the activations, in the GEMM epilogue), so the tiles and KL of every step are the bits the step's own prep
    would write.  A BBB prep draws the weights of its step and stays in the step.  A mixture-prior layer's tiles are
    cached; its KL, a Monte-Carlo draw per sample, stays in the step.

    ``fill()`` enqueues the preps on the current stream.  A chain entered under ``use_prep(cache)`` launches only its GEMM
    kernels (and the mixture draws), reading the cache; ordering the fill against the steps is the caller's job."""

    def __init__(self, steps, fold, dev):
        self.steps, self.fold = steps, fold
        self.layers = [st.layer for st in steps]
        self.kl = torch.zeros(len(steps), dtype=torch.float32, device=dev)    # per-layer KL scalars (stable address)
        self.ws = [None] * len(steps)

    @staticmethod
    def eligible(steps) -> bool:
        return bool(steps) and all(st.layer._variant == L.VARIANT_LRT for st in steps)

    def covers(self, steps) -> bool:
        return len(steps) == len(self.layers) and all(st.layer is m for st, m in zip(steps, self.layers))

    def fill(self):
        """The preps of every layer, in layer order, on the current stream; they take no debug-timeline slot."""
        lib = L.lib()
        for i, st in enumerate(self.steps):
            if self.ws[i] is None:
                d = _step_desc(st, L.FUSED_PREP_ONLY, self.fold)
                self.ws[i] = torch.zeros(int(lib.bbb_workspace_bytes(C.byref(d))), dtype=torch.uint8,
                                         device=self.kl.device)
            run_step(st, None, None, None, 0, kl=self.kl[i], noise=(None, None, 0, 0, None, None),
                     phase=L.FUSED_PREP_ONLY, fold=self.fold, ws=self.ws[i], fill=True)


class use_prep:
    """``with fused.use_prep(cache): ...`` -- a chain run inside whose layers are those of ``cache`` (a PrepCache) reads
    their operand tiles and KL from it instead of preparing them."""

    def __init__(self, cache):
        self.cache = cache

    def __enter__(self):
        self.prev, _cached["prep"] = _cached["prep"], self.cache
        return self

    def __exit__(self, *exc):
        _cached["prep"] = self.prev
        return False


class direct_output:
    """``with fused.direct_output(buf): logits, kls = net(x)`` -- a fused chain entered inside writes its final fp32
    logits straight into ``buf`` ([B, C], contiguous) and returns the per-layer KL scalars UN-summed (the caller's
    kernel sums them: bbb_mc_exchange), so the Monte-Carlo step has no copy and no aten reduction behind the chain.
    ``.used`` tells whether a fused chain really took the buffer (non-fusable nets ignore the hook)."""

    def __init__(self, out, kl_buf=None):
        """``kl_buf``: optional fp32 device vector the per-layer KL scalars are written to (its first n entries are
        returned) instead of a tensor allocated by the chain -- a stable address for a kernel captured separately."""
        self.out, self.used, self.kl_buf = out, False, kl_buf

    def __enter__(self):
        self.prev = dict(_direct)
        _direct.update(out=self.out, terms=True, owner=self, kl_buf=self.kl_buf)
        return self

    def __exit__(self, *exc):
        _direct.clear()
        _direct.update(self.prev)
        return False


def _side_stream(dev, i=0):
    st = _side_streams.get((dev.index, i))
    if st is None:
        st = _side_streams[(dev.index, i)] = torch.cuda.Stream(device=dev)
    return st


def _prep_chains():
    return max(1, int(os.environ.get("BBB_B200_PREP_CHAINS", "3")))


def run(steps, x: torch.Tensor, overlap_prep: bool = True):
    return _run(steps, x, overlap_prep, _direct.get("out"), _direct.get("terms", False), _direct.get("owner"),
                kls_out=_direct.get("kl_buf"))


def _run(steps, x, overlap_prep, out, terms, owner, fold=None, kls_out=None):
    """Execute a planned chain.  Returns (network output fp32, summed KL 0-dim tensor).

    The parameter-only half of every layer (softplus / eps / bf16 operand tiles / KL) runs on side
    streams (parallel branches of a captured graph), joined to the GEMM chain by events, so only the
    first layer's prep is on the activation critical path.  The preps are issued in layer order over
    a few serial chains (default 3: layers 1,4 / 2,5 / 3) rather than all at once: six concurrent prep
    grids fill the machine and the first layer's prep -- the one the GEMM chain is waiting for -- was
    scheduled last (tools/timeline.py shows the start of each GEMM).  The KL sum
    depends on the preps only and runs on the side as well.

    A layer with a mixture prior (set_mixture_prior) computes no KL in its prep: its term is a Monte-Carlo draw per MC
    sample (one, or the fold's samples), launched behind its prep on the prep's stream.  The chain then returns the
    per-sample KL -- the layers' terms added in layer order, 0-dim or [samples] under a fold -- with ``terms`` as well.

    Under ``use_prep(cache)`` with a cache of this chain (same layers, fold and batch) the preps are not launched: every
    layer's operand tiles, bias rows and Gaussian KL are read from the cache, the GEMM kernels run back to back on the
    current stream -- the first one launched programmatically behind whatever heads the step -- and a mixture-prior
    layer's Monte-Carlo KL draw runs on a side stream beside them.  Noise is drawn per layer either way, so every
    output is the same."""
    cache = _cached["prep"]
    if not (cache is not None and cache.covers(steps) and cache.fold == fold and steps[0].batch == cache.steps[0].batch):
        cache = None
    dev = x.device
    n = len(steps)
    if cache is not None:
        kls = cache.kl[:n]
    else:
        kls = kls_out[:n] if kls_out is not None else torch.empty(n, dtype=torch.float32, device=dev)
    mixed = [i for i, st in enumerate(steps) if st.layer.mixture_values() is not None]
    if mixed:
        n_draws = 1 if fold is None else steps[0].batch // fold[0]
        mix = torch.empty(len(mixed), n_draws, dtype=torch.float32, device=dev)
        kl_of = [mix[mixed.index(i)] if i in mixed else kls[i] for i in range(n)]
    else:
        kl_of = [kls[i] for i in range(n)]
    snap = Fn.noise_snapshot()
    main = torch.cuda.current_stream(dev)
    # Where each layer's prep comes from: the cache; inline, in the launch of its GEMM kernel (phase 0); or a launch of
    # its own on prep_on[i] (overlap).  The FIRST layer's prep then stays on the main stream, right in front of its GEMM
    # kernel: launched with programmatic serialization the GEMM kernel's CTAs start while the prep runs and stage their
    # input images meanwhile (conv_s4_tc.cuh); only its weight producer waits for the prep.  The other preps go to the
    # side chains.
    overlap = overlap_prep and cache is None
    inline = not overlap_prep and cache is None
    chains, prep_on = [], [None] * n
    if overlap:
        chains = [_side_stream(dev, c) for c in range(min(_prep_chains(), n))]
        if os.environ.get("BBB_B200_PREP0_MAIN", "1") == "1":
            prep_on = [main] + [chains[(i - 1) % len(chains)] for i in range(1, n)]
        else:
            prep_on = [chains[i % len(chains)] for i in range(n)]
    elif cache is not None and mixed:
        chains = [_side_stream(dev)]           # the mixture draws
    forked = False
    try:
        if fold is not None and Fn.external_eps_active():
            raise L.EngineError("MC-sample folding draws its noise in-kernel (no external eps)")
        noise = [_draw_noise(st, x.shape[0], dev) for st in steps]
        for side in chains:
            side.wait_stream(main)
        forked = bool(chains)
        events, ev0 = [None] * n, None         # the GEMM kernel of layer i waits for events[i]
        for i, st in enumerate(steps):
            if cache is not None and i in mixed:
                with torch.cuda.stream(chains[0]):
                    kl_of[i] = _kl_mc(st.layer, kl_of[i], noise[i], fold)
            elif cache is not None:
                st.layer._kl_cache = (kls[i], st.layer._versions(), torch.is_grad_enabled())
            elif prep_on[i] is not None:
                with torch.cuda.stream(prep_on[i]):
                    run_step(st, None, None, None, 0, kl=kl_of[i], noise=noise[i], phase=L.FUSED_PREP_ONLY, fold=fold)
                    ev = torch.cuda.Event()
                    ev.record(prep_on[i])
                if prep_on[i] is main:
                    ev0 = ev
                else:
                    events[i] = ev
        for side in chains[1:]:
            chains[0].wait_stream(side)
        if overlap and not terms and not mixed:
            with torch.cuda.stream(chains[0]):
                if ev0 is not None:
                    chains[0].wait_event(ev0)
                kl_total = kls.sum()
        cur, cur_sq, cur_pitch = x.contiguous().float(), None, 0
        last = steps[-1]
        take = (out is not None and last.out_layout == L.LAYOUT_ROWMAJOR_F32 and out.is_contiguous()
                and out.dtype == torch.float32 and tuple(out.shape) == (last.batch, last.out_chw[0]))
        for i, st in enumerate(steps):
            nxt = steps[i + 1].layer if i + 1 < n else None
            y_into = out if (take and i == n - 1) else None
            if events[i] is not None:
                main.wait_event(events[i])
            cur, cur_sq, cur_pitch = run_step(st, nxt, cur, cur_sq, cur_pitch, kl=kl_of[i], noise=noise[i],
                                              phase=0 if inline else L.FUSED_SKIP_PREP, y_into=y_into,
                                              fold=fold, ws=cache.ws[i] if cache is not None else None)
        if cache is not None and forked:       # the cached chain's mixture draws: no event of theirs was waited for
            main.wait_stream(chains[0])
            forked = False
        if mixed:
            # element-wise adds in layer order (the main stream has waited for every prep and draw): sample j's sum is the
            # same whether the samples are folded or run one by one
            kl_total = kl_of[0]
            for t in kl_of[1:]:
                kl_total = kl_total + t
            if fold is None:
                kl_total = kl_total.reshape(())
        elif terms:
            kl_total = kls
        elif not overlap:
            kl_total = kls.sum()
        if terms and owner is not None:
            owner.used = True
    except BaseException:
        Fn.noise_restore(snap)                 # a retry / fallback sees the stream ids and eps queue it would have seen
        raise
    finally:
        if forked:                             # ALWAYS re-join the forked side streams: `kls` and the layer workspaces are
            for side in chains[1:]:            # written there, and an active graph capture must not be left with dangling forks
                chains[0].wait_stream(side)
            main.wait_stream(chains[0])
    return cur, kl_total


def _kl_mc(m, kl, noise, fold):
    """A mixture-prior layer's Monte-Carlo KL of one layer call into ``kl`` (one entry per folded MC sample, each from
    its own stream); returns it as the call returns it (0-dim unfolded) and keeps it as the layer's KL."""
    kl_stream = noise[5]
    Fn.kl_mc_forward(kl, m.W_mu, m.W_rho, m.bias_mu, m.bias_rho, m.mixture_values(), kl_stream[0], kl_stream[1],
                     Fn._noise.base, fold[1] if fold is not None else 0, m)
    if fold is None:
        kl = kl.reshape(())
    m._kl_cache = (kl, m._versions(), torch.is_grad_enabled())
    return kl


def _draw_noise(st, B, dev):
    """(eps_a, eps_b, seed, stream_id, base, kl_stream) for one layer call, consuming the external-eps
    queue / the Philox stream counter exactly like the unfused layer would.  kl_stream: (seed, stream id) of the
    Monte-Carlo KL draw of a layer with a mixture prior -- the next id behind the layer's own -- else None."""
    m = st.layer
    eps_a = eps_b = None
    seed = stream_id = 0
    base = None
    if Fn.external_eps_active():
        if m._variant == L.VARIANT_LRT:
            eps_a = Fn._pop_eps((B,) + st.eps_shape if not st.linear else (B, st.eps_shape[0]), dev)
        else:
            eps_a = Fn._pop_eps(m.W_mu.shape, dev)
            if m.use_bias:
                eps_b = Fn._pop_eps(m.bias_mu.shape, dev)
    else:
        seed, stream_id = Fn.next_stream()
        base = Fn._noise.base
    kl_stream = Fn.next_stream() if m.mixture_values() is not None else None
    return eps_a, eps_b, seed, stream_id, base, kl_stream


def run_step(st, nxt, cur, cur_sq, cur_pitch, kl=None, noise=None, phase=0, y_into=None, fold=None, ws=None,
             fill=False):
    """One fused layer call: (y, y_sq, pitch) = step(cur, cur_sq).  phase: 0 = prep + GEMM,
    FUSED_PREP_ONLY / FUSED_SKIP_PREP = one half (see include/bbb_b200.h).  ``ws``: the workspace of the operand tiles
    (default: the layer's own, Fn.workspace).  ``fill``: a PREP_ONLY call filling a PrepCache -- off the debug timeline,
    and a mixture prior's Monte-Carlo KL is left to the steps."""
    lib = L.lib()
    m = st.layer
    dev = m.W_mu.device
    B = st.batch                                    # (packed inputs carry rows padded to the 128-row tile)
    cin, h, w = st.in_shape
    d = _step_desc(st, phase | (L.FUSED_NO_TIMELINE if fill else 0), fold)
    in_pitch = cur_pitch if st.in_layout == L.LAYOUT_NCHW_F32 else cin * h * w
    cout, oh, ow = st.out_chw
    if phase == L.FUSED_PREP_ONLY:
        pitch, y, y_sq = cout * oh * ow if st.out_layout == L.LAYOUT_PACKED_BF16 else 0, None, None
    elif st.out_layout == L.LAYOUT_PACKED_BF16:
        pitch = cout * oh * ow                   # tiled packed: [ceil(B/128)][F/64][planes][128 x 64] bf16
        planes = 2 if (nxt is not None and nxt._variant == L.VARIANT_LRT) else 1
        y = torch.empty((B + 127) // 128 * 128, pitch * planes, dtype=torch.bfloat16, device=dev)
        y_sq = y.view(-1)[128 * 64:] if planes == 2 else None      # x^2 blocks interleaved behind the x blocks
    elif st.out_layout == L.LAYOUT_ROWMAJOR_F32:
        pitch, y, y_sq = 0, (y_into if y_into is not None else torch.empty(B, cout, dtype=torch.float32, device=dev)), None
    else:
        pitch, y, y_sq = 0, torch.empty(B, cout, oh, ow, dtype=torch.float32, device=dev), None
    if kl is None:
        kl = torch.empty(st.batch // fold[0] if (fold is not None and m.mixture_values() is not None) else (),
                         dtype=torch.float32, device=dev)
    if noise is None:
        noise = _draw_noise(st, B, dev)
    eps_a, eps_b, seed, stream_id, base, kl_stream = noise
    mixture = m.mixture_values()
    if ws is None:
        ws = Fn.workspace(dev, d, m)
    parg, flag = Fn.masked_prior_arg(m.prior_tensors(), m.mask_tensors())
    rc = lib.bbb_layer_forward_fused_prior(
        C.byref(Fn.desc_with(d, flag)), Fn._ptr(cur), Fn._ptr(cur_sq), st.in_layout, in_pitch, st.prev_hw,
        Fn._ptr(m.W_mu), Fn._ptr(m.W_rho), Fn._ptr(m.bias_mu), Fn._ptr(m.bias_rho),
        Fn._ptr(y), Fn._ptr(y_sq), st.out_layout, pitch, None if mixture is not None else Fn._ptr(kl),
        Fn._ptr(eps_a), Fn._ptr(eps_b),
        C.c_uint64(seed), C.c_uint64(stream_id), Fn._ptr(base), Fn._ptr(ws), C.c_size_t(ws.numel()),
        Fn._stream(dev), parg)
    L.check(rc, "bbb_layer_forward_fused_prior")
    if phase != L.FUSED_SKIP_PREP and not fill:
        if mixture is not None:             # kl: one entry per folded MC sample, each from its own stream
            _kl_mc(m, kl, noise, fold)
        else:
            m._kl_cache = (kl, m._versions(), torch.is_grad_enabled())
    return y, y_sq, pitch

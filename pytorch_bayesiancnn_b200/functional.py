"""Host side of the boundary: torch.autograd.Functions that call the C ABI.

PyTorch supplies device memory, the current stream and autograd; every number on
the Bayesian layer path is produced by libbbb_b200.so.  Nothing here computes a
layer with aten ops.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import itertools
import os
import threading
import weakref
from typing import Iterable, Optional

import torch

from . import _lib as L


# --------------------------------------------------------------------------- #
# noise bookkeeping (Python owns (seed, stream_id); kernels own the draws)
# --------------------------------------------------------------------------- #
_MASK64 = 0xFFFFFFFFFFFFFFFF
_MC_NAMESPACE = 1 << 63            # stream ids of Monte-Carlo evaluation samples (mc_sample): disjoint from training's
_instances = itertools.count()     # one _Noise per thread; the index keeps DataParallel replica threads apart


def _rank() -> int:
    try:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized():
            return dist.get_rank()
    except Exception:
        pass
    return int(os.environ.get("RANK", "0"))


class _Noise(threading.local):
    """(seed, stream counter) of the calling thread.

    Default seed: derived from ``torch.initial_seed()``, the process rank and the thread's index, so that
    ``torch.manual_seed(s)`` reseeds the engine like it reseeds the reference's CPU generator, and so that ranks /
    DataParallel replica threads do not draw identical noise.  ``manual_seed`` pins an explicit seed instead
    (same value on every rank = same noise on every rank, which is what MC sharding wants: see mc.py)."""

    def __init__(self):
        self.index = next(_instances)
        self.explicit = False
        self.seed = None
        self.torch_seed = None
        self.counter = 0
        self.queue = None          # external-eps queue (parity mode)
        self.base = None           # device int64[1] stream base (CUDA-graph capture mode)
        self.fold = None           # (rows per MC sample, Philox stream stride) of layer_fold
        self.fold_grad = False     # layer_fold(grad=True): folded LRT calls record autograd
        self.first_image = 0       # global index of image 0 of the layer calls (first_image)

    def current_seed(self) -> int:
        if not self.explicit:
            ts = torch.initial_seed()
            if self.seed is None or ts != self.torch_seed:      # first use, or torch.manual_seed() was called since
                self.torch_seed = ts
                mix = (ts * 0x9E3779B97F4A7C15 + _rank() * 0xD1B54A32D192ED03 + self.index * 0x94D049BB133111EB
                       + 0x5EEDB200) & _MASK64
                self.seed, self.counter = mix, 0
        return self.seed


_noise = _Noise()


def manual_seed(seed: int, counter: int = 0):
    """Seed the engine's Philox streams.  Every stochastic layer call consumes one
    stream id (counter += 1), so a fixed seed replays the same noise."""
    _noise.explicit = True
    _noise.seed = int(seed) & _MASK64
    _noise.counter = int(counter)


def current_seed() -> int:
    return _noise.current_seed()


def begin_sample(sample_id: int):
    """Position the stream counter for Monte-Carlo sample `sample_id` (global id):
    layer calls of that sample use stream ids (sample_id << 32) + 0, 1, 2, ...  so
    results do not depend on how samples are sharded over ranks (SURVEY.md 8e).
    Moves the calling thread's counter for good: prefer the ``mc_sample`` context manager,
    which restores the training counter afterwards."""
    _noise.counter = int(sample_id) << 32


@contextlib.contextmanager
def mc_sample(sample_id: int, seed: Optional[int] = None, offset: int = 0):
    """Layer calls inside draw Monte-Carlo evaluation sample `sample_id` (global id): stream ids
    2^63 + (sample_id << 40) + 0, 1, 2, ... (2^40 ids per sample: room for 2^20 CUDA-graph replays of 2^20 layer calls)
    -- a namespace training never reaches, independent of how the samples are sharded over ranks.  The thread's training counter (and seed) are restored on exit, so an evaluation pass
    between epochs does not make training replay its noise."""
    _noise.current_seed()
    saved = (_noise.seed, _noise.counter, _noise.explicit)
    if seed is not None:
        _noise.seed, _noise.explicit = int(seed) & _MASK64, True
    _noise.counter = (_MC_NAMESPACE | (int(sample_id) << 40)) + int(offset)     # offset: e.g. training step * 2^20
    try:
        yield
    finally:
        _noise.seed, _noise.counter, _noise.explicit = saved


@contextlib.contextmanager
def stream_base(base: Optional[torch.Tensor]):
    """Graph-capture mode: layer calls inside take stream ids 0, 1, 2, ... RELATIVE to
    the device scalar `base` (int64[1]), which kernels read at run time; advancing it
    (bbb_noise_advance, captured in the graph) gives every replay fresh noise."""
    prev, prev_ctr = _noise.base, _noise.counter
    _noise.base = base
    _noise.counter = 0
    try:
        yield
    finally:
        _noise.base, _noise.counter = prev, prev_ctr


@contextlib.contextmanager
def layer_fold(rows: int, stride: int, grad: bool = False):
    """Layer calls inside fold Monte-Carlo samples into the batch (include/bbb_b200.h, bbb_conv2d_forward): image b of
    the batch is image b % rows of sample b // rows, which draws from Philox stream stream_id + (b // rows) * stride --
    the same numbers as one call per sample.  What uncertainty_estimation.py:38-41 does by repeating the input, with
    each repeat its own sample.  In-kernel noise only: a layer call with external eps raises EngineError.

    ``grad=False`` (default): forward only -- a layer call under autograd raises EngineError.
    ``grad=True``: an LRT layer call on a tensor-core math mode (bf16, tf32, or auto resolving to one) records autograd.
    Its backward runs the tensor-core contractions over all rows (a weight gradient sums the rows of every sample, an
    input-gradient row depends on its own row only) and draws the noise term's gradient row by row from the same
    streams (bbb_lrt_noise_grad); the KL backward runs once.  Refused with EngineError: a BBB layer, math='fp32', external
    eps, and any geometry whose backward would fall back to the CUDA-core kernels (tc_backward_refusal), which do not
    know the fold."""
    prev = _noise.fold, _noise.fold_grad
    _noise.fold, _noise.fold_grad = (int(rows), int(stride)), bool(grad)
    try:
        yield
    finally:
        _noise.fold, _noise.fold_grad = prev


@contextlib.contextmanager
def first_image(b0: int):
    """Layer calls inside hold images [b0, b0 + batch) of a larger batch (a row block of a sharded Monte-Carlo step,
    mc.MCForward(batch_shards=...)): the LRT activation noise of image b is drawn at image b0 + b, so a block's outputs
    equal the whole batch's outputs at its rows bit for bit -- on every forward path and the backward.  BBB weight noise
    does not depend on rows.  Only the Philox element index moves (include/bbb_b200.h, desc->reserved[0])."""
    b0 = int(b0)
    if not 0 <= b0 <= FIRST_IMAGE_MAX:
        raise L.EngineError(f"first_image: {b0} is outside [0, {FIRST_IMAGE_MAX}]")
    prev = _noise.first_image
    _noise.first_image = b0
    try:
        yield
    finally:
        _noise.first_image = prev


def current_first_image() -> int:
    return _noise.first_image


FIRST_IMAGE_MAX = (1 << 23) - 1       # bits 8..30 of desc->reserved[0]


def first_image_word(b0: int) -> int:
    """desc->reserved[0] bits of first image b0 (an int32; a value the engine refuses when b0 is out of range)."""
    return C.c_int32((int(b0) << 8) & 0xFFFFFFFF).value if 0 <= int(b0) <= FIRST_IMAGE_MAX else -1


def layer_fold_active() -> bool:
    return _noise.fold is not None


def noise_advance(base: torch.Tensor, inc: int):
    rc = L.lib().bbb_noise_advance(_ptr(base), C.c_uint64(inc), _stream(base.device))
    L.check(rc, "bbb_noise_advance")


def next_stream() -> tuple[int, int]:
    seed = _noise.current_seed()
    s = _noise.counter
    _noise.counter += 1
    return seed, s


def noise_snapshot():
    """(counter, eps queue) -- lets a multi-layer caller roll the noise state back if it fails half-way."""
    return _noise.counter, (list(_noise.queue) if _noise.queue is not None else None)


def noise_restore(snap):
    _noise.counter = snap[0]
    if snap[1] is not None and _noise.queue is not None:
        _noise.queue[:] = snap[1]


@contextlib.contextmanager
def external_eps(tensors: Iterable[torch.Tensor]):
    """Parity mode: feed the layers the eps tensors the reference drew, in the
    reference's draw order (BBB: W_eps then bias_eps per layer -- BBB/BBBConv.py:63,68;
    LRT: one activation-shaped eps per layer -- BBB_LRT/BBBConv.py:78)."""
    prev = _noise.queue
    _noise.queue = list(tensors)
    try:
        yield
        if _noise.queue:
            raise RuntimeError(f"external_eps: {len(_noise.queue)} eps tensors were not consumed")
    finally:
        _noise.queue = prev


def _pop_eps(shape, device):
    q = _noise.queue
    if q is None:
        return None
    if not q:
        raise RuntimeError("external_eps: queue exhausted")
    e = q.pop(0)
    if tuple(e.shape) != tuple(shape):
        raise RuntimeError(f"external_eps: expected shape {tuple(shape)}, got {tuple(e.shape)}")
    return e.to(device=device, dtype=torch.float32).contiguous()


def external_eps_active() -> bool:
    return _noise.queue is not None


# --------------------------------------------------------------------------- #
# helpers
# --------------------------------------------------------------------------- #
def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def prior_arg(prior, bias: bool = False):
    """The ``const bbb_prior*`` argument of a *_prior entry point: None (NULL, the scalar prior of the desc / call) when
    ``prior`` is None, else a reference to the bbb_prior of ``prior`` = (w_mu, w_sigma, b_mu, b_sigma) -- contiguous fp32
    CUDA tensors, b_* None without a bias.  ``bias=True``: the bias part in the w_ fields, as bbb_kl_backward_prior reads
    the prior of the n elements it is called on."""
    if prior is None:
        return None
    w_mu, w_sigma, b_mu, b_sigma = prior
    if bias:
        w_mu, w_sigma, b_mu, b_sigma = b_mu, b_sigma, None, None
    for t in (w_mu, w_sigma, b_mu, b_sigma):
        if t is not None:
            _require_cuda(t, "tensor prior")
    p = lambda t: None if t is None else t.data_ptr()
    return C.byref(L.Prior(p(w_mu), p(w_sigma), p(b_mu), p(b_sigma)))


def masked_prior_arg(prior, mask, bias: bool = False):
    """(the ``prior`` argument, the flag for kl_convention) of a *_prior entry point for a layer with the tensor prior
    ``prior`` (or None) and the pruning mask ``mask`` = (w_mask, b_mask) (or None): without a mask, (prior_arg, 0);
    with one, a reference to a bbb_masked_prior and PRIOR_MASKED.  ``bias=True`` as in prior_arg, b_mask in w_mask."""
    w_mask, b_mask = mask if mask is not None else (None, None)
    if bias:
        w_mask, b_mask = b_mask, None
    if w_mask is None:
        return prior_arg(prior, bias), 0
    w_mu, w_sigma, b_mu, b_sigma = prior if prior is not None else (None, None, None, None)
    if bias:
        w_mu, w_sigma, b_mu, b_sigma = b_mu, b_sigma, None, None
    for t in (w_mu, w_sigma, b_mu, b_sigma, w_mask, b_mask):
        if t is not None:
            _require_cuda(t, "tensor prior / weight mask")
    p = lambda t: None if t is None else t.data_ptr()
    return C.byref(L.MaskedPrior(p(w_mu), p(w_sigma), p(b_mu), p(b_sigma), p(w_mask), p(b_mask))), L.PRIOR_MASKED


def desc_with(d: L.LayerDesc, flag: int) -> L.LayerDesc:
    """``d``, or a copy of it with ``flag`` (masked_prior_arg) in its kl_convention."""
    if not flag:
        return d
    c = L.LayerDesc.from_buffer_copy(d)
    c.kl_convention |= flag
    return c


def _stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _require_cuda(t: torch.Tensor, what: str):
    if not t.is_cuda:
        raise L.EngineError(
            f"{what}: tensor is on {t.device}; the Bayesian layer engine runs on CUDA (sm_90a) only "
            "and has no CPU fallback")


_ws_cache: dict = {}                              # shared scratch: (device, stream) -> buffer
_ws_layer = weakref.WeakKeyDictionary()           # layer-private scratch: module -> {(device, slot): buffer}; dies with the layer
_ws_slot = 0


def current_workspace_slot() -> int:
    return _ws_slot


@contextlib.contextmanager
def workspace_slot(k: int):
    """Layer workspaces (prepared operand tiles, KL partials and counters) are private per (layer, slot).
    Forwards that may run CONCURRENTLY -- e.g. two captured graphs replayed on two streams -- must be built
    under different slots; everything on one stream can share slot 0 (the default)."""
    global _ws_slot
    prev, _ws_slot = _ws_slot, int(k)
    try:
        yield
    finally:
        _ws_slot = prev


def workspace(device, desc=None, owner=None, kl_mc_draws: int = 0) -> torch.Tensor:
    """Zero-initialised scratch.  Without `owner`: one per (device, stream) -- calls on
    one stream are ordered, so sharing is safe and the kernels leave the counters
    zeroed.  With `owner` (a layer module): a private buffer sized by bbb_workspace_bytes(desc),
    which on the tensor-core path also holds that layer's prepared bf16 operand tiles; it is held
    through a weak reference to the layer, so it is freed with it and never re-bound to another one.
    ``kl_mc_draws`` > 0: the scratch of a Monte-Carlo KL call of that many draws instead
    (bbb_kl_mc_workspace_bytes), a buffer of its own beside the layer call's."""
    if kl_mc_draws:
        n = int(L.lib().bbb_kl_mc_workspace_bytes(int(kl_mc_draws)))
    else:
        n = int(L.lib().bbb_workspace_bytes(C.byref(desc) if desc is not None else None))
    kind = ("kl_mc",) if kl_mc_draws else ()
    if owner is None:
        cache, key = _ws_cache, (device.index, torch.cuda.current_stream(device).cuda_stream) + kind
    else:
        cache = _ws_layer.get(owner)
        if cache is None:
            cache = _ws_layer[owner] = {}
        key = (device.index, _ws_slot) + kind
    ws = cache.get(key)
    if ws is None or ws.numel() < n:
        if ws is not None:                        # a larger call (a BBB MC-sample fold) grows it: a graph captured on
            cache.setdefault("retired", []).append(ws)   # the old buffer still writes there, so it stays allocated
        ws = torch.zeros(n, dtype=torch.uint8, device=device)
        cache[key] = ws
    return ws


def make_desc(x_shape, w_shape, conv, variant, sample, has_bias, prior_mu, prior_sigma,
              math=L.MATH_FP32, kl_convention=L.KL_REFERENCE, act=L.ACT_NONE,
              act_dtype=L.DTYPE_F32, fold=None, first_image: int = 0) -> L.LayerDesc:
    """``fold`` = (rows per MC sample, Philox stream stride): the desc folds MC samples into its batch (layer_fold).
    ``first_image``: global index of image 0 (of each sample block when folded), in reserved[0] bits 8..30."""
    d = L.LayerDesc()
    if conv is None:
        d.batch, d.in_channels, d.in_h, d.in_w = x_shape[0], x_shape[1], 1, 1
        d.out_channels, d.kernel_h, d.kernel_w = w_shape[0], 1, 1
        d.stride_h = d.stride_w = d.dil_h = d.dil_w = 1
        d.pad_h = d.pad_w = 0
    else:
        (sh, sw), (ph, pw), (dh, dw) = conv
        d.batch, d.in_channels, d.in_h, d.in_w = x_shape
        d.out_channels, _, d.kernel_h, d.kernel_w = w_shape
        d.stride_h, d.stride_w, d.pad_h, d.pad_w, d.dil_h, d.dil_w = sh, sw, ph, pw, dh, dw
    d.variant, d.sample, d.has_bias = variant, int(bool(sample)), int(bool(has_bias))
    d.act_dtype, d.math, d.kl_convention, d.epilogue_act = act_dtype, math, kl_convention, act
    d.pool_k = d.pool_s = 0
    d.prior_mu, d.prior_sigma = float(prior_mu), float(prior_sigma)
    if fold is not None:
        rows, stride = fold
        d.reserved[1] = int(rows)
        d.reserved[2] = C.c_int32(stride & 0xFFFFFFFF).value
        d.reserved[3] = C.c_int32((stride >> 32) & 0xFFFFFFFF).value
    if first_image:
        d.reserved[0] = first_image_word(first_image)
    return d


def out_hw(h, w, kh, kw, conv):
    (sh, sw), (ph, pw), (dh, dw) = conv
    return ((h + 2 * ph - dh * (kh - 1) - 1) // sh + 1, (w + 2 * pw - dw * (kw - 1) - 1) // sw + 1)


# --------------------------------------------------------------------------- #
# tensor-core backward: wgrad / dgrad as role-swapped calls of the tensor-core layer kernel
# --------------------------------------------------------------------------- #
_TC_K_MAX = 8192          # the gather kernel keeps an 8-byte table entry per reduction index in shared memory


_tc_math = L.MATH_BF16_TC          # operand type of the backward contractions (set per call by _backward_tc)


def _tc_operand_math(math):
    """The operand type of the backward contractions of a layer on math mode `math`: the forward's (tf32, else bf16)."""
    return L.MATH_TF32_TC if math == L.MATH_TF32_TC else L.MATH_BF16_TC


def _tc_contract_desc(x_shape, w_shape, conv, math):
    """The desc of one contraction of the tensor-core backward (_tc_contract): the engine's forward of an x of
    `x_shape` with a weight of `w_shape`, sample=0, no bias -- host-only, so that support can be asked ahead."""
    return make_desc(tuple(x_shape), tuple(w_shape), conv, L.VARIANT_BBB, False, False, 0.0, 1.0, math)


def _tc_contract(x, w, conv):
    """Plain (mean-only, bias-free) conv2d / linear of fp32 `x` with the fp32 tensor `w` on the tensor-core layer kernel
    (bf16 or tf32 operands like the layer's forward, fp32 accumulators): the engine's forward with sample=0, no KL."""
    lib = L.lib()
    x, w = x.contiguous(), w.contiguous()
    d = _tc_contract_desc(x.shape, w.shape, conv, _tc_math)
    if conv is None:
        y = torch.empty(x.shape[0], w.shape[0], dtype=torch.float32, device=x.device)
        fn = lib.bbb_linear_forward
    else:
        oh, ow = out_hw(x.shape[2], x.shape[3], w.shape[2], w.shape[3], conv)
        y = torch.empty(x.shape[0], w.shape[0], oh, ow, dtype=torch.float32, device=x.device)
        fn = lib.bbb_conv2d_forward
    ws = workspace(x.device, d)
    rc = fn(C.byref(d), _ptr(x), _ptr(w), _ptr(w), None, None, _ptr(y), None, None, None, None,
            C.c_uint64(0), C.c_uint64(0), None, _ptr(ws), C.c_size_t(ws.numel()), _stream(x.device))
    L.check(rc, "tensor-core contraction (backward)")
    return y


def _tc_dgrad(g, w, conv, x_shape, contract=None):
    """d x of y = conv(x, w): the full correlation of (zero-inserted) g with the flipped, channel-transposed kernel --
    itself a stride-1 convolution, so it runs on the same tensor-core layer kernel.  ``contract``: what runs each
    contraction (default _tc_contract)."""
    contract = contract or _tc_contract
    if conv is None:
        return contract(g, w.t(), None)                                   # [B,N] x [K,N]^T -> [B,K]
    (sh, sw), (ph, pw), (dh, dw) = conv
    kh, kw = w.shape[2], w.shape[3]
    H, W = x_shape[2], x_shape[3]
    OH, OW = g.shape[2], g.shape[3]
    qh, qw = dh * (kh - 1) - ph, dw * (kw - 1) - pw
    if qh < 0 or qw < 0:
        return None
    hup = H - (dh * (kh - 1) - 2 * ph)                # rows of the zero-inserted gradient map: hup + 2*qh - dh*(kh-1) == H
    wup = W - (dw * (kw - 1) - 2 * pw)
    if (sh, sw) != (1, 1) or hup != OH or wup != OW:
        gu = g.new_zeros(g.shape[0], g.shape[1], hup, wup)
        gu[:, :, 0:(OH - 1) * sh + 1:sh, 0:(OW - 1) * sw + 1:sw] = g
        g = gu
    wt = w.flip(2, 3).transpose(0, 1)
    return contract(g, wt, ((1, 1), (qh, qw), (dh, dw)))


def _tc_wgrad(x, g, conv, w_shape, contract=None):
    """d w of y = conv(x, w): a convolution with the batch as the reduction ("channel") axis -- input x^T [C,B,H,W],
    kernel g^T [N,B,OH,OW], stride <-> dilation swapped -- on the tensor-core layer kernel.  Deterministic (no atomics);
    the batch is cut so that the reduction index fits the kernel's shared-memory table and the partial results summed.
    ``contract``: what runs each contraction (default _tc_contract)."""
    contract = contract or _tc_contract
    if conv is None:
        out = contract(x.t(), g.t(), None)                                 # [K,B] x [N,B]^T -> [K,N]
        return out.t()
    (sh, sw), (ph, pw), (dh, dw) = conv
    kh, kw = w_shape[2], w_shape[3]
    B = x.shape[0]
    per = max(1, _TC_K_MAX // (g.shape[2] * g.shape[3]))
    acc = None
    for b0 in range(0, B, per):
        xt = x[b0:b0 + per].transpose(0, 1)
        gt = g[b0:b0 + per].transpose(0, 1)
        part = contract(xt, gt, ((dh, dw), (ph, pw), (sh, sw)))[:, :, :kh, :kw]
        acc = part if acc is None else acc + part
    return acc.transpose(0, 1)


def _tc_backward_ok(cfg):
    return cfg["math"] in (L.MATH_BF16_TC, L.MATH_AUTO, L.MATH_TF32_TC) and os.environ.get("BBB_B200_BWD", "tc") != "simt"


def _tc_backward_contractions(x_shape, w_shape, conv, need_x=True):
    """(x shape, w shape, conv) of every distinct contraction the tensor-core backward of a layer call on an input of
    `x_shape` issues (_tc_wgrad, and _tc_dgrad with ``need_x``), recorded on the meta device without computing; None
    when _tc_dgrad gives up (padding > dilation * (kernel - 1): no stride-1 correlation gives the input gradient)."""
    calls = {}

    def out_shape(xs, ws, cv):
        return (xs[0], ws[0]) + (() if cv is None else out_hw(xs[2], xs[3], ws[2], ws[3], cv))

    def record(x, w, cv):
        calls[(tuple(x.shape), tuple(w.shape), cv)] = None
        return torch.empty(out_shape(x.shape, w.shape, cv), device="meta")

    x = torch.empty(tuple(x_shape), device="meta")
    w = torch.empty(tuple(w_shape), device="meta")
    g = torch.empty(out_shape(x.shape, w.shape, conv), device="meta")
    _tc_wgrad(x, g, conv, w.shape, contract=record)
    if need_x and _tc_dgrad(g, w, conv, x.shape, contract=record) is None:
        return None
    return list(calls)


def tc_backward_refusal(x_shape, w_shape, conv, math, need_x=True) -> Optional[str]:
    """Why the tensor-core backward of a layer call on an input of `x_shape` (math mode `math`) would not run -- the
    layer would then fall back to the CUDA-core kernels -- or None when it runs.  Host-only: it asks
    bbb_forward_supported, the check the kernel itself makes, about every contraction the backward would issue."""
    calls = _tc_backward_contractions(x_shape, w_shape, conv, need_x)
    if calls is None:
        return "the input gradient has no tensor-core contraction (padding > dilation * (kernel - 1))"
    lib = L.lib()
    for xs, ws, cv in calls:
        if lib.bbb_forward_supported(C.byref(_tc_contract_desc(xs, ws, cv, _tc_operand_math(math)))) != 0:
            return f"the contraction of x {xs} with w {ws} is refused: {lib.bbb_last_error().decode('utf-8', 'replace')}"
    return None


def _fold_grad_refusal(cfg, x_shape, w_shape, need_x) -> Optional[str]:
    """Why a layer call under layer_fold(grad=True) cannot record autograd, or None.  The CUDA-core backward does not
    know the fold: a call whose backward would fall back to it is refused here rather than given wrong gradients."""
    if cfg["variant"] != L.VARIANT_LRT:
        return "a BBB layer draws one weight sample per MC sample; only LRT layers train folded"
    if cfg["math"] == L.MATH_FP32:
        return "math='fp32' does not fold; use a tensor-core math mode (bf16, tf32 or auto)"
    if not _tc_backward_ok(cfg):
        return "the CUDA-core backward (BBB_B200_BWD=simt) does not fold"
    if external_eps_active():
        return "MC-sample folding draws its noise in-kernel (no external eps)"
    why = tc_backward_refusal(x_shape, w_shape, cfg["conv"], cfg["math"], need_x)
    return None if why is None else f"the backward would leave the tensor cores: {why}"


def layer_io(d: L.LayerDesc, x_dtype: torch.dtype) -> tuple[bool, torch.dtype]:
    """(bf16 activations, y dtype) of a layer call of desc ``d`` on an input of ``x_dtype``; sets ``d.act_dtype``.
    A bf16 input on math 'bf16' or 'auto' keeps its dtype: the engine reads bf16 x and writes bf16 y (act_dtype =
    BBB_DTYPE_BF16) wherever it accepts that desc (bbb_forward_supported, host-only), and otherwise the call runs on the
    upcast input and y is rounded to bf16 -- so y is bf16 either way.  Any other input (and a bf16 one on 'fp32' or
    'tf32') runs as fp32, with an fp32 y."""
    d.act_dtype = L.DTYPE_F32
    if x_dtype != torch.bfloat16 or d.math not in (L.MATH_BF16_TC, L.MATH_AUTO):
        return False, torch.float32
    d.act_dtype = L.DTYPE_BF16
    if L.lib().bbb_forward_supported(C.byref(d)) == 0:
        return True, torch.bfloat16
    d.act_dtype = L.DTYPE_F32
    return False, torch.bfloat16


# --------------------------------------------------------------------------- #
# the layer op
# --------------------------------------------------------------------------- #
class BayesLayerFn(torch.autograd.Function):
    """(y, kl) = layer(x; W_mu, W_rho, bias_mu, bias_rho).  One fused kernel forward;
    backward = bbb_*_backward + bbb_kl_backward accumulating into the same grads.
    A bf16 x on math 'bf16' / 'auto' gives a bf16 y (layer_io) and is saved as bf16; the backward runs on it and gy
    upcast to fp32 (both exact) and returns gx in x's dtype; parameter gradients and KL are fp32."""

    @staticmethod
    def forward(ctx, x, W_mu, W_rho, bias_mu, bias_rho, cfg):
        lib = L.lib()
        _require_cuda(x, "BayesLayerFn")
        _require_cuda(W_mu, "BayesLayerFn (parameters)")
        dev = x.device
        conv = cfg["conv"]
        variant, sample = cfg["variant"], cfg["sample"]
        x = x.contiguous()
        x_dtype = x.dtype
        W_mu_c, W_rho_c = W_mu.contiguous(), W_rho.contiguous()
        has_bias = bias_mu is not None
        need_grad = any(ctx.needs_input_grad[:5])      # grad mode is off inside Function.forward
        fold = _noise.fold
        if fold is not None and need_grad and cfg.get("grad_enabled", True):
            if not _noise.fold_grad:
                raise L.EngineError("layer_fold: MC-sample folding is forward-only (call under torch.no_grad())")
            why = _fold_grad_refusal(cfg, tuple(x.shape), tuple(W_mu.shape), ctx.needs_input_grad[0])
            if why is not None:
                raise L.EngineError(f"layer_fold(grad=True): {why}")
        if fold is not None and external_eps_active():
            raise L.EngineError("layer_fold: MC-sample folding draws its noise in-kernel (no external eps)")
        d = make_desc(tuple(x.shape), tuple(W_mu.shape), conv, variant, sample, has_bias,
                      cfg["prior_mu"], cfg["prior_sigma"], cfg["math"], cfg["kl_convention"], cfg["act"], fold=fold,
                      first_image=_noise.first_image)
        bf16_io, y_dtype = layer_io(d, x_dtype)
        if not bf16_io and x.dtype != torch.float32:
            x = x.float()
        if conv is None:
            if x.dim() != 2 or x.shape[1] != W_mu.shape[1]:
                raise L.EngineError(f"linear: x {tuple(x.shape)} vs weight {tuple(W_mu.shape)}")
            yshape = (x.shape[0], W_mu.shape[0])
        else:
            if x.dim() != 4 or x.shape[1] != W_mu.shape[1]:
                raise L.EngineError(f"conv2d: x {tuple(x.shape)} vs weight {tuple(W_mu.shape)}")
            oh, ow = out_hw(x.shape[2], x.shape[3], W_mu.shape[2], W_mu.shape[3], conv)
            yshape = (x.shape[0], W_mu.shape[0], oh, ow)
        y = torch.empty(yshape, dtype=x.dtype, device=dev)
        # a mixture prior has no closed-form KL: the forward computes none (kl_out NULL) and the caller takes the layer's
        # KL from KLMCFn; the `kl` returned here is then not a value
        kl = torch.empty((), dtype=torch.float32, device=dev)
        no_kl = cfg.get("mixture") is not None
        eps_a = eps_b = None
        seed = stream_id = 0
        base = None
        if sample:
            if external_eps_active():
                if variant == L.VARIANT_BBB:
                    eps_a = _pop_eps(W_mu.shape, dev)
                    if has_bias:
                        eps_b = _pop_eps(bias_mu.shape, dev)
                else:
                    eps_a = _pop_eps(yshape, dev)
            else:
                seed, stream_id = next_stream()
                base = _noise.base
        act_std = None
        if variant == L.VARIANT_LRT and sample and need_grad:
            act_std = torch.empty(yshape, dtype=torch.float32, device=dev)
        ws = workspace(dev, d, cfg.get("owner"))
        fn = lib.bbb_linear_forward_prior if conv is None else lib.bbb_conv2d_forward_prior
        parg, flag = masked_prior_arg(cfg.get("prior"), cfg.get("mask"))
        rc = fn(C.byref(desc_with(d, flag)), _ptr(x), _ptr(W_mu_c), _ptr(W_rho_c), _ptr(bias_mu), _ptr(bias_rho),
                _ptr(y), None if no_kl else _ptr(kl), _ptr(act_std), _ptr(eps_a), _ptr(eps_b),
                C.c_uint64(seed), C.c_uint64(stream_id), _ptr(base), _ptr(ws), C.c_size_t(ws.numel()), _stream(dev),
                parg)
        L.check(rc, "bbb_linear_forward" if conv is None else "bbb_conv2d_forward")
        if y.dtype != y_dtype:                      # a bf16 input the engine took as fp32
            y = y.to(y_dtype)
        d.act_dtype = L.DTYPE_F32                   # the backward runs on x and gy upcast to fp32
        ctx.cfg = cfg
        ctx.desc = d
        ctx.x_dtype = x_dtype
        ctx.noise = (seed, stream_id, base)
        ctx.first_image = _noise.first_image
        ctx.fold = fold
        ctx.has_bias = has_bias
        ctx.save_for_backward(x, W_mu_c, W_rho_c, bias_mu, bias_rho, act_std, eps_a, eps_b)
        if no_kl:
            ctx.mark_non_differentiable(kl)
        return y, kl

    @staticmethod
    def backward(ctx, gy, gkl):
        lib = L.lib()
        x, W_mu, W_rho, bias_mu, bias_rho, act_std, eps_a, eps_b = ctx.saved_tensors
        cfg, d = ctx.cfg, ctx.desc
        dev = x.device
        if cfg["act"] != L.ACT_NONE:
            raise L.EngineError("backward through a fused activation epilogue is not available")
        g_W_mu = torch.zeros_like(W_mu)
        g_W_rho = torch.zeros_like(W_rho)
        g_b_mu = torch.zeros_like(bias_mu) if ctx.has_bias else None
        g_b_rho = torch.zeros_like(bias_rho) if ctx.has_bias else None
        gx = None
        done = False
        if gy is not None and _tc_backward_ok(cfg):
            try:
                out = BayesLayerFn._backward_tc(ctx, gy.contiguous().float())
            except L.EngineError as e:
                if "code -2" not in str(e):                # BBB_E_UNSUPPORTED: a shape the tensor-core kernel does not take
                    raise
                out = None
            if out is None and ctx.fold is not None:
                raise L.EngineError("layer_fold(grad=True): the tensor-core backward refused a folded call")
            if out is not None:
                gx, gw_mu, gw_rho, gb_mu, gb_rho = out
                g_W_mu += gw_mu.reshape(g_W_mu.shape)
                g_W_rho += gw_rho.reshape(g_W_rho.shape)
                if ctx.has_bias:
                    g_b_mu += gb_mu
                    g_b_rho += gb_rho
                done = True
        if gy is not None and not done:
            gy = gy.contiguous().float()
            x = x.float()                                  # a saved bf16 x: exact (_backward_tc upcasts its own)
            if ctx.needs_input_grad[0]:
                gx = torch.zeros_like(x)
            ws = workspace(dev)
            fn = lib.bbb_linear_backward_prior if cfg["conv"] is None else lib.bbb_conv2d_backward_prior
            seed, stream_id, base = ctx.noise
            parg, flag = masked_prior_arg(None, cfg.get("mask"))
            rc = fn(C.byref(desc_with(d, flag)), _ptr(x), _ptr(gy), _ptr(W_mu), _ptr(W_rho), _ptr(bias_mu), _ptr(bias_rho),
                    _ptr(act_std), _ptr(eps_a), _ptr(eps_b), C.c_uint64(seed), C.c_uint64(stream_id), _ptr(base),
                    _ptr(gx), _ptr(g_W_mu), _ptr(g_W_rho), _ptr(g_b_mu), _ptr(g_b_rho),
                    _ptr(ws), C.c_size_t(ws.numel()), _stream(dev), parg)
            L.check(rc, "bbb_*_backward")
        if gx is not None and gx.dtype != ctx.x_dtype:
            gx = gx.to(ctx.x_dtype)
        if gkl is not None and cfg.get("mixture") is None:
            _kl_backward(gkl, (W_mu, W_rho, bias_mu, bias_rho), (g_W_mu, g_W_rho, g_b_mu, g_b_rho), cfg["prior_mu"],
                         cfg["prior_sigma"], cfg["kl_convention"], cfg.get("prior"), cfg.get("mask"))
        return gx, g_W_mu, g_W_rho, g_b_mu, g_b_rho, None


    @staticmethod
    def _backward_tc(ctx, gy):
        """SURVEY.md Appendix A on the tensor cores: every contraction of the backward (wgrad of the mean and of the
        variance path, dgrad of both) is a call of the tensor-core layer kernel with the operands' roles swapped; eps is
        regenerated from the forward's Philox stream; the element-wise chain rule through sigma = softplus(rho) is
        parameter-sized glue.  Returns None when a shape does not fit (the caller then uses the CUDA-core kernels).
        LRT: the noise term's gradient gv = gy * eps / (2 act_std) is one kernel (bbb_lrt_noise_grad) on the forward's
        desc, folded or not, which reads the stream base on the device.
        A weight mask selects, as in the forward: the dgrad operands are 0 at pruned elements and the parameter
        gradients are set to exactly 0 there (torch.where, so a pruned element's mu / rho never reach a value)."""
        x, W_mu, W_rho, bias_mu, bias_rho, act_std, eps_a, eps_b = ctx.saved_tensors
        x = x.float()
        cfg = ctx.cfg
        conv, variant, sample = cfg["conv"], cfg["variant"], cfg["sample"]
        dev = x.device
        global _tc_math
        _tc_math = _tc_operand_math(cfg["math"])           # same operand type as the forward
        seed, stream_id, base = ctx.noise
        need_x = ctx.needs_input_grad[0]
        w_keep, b_keep = cfg.get("mask") or (None, None)
        sig = torch.log1p(torch.exp(W_rho))
        dsig = torch.sigmoid(W_rho)
        if w_keep is not None:
            W_mu, sig = W_mu.where(w_keep, 0.0), sig.where(w_keep, 0.0)
        gb_mu = gb_rho = None
        red = (0,) if conv is None else (0, 2, 3)
        if variant == L.VARIANT_LRT:
            gw_mu = _tc_wgrad(x, gy, conv, W_mu.shape)
            if sample:
                if eps_a is None:
                    gv = lrt_noise_grad(ctx.desc, gy, act_std, seed, stream_id, base)
                else:
                    gv = gy * eps_a / (2.0 * act_std)
                gw_rho = _tc_wgrad(x * x, gv, conv, W_mu.shape) * (2.0 * sig * dsig)
            else:
                gv, gw_rho = None, torch.zeros_like(W_rho)
            gx = None
            if need_x:
                gx = _tc_dgrad(gy, W_mu, conv, x.shape)
                if gx is None:
                    return None
                if sample:
                    gx2 = _tc_dgrad(gv, sig * sig, conv, x.shape)
                    gx = gx + 2.0 * x * gx2
            if ctx.has_bias:
                gb_mu = gy.sum(red)
                if sample:
                    sb = torch.log1p(torch.exp(bias_rho))
                    gb_rho = gv.sum(red) * (2.0 * sb * torch.sigmoid(bias_rho))
                else:
                    gb_rho = torch.zeros_like(bias_rho)
        else:
            nw = W_mu.numel()
            if base is not None:
                stream_id = int(stream_id) + int(base.item())
            if sample:
                ew = eps_a if eps_a is not None else philox_normal(nw, seed, stream_id, 0, device=dev).view(W_mu.shape)
                W = W_mu + ew * sig
            else:
                ew, W = None, W_mu
            gw_mu = _tc_wgrad(x, gy, conv, W_mu.shape)
            gw_rho = gw_mu.reshape(W_mu.shape) * ew * dsig if sample else torch.zeros_like(W_rho)
            gx = None
            if need_x:
                gx = _tc_dgrad(gy, W, conv, x.shape)
                if gx is None:
                    return None
            if ctx.has_bias:
                gb_mu = gy.sum(red)
                if sample:
                    eb = eps_b if eps_b is not None else philox_normal(bias_mu.numel(), seed, stream_id, nw, device=dev)
                    gb_rho = gb_mu * eb * torch.sigmoid(bias_rho)
                else:
                    gb_rho = torch.zeros_like(bias_rho)
        if w_keep is not None:
            gw_mu = gw_mu.reshape(W_mu.shape).where(w_keep, 0.0)
            gw_rho = gw_rho.reshape(W_mu.shape).where(w_keep, 0.0)
        if b_keep is not None and ctx.has_bias:
            gb_mu, gb_rho = gb_mu.where(b_keep, 0.0), gb_rho.where(b_keep, 0.0)
        return gx, gw_mu, gw_rho, gb_mu, gb_rho


class KLFn(torch.autograd.Function):
    """kl_loss() with no preceding forward: sigma recomputed from rho in the kernel.  ``prior``: None (the scalar
    prior_mu / prior_sigma) or the tensor prior (w_mu, w_sigma, b_mu, b_sigma) of the layer (no gradient flows to it)."""

    @staticmethod
    def forward(ctx, W_mu, W_rho, bias_mu, bias_rho, prior_mu, prior_sigma, kl_convention, prior=None, mask=None):
        lib = L.lib()
        _require_cuda(W_mu, "kl_loss")
        dev = W_mu.device
        W_mu_c, W_rho_c = W_mu.contiguous(), W_rho.contiguous()
        kl = torch.empty((), dtype=torch.float32, device=dev)
        ws = workspace(dev)
        nb = 0 if bias_mu is None else bias_mu.numel()
        parg, flag = masked_prior_arg(prior, mask)
        rc = lib.bbb_kl_forward_prior(_ptr(W_mu_c), _ptr(W_rho_c), C.c_uint64(W_mu.numel()), _ptr(bias_mu),
                                      _ptr(bias_rho), C.c_uint64(nb), C.c_float(prior_mu), C.c_float(prior_sigma),
                                      C.c_int32(kl_convention | flag), _ptr(kl), _ptr(ws), C.c_size_t(ws.numel()),
                                      _stream(dev), parg)
        L.check(rc, "bbb_kl_forward_prior")
        ctx.save_for_backward(W_mu_c, W_rho_c, bias_mu, bias_rho)
        ctx.cfg = (float(prior_mu), float(prior_sigma), int(kl_convention))
        ctx.prior, ctx.mask = prior, mask
        return kl

    @staticmethod
    def backward(ctx, gkl):
        params = ctx.saved_tensors
        grads = tuple(None if t is None else torch.zeros_like(t) for t in params)
        _kl_backward(gkl, params, grads, *ctx.cfg, ctx.prior, ctx.mask)
        return grads + (None, None, None, None, None)


def _kl_backward(gkl, params, grads, prior_mu, prior_sigma, kl_convention, prior, mask=None):
    """gkl * d kl / d (mu, rho) added into ``grads``, the weight's then the bias's (bbb_kl_backward_prior; no call for a
    layer without a bias).  params = (W_mu, W_rho, bias_mu, bias_rho) and grads likewise; ``prior``: None or the layer's
    tensor prior; ``mask``: None or the layer's (W_mask, bias_mask) (nothing is added at a pruned element)."""
    lib = L.lib()
    gkl = gkl.contiguous().float()
    for k, bias in ((0, False), (2, True)):
        mu, rho = params[k], params[k + 1]
        if mu is None:
            continue
        parg, flag = masked_prior_arg(prior, mask, bias=bias)
        rc = lib.bbb_kl_backward_prior(_ptr(mu), _ptr(rho), C.c_uint64(mu.numel()), C.c_float(prior_mu),
                                       C.c_float(prior_sigma), C.c_int32(kl_convention | flag), _ptr(gkl),
                                       _ptr(grads[k]), _ptr(grads[k + 1]), _stream(mu.device), parg)
        L.check(rc, "bbb_kl_backward_prior")


def mixture_arg(mixture):
    """The ``const bbb_mixture_prior*`` argument of the Monte-Carlo KL entry points, from (pi, sigma1, sigma2)."""
    pi, sigma1, sigma2 = mixture
    return C.byref(L.MixturePrior(float(pi), float(sigma1), float(sigma2)))


def kl_draw_index(n_w: int, n: int, bias: bool = False) -> int:
    """Which normal of the KL draw's Philox stream element `n` of W (or of the bias: |W| + n) takes."""
    return int(n_w) + int(n) if bias else int(n)


def fold_draws(rows_total: int):
    """(n_draws, stream stride) of the Monte-Carlo KL of a layer call on `rows_total` rows: one draw per MC sample folded
    into the batch (layer_fold), else None -- one draw, a 0-dim KL."""
    if _noise.fold is None:
        return None
    rows, stride = _noise.fold
    return int(rows_total) // rows, stride


def kl_mc_forward(kl, W_mu, W_rho, bias_mu, bias_rho, mixture, seed, stream_id, base, stride=0, owner=None):
    """bbb_kl_mc_forward into the fp32 device tensor ``kl``: kl.numel() draws, draw d from Philox stream stream_id
    (+ the device scalar ``base``) + d * stride.  W_mu / W_rho contiguous."""
    dev = W_mu.device
    ws = workspace(dev, owner=owner, kl_mc_draws=kl.numel())
    nb = 0 if bias_mu is None else bias_mu.numel()
    rc = L.lib().bbb_kl_mc_forward(_ptr(W_mu), _ptr(W_rho), C.c_uint64(W_mu.numel()), _ptr(bias_mu), _ptr(bias_rho),
                                   C.c_uint64(nb), mixture_arg(mixture), C.c_uint64(seed), C.c_uint64(stream_id),
                                   _ptr(base), kl.numel(), C.c_uint64(stride & _MASK64), _ptr(kl), _ptr(ws),
                                   C.c_size_t(ws.numel()), _stream(dev))
    L.check(rc, "bbb_kl_mc_forward")


class KLMCFn(torch.autograd.Function):
    """Monte-Carlo KL(q || p) of a layer against the scale-mixture prior ``mixture`` = (pi, sigma1, sigma2)
    (bbb_kl_mc_forward; Blundell et al. 2015, section 3.3).  Takes the next Philox stream id of the calling thread, as a
    layer call takes its noise stream (next_stream, relative to the device base under stream_base), so the draw belongs
    to the Monte-Carlo sample the call is made in.  ``draws`` = (n, stride): n estimates [n], draw d from stream id +
    d * stride (the samples of an MC fold); None: one draw, 0-dim.  ``owner``: the layer whose private scratch the call
    uses (calls that may run concurrently); None: the stream's shared scratch.  The backward draws the same eps again."""

    @staticmethod
    def forward(ctx, W_mu, W_rho, bias_mu, bias_rho, mixture, draws=None, owner=None):
        _require_cuda(W_mu, "kl_loss (mixture prior)")
        W_mu_c, W_rho_c = W_mu.contiguous(), W_rho.contiguous()
        n_draws, stride = (1, 0) if draws is None else (int(draws[0]), int(draws[1]))
        seed, stream_id = next_stream()
        base = _noise.base
        kl = torch.empty(n_draws, dtype=torch.float32, device=W_mu.device)
        kl_mc_forward(kl, W_mu_c, W_rho_c, bias_mu, bias_rho, mixture, seed, stream_id, base, stride, owner)
        ctx.save_for_backward(W_mu_c, W_rho_c, bias_mu, bias_rho)
        ctx.call = (tuple(mixture), seed, stream_id, base, n_draws, stride)
        return kl if draws is not None else kl.view(())

    @staticmethod
    def backward(ctx, gkl):
        lib = L.lib()
        W_mu, W_rho, bias_mu, bias_rho = ctx.saved_tensors
        mixture, seed, stream_id, base, n_draws, stride = ctx.call
        dev = W_mu.device
        gkl = gkl.contiguous().float().reshape(-1)
        out = []
        for mu, rho, first in ((W_mu, W_rho, 0), (bias_mu, bias_rho, W_mu.numel())):
            if mu is None:
                out += [None, None]
                continue
            g_mu, g_rho = torch.zeros_like(mu), torch.zeros_like(rho)
            rc = lib.bbb_kl_mc_backward(_ptr(mu), _ptr(rho), C.c_uint64(mu.numel()), C.c_uint64(first),
                                        mixture_arg(mixture), C.c_uint64(seed), C.c_uint64(stream_id), _ptr(base),
                                        n_draws, C.c_uint64(stride & _MASK64), _ptr(gkl), _ptr(g_mu), _ptr(g_rho),
                                        _stream(dev))
            L.check(rc, "bbb_kl_mc_backward")
            out += [g_mu, g_rho]
        return out[0], out[1], out[2], out[3], None, None, None


# --------------------------------------------------------------------------- #
# small direct wrappers
# --------------------------------------------------------------------------- #
def philox_normal(n: int, seed: int, stream_id: int, offset: int = 0, device="cuda") -> torch.Tensor:
    """The engine's own noise stream, drawn on the host side of the boundary."""
    out = torch.empty(n, dtype=torch.float32, device=device)
    rc = L.lib().bbb_philox_normal_fill(_ptr(out), C.c_uint64(n), C.c_uint64(seed), C.c_uint64(stream_id),
                                        C.c_uint64(offset), _stream(out.device))
    L.check(rc, "bbb_philox_normal_fill")
    return out


def lrt_noise_grad(desc: L.LayerDesc, gy: torch.Tensor, act_std: torch.Tensor, seed: int, stream_id: int,
                   base: Optional[torch.Tensor] = None) -> torch.Tensor:
    """gv = gy * eps / (2 * act_std) of an LRT layer call, with eps drawn again from the streams of the forward of `desc`
    (its first image and MC-sample fold included; ``base``: the device stream base of a captured call) -- one kernel,
    no eps tensor (bbb_lrt_noise_grad).  gy and act_std: contiguous fp32 in y's shape."""
    gv = torch.empty_like(gy)
    rc = L.lib().bbb_lrt_noise_grad(C.byref(desc), _ptr(gy), _ptr(act_std), C.c_uint64(seed), C.c_uint64(stream_id),
                                    _ptr(base), _ptr(gv), _stream(gy.device))
    L.check(rc, "bbb_lrt_noise_grad")
    return gv


def mc_combine(logits: torch.Tensor, want_moments: bool = False):
    """logits [S,B,C] -> log_outputs [B,C] (main_bayesian.py:46-53) and optionally the
    [3,B,C] raw sums over the samples of (softmax, softmax^2, logits).  Do not form the epistemic variance as
    sum(p^2)/S - (sum(p)/S)^2 from them: when the samples agree the two terms are nearly equal and the fp32 difference is
    mostly rounding, often negative.  The exchange (mc_forward / MCForward) returns a centred epistemic variance."""
    _require_cuda(logits, "mc_combine")
    logits = logits.contiguous().float()
    S, B, Cc = logits.shape
    out = torch.empty(B, Cc, dtype=torch.float32, device=logits.device)
    mom = torch.empty(3, B, Cc, dtype=torch.float32, device=logits.device) if want_moments else None
    rc = L.lib().bbb_mc_combine(_ptr(logits), S, B, Cc, _ptr(out), _ptr(mom), _stream(logits.device))
    L.check(rc, "bbb_mc_combine")
    return (out, mom) if want_moments else out

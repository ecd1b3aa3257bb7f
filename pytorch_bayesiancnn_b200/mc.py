"""Monte-Carlo sample sharding, the one exchange of the forward path, and the heads above it (SURVEY.md 8e, f3, f4).

The reference's ``num_ens`` loop (main_bayesian.py:46-53, validate :75-80; uncertainty_estimation.py:70-78) runs S
independent weight samples of the SAME batch and combines them with logmeanexp of log-softmax.  Samples only differ in
their noise, so rank r of R takes the global sample ids {j : j mod R == r} (Philox stream namespace of sample j:
results do not depend on R) and ONE exchange carries the per-(image, class) partials and the KL.

Two implementations of the same contract:

* ``MCForward`` / ``mc_forward(net, ...)`` -- the product path on the CUDA engine: the local samples run through the
  engine (fused tensor-core chain where the net allows), then ONE kernel (``bbb_mc_exchange``, csrc/mc_head.cuh) reduces
  them, pushes the partials into every peer's receive buffer over NVLink (CUDA-IPC peer-mapped memory, no NCCL on the
  data path), waits for the peers and finishes logmeanexp, KL/num_ens, the ELBO head (metrics.py:12-14, 23-24) and the
  uncertainty outputs (uncertainty_estimation.py:80-96, softmax or softplus-normalised :73-77) on the device.  The whole
  step is one captured CUDA graph.
* ``mc_forward(forward_fn, ...)`` with a plain callable -- backend-agnostic host logic on torch.distributed (gloo on
  CPU in the tests): same sharding, same exact (max, sum-exp) partials, one all-gather.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import math
from typing import Callable, Optional

import os
import torch

from . import _lib as L
from . import functional as Fn


def local_samples(num_ens: int, world: int, rank: int):
    """Global sample ids owned by `rank` (round-robin; C4: 25 samples over 8 ranks -> 4,3,3,...)."""
    return list(range(rank, num_ens, world))


def row_block(B: int, batch_shards: int, block: int):
    """Images [b0, b1) of row block `block` of `batch_shards`: blocks as equal as possible, the first B % batch_shards one
    image longer (include/bbb_b200.h, bbb_mc_exchange_sharded)."""
    q, r = divmod(int(B), int(batch_shards))
    b0 = block * q + min(block, r)
    return b0, b0 + q + (1 if block < r else 0)


def shard_layout(world: int, rank: int, batch_shards: int = 1):
    """(sample_shards Rs, sample group g, row block k) of `rank` when `world` = Rs x batch_shards ranks split the samples
    into Rs groups and the batch into batch_shards row blocks: g = rank % Rs, k = rank // Rs."""
    rb = int(batch_shards)
    if rb < 1 or world % rb:
        raise L.EngineError(f"batch_shards={rb}: the world size {world} must be a multiple of it")
    rs = world // rb
    return rs, rank % rs, rank // rs


def _check_tensor(t, what, shape=None, dtype=None, device=None):
    """Raise EngineError unless ``t`` is contiguous and has the ``shape``, ``dtype`` and ``device`` given (None: any)."""
    shape = None if shape is None else tuple(shape)
    if t.is_contiguous() and all(w is None or w == g for w, g in ((shape, tuple(t.shape)), (dtype, t.dtype),
                                                                    (device, t.device))):
        return
    want = "".join((f" {dtype}" if dtype else "", " tensor", "" if shape is None else f" of shape {shape}",
                    f" on {device}" if device else ""))
    raise L.EngineError(f"{what}: expected a contiguous{want}, got {t.dtype} {tuple(t.shape)} on {t.device}")


def get_beta(batch_idx, m, beta_type, epoch=None, num_epochs=None):
    """metrics.py:32-46 (host scalar; it only feeds the `beta` argument of the ELBO head)."""
    if isinstance(beta_type, (int, float)):
        return float(beta_type)
    if beta_type == "Blundell":
        return 2 ** (m - (batch_idx + 1)) / (2 ** m - 1)
    if beta_type == "Soenderby":
        if epoch is None or num_epochs is None:
            raise ValueError("Soenderby method requires both epoch and num_epochs to be passed.")
        return min(epoch / (num_epochs // 4), 1)
    if beta_type == "Standard":
        return 1 / m
    return 0


# Memory budget of one folded pass on the per-layer path (MCForward, nets the fused chain does not take): G samples share
# a pass while G times the bytes one sample's pass holds at once stays within it.  Chosen from tools/mc_layer_fold_bench.py
# on C5 (one H100 80GB HBM3, 400 W power limit; README, Status): one step at a time G = 2 / 4 / 8 / 15 took 483 / 477 /
# 473 / 475 ms against 496 ms sample by sample, but with four steps in flight G = 4 / 8 took 470 / 478 ms against 466 ms.
# 2 GiB (G = 4 for C5) keeps most of the first gain and stays near even in flight.
LAYER_FOLD_BUDGET = 2 << 30
_INT32_MAX = (1 << 31) - 1


def layer_fold_groups(n_local: int, pass_bytes: int, max_elems: int, budget: int = LAYER_FOLD_BUDGET,
                      fold_group: Optional[int] = None):
    """How the per-layer fold groups a rank's ``n_local`` samples: a list of (first local index, size), consecutive and
    covering every local index once, in order, with sizes as equal as possible; None when no group would hold two samples.
    ``pass_bytes``: what one sample's pass holds at once (the largest fp32 input + output of any of its modules; aten ops
    between the layers are not in place).  ``max_elems``: the largest element count of one sample's activations -- a
    layer call keeps its counts in int32, so a group never exceeds 2^31 - 1 elements.  ``fold_group`` (> 0) replaces the
    byte budget as the largest group size."""
    cap = _INT32_MAX // max(1, int(max_elems))
    want = int(fold_group) if fold_group is not None else int(budget) // max(1, int(pass_bytes))
    g = min(int(n_local), want, cap)
    if g < 2:
        return None
    n = -(-int(n_local) // g)
    q, r = divmod(int(n_local), n)
    groups, start = [], 0
    for i in range(n):
        size = q + (1 if i < r else 0)
        groups.append((start, size))
        start += size
    return groups


def _per_image_chain(kids, x_shape):
    """What the children of a ModuleWrapper do, run one after another on a batch of ``x_shape``: (the Bayesian layers
    with their input shapes, pass bytes, largest element count) -- or None when a child is not known to treat every image
    on its own (then folding samples into the batch could change a result)."""
    from torch import nn
    from .modules import FlattenLayer, _BayesLayer
    shape, layers, pass_bytes, big = tuple(x_shape), [], 0, 0
    for m in kids:
        if isinstance(m, _BayesLayer):
            conv = m._conv_geometry()
            if conv is None:
                if len(shape) != 2 or shape[1] != m.in_features:
                    return None
                out = (shape[0], m.out_features)
            else:
                if len(shape) != 4 or shape[1] != m.in_channels:
                    return None
                out = (shape[0], m.out_channels) + Fn.out_hw(shape[2], shape[3], *m.kernel_size, conv)
            layers.append((m, shape))
        elif isinstance(m, FlattenLayer):
            if math.prod(shape[1:]) != m.num_features:
                return None                                  # view(-1, F) would mix the images of the batch
            out = (shape[0], m.num_features)
        elif isinstance(m, (nn.Softplus, nn.ReLU, nn.MaxPool2d)):
            out = tuple(m(torch.empty(shape, device="meta")).shape)
        else:
            return None
        a, b = math.prod(shape), math.prod(out)
        pass_bytes, big = max(pass_bytes, 4 * (a + b)), max(big, a, b)
        shape = out
    return layers, pass_bytes, big


def _dist_info(group):
    import torch.distributed as dist
    on = dist.is_available() and dist.is_initialized()
    return (dist if on else None), (dist.get_world_size(group) if on else 1), (dist.get_rank(group) if on else 0)


def _from_rank0(value, group):
    """Rank 0's ``value`` on every rank of ``group`` (torch.distributed's default group when None); on one rank
    ``value`` itself."""
    dist, world, _ = _dist_info(group)
    if world > 1:
        box = [value]
        dist.broadcast_object_list(box, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        value = box[0]
    return value


class MCForward:
    """``out = MCForward(net, example_x, num_ens, ...)(x, labels=None)`` -- the sharded MC step on the engine.

    Returns a dict of device tensors (the same objects every call; identical on all ranks):
      log_outputs [B,C], kl (= sum_j kl_j / num_ens; with mixture-prior layers kl_j is sample j's own Monte-Carlo
      estimate, drawn on sample j's streams whatever the sharding or fold), and with ``want_uncertainty`` pred /
      epistemic / aleatoric [B,C] and entropy [B]; with ``with_labels`` head = [loss, nll, accuracy, beta*kl] (metrics.py:12-14, 23-24); with
      ``want_information`` (needs ``want_uncertainty``) expected_entropy = mean_s H[p_hat_s] and mutual_info = entropy -
      expected_entropy [B] (include/bbb_b200.h, bbb_mc_exchange_info).

    ``metrics`` (needs ``with_labels``): an evaluation accumulator from ``new_metrics``; every step adds its validation
    loss and accuracy inputs and its calibration sums to it on the device (bbb_mc_exchange_metrics), so a held-out set
    needs one host read at the end (``read_metrics``).  Engines of different batch sizes may share one accumulator as long
    as their steps run one after another (``wait()`` the last step of one engine before the next engine's first); the
    warm-up steps the constructor runs do not count.

    ``batch_shards=Rb`` splits the batch as well as the samples: world = Rs x Rb ranks, rank r is sample group
    g = r % Rs (samples local_samples(num_ens, Rs, g)) and row block k = r // Rs (images ``rows`` = [b0, b1), row_block).
    Every rank is given the full x (and labels) and runs its samples on its rows only, with the LRT noise of image b drawn
    at b (Fn.first_image): the per-sample logits do not depend on (Rs, Rb), and every rank returns the same full
    outputs (bbb_mc_exchange_sharded).  Rb = 1 (default) is the sample-only split.
    """

    def __init__(self, net, example_x: torch.Tensor, num_ens: int, group=None, want_uncertainty: bool = False,
                 normalized: bool = False, with_labels: bool = False, train_size: float = 1.0, beta: float = 0.0,
                 seed: Optional[int] = None, graph: bool = True, num_classes: Optional[int] = None,
                 static_inputs=None, first_replay: int = 0, fold: bool = True, overlap: bool = False, inflight: int = 1,
                 fold_group: Optional[int] = None, fold_budget: int = LAYER_FOLD_BUDGET, want_information: bool = False,
                 batch_shards: int = 1, metrics: Optional[torch.Tensor] = None, cache_prep: bool = True,
                 score_log: Optional["ScoreLog"] = None, prob_bank: Optional["ProbBank"] = None,
                 conformal: Optional["ConformalLog"] = None, logit_bank: Optional["LogitBank"] = None,
                 temperature=None, scaling: Optional["LogitScaling"] = None):
        """``static_inputs``: device tensors the caller fills in place (e.g. targets of its host->device copies, or a
        rotation of resident batches); one graph is captured per tensor and ``self(slot=k)`` runs the step on
        ``static_inputs[k]`` with no staging copy.  ``first_replay``: index of the first replay's noise block.
        ``overlap``: run the exchange kernel of step t on its own stream, beside the first kernels of step t+1 (the
        layer chain of a step does not depend on the previous step's exchange; logits / KL terms / labels are double
        buffered).  The returned tensors are then complete on ``result_stream`` -- call ``wait()`` before using them on the
        current stream (a device synchronize covers it too).  ``inflight=k`` (with ``overlap``): consecutive steps are
        independent, so steps t, t+1, .. t+k-1 run on k streams with their own layer workspaces and Philox counters -- the
        head of step t+1 (parameter preps, first layers) fills the SMs the tail of step t leaves idle.  Results are
        identical to the serial engine; ``wait()`` also covers the inputs (they may be rewritten afterwards).
        ``fold_group``: the largest number of samples one pass of the per-layer fold takes (nets the fused chain does not
        take); None = as many as ``fold_budget`` bytes of activations allow (layer_fold_groups).
        ``cache_prep`` (captured engines whose fused chain is all LRT layers): the layers' bf16 operand tiles, bias rows
        and Gaussian KL are prepared by a graph of their own once per parameter version, into one workspace the steps
        read, instead of in every step (fused.PrepCache).  Before each step the host compares the version counters of
        the layers' parameters and prior buffers with those of the last prep and, when one moved, replays the prep first -- after the work enqueued on the current stream so far and after every step still in
        flight.  So an in-place update through an autograd-visible tensor (optimizer.step(), p.copy_() under no_grad,
        set_prior, load_state_dict) is read by the next step; a write through p.data or a raw pointer is not.  False:
        every step prepares its own operands, as a net with BBB layers always does.
        ``score_log``: a ScoreLog every step appends its B images' scores to (bbb_mc_score_log, one more kernel behind
        the exchange on the same stream): the outputs this engine computes, so ``want_uncertainty`` /
        ``want_information`` decide which planes hold numbers, and ``with_labels`` whether ``correct`` does.  Steps
        append in call order, in every mode; the warm-up steps the constructor runs do not.
        ``prob_bank``: a ProbBank every step appends its B images' per-sample probability rows to (bbb_mc_prob_log,
        behind the exchange on the same stream, as the score log), in call order, in every mode; the warm-up steps are
        not logged, and every output keeps its bits.  On several ranks the bank must have been made with this step's
        ``group``: every rank then gathers the step's per-sample logits of all S samples and B images (one more kernel
        per step, bbb_mc_logit_gather, in front of the temper) and fills its bank with the one-rank bank's bits.
        ``conformal``: a ConformalLog every step appends its B images' conformity scores and prediction sets to
        (bbb_mc_conformal_log, behind the exchange on the same stream, as the score log), from log_outputs and, with
        ``with_labels``, the labels; in call order, in every mode and with any sharding (every rank holds all B rows of
        log_outputs); the warm-up steps are not logged, and every output keeps its bits.
        ``logit_bank``: a LogitBank every step appends its B images' raw per-sample logits and labels to (bbb_mc_logit_log,
        in front of the temper and the exchange, on the same stream), in call order, in every mode; the warm-up steps are
        not logged.  On several ranks, as ``prob_bank``: made with this step's ``group``, filled from the gathered
        logits.
        ``temperature``: temper every sample's logits, z <- z / T, before the exchange (bbb_mc_temper, one more kernel per
        step): every output -- log_outputs, pred, the uncertainty and information planes, head, metrics and the logs behind
        the exchange -- is then that of p_bar_T = mean_s softmax(z_s / T).  A float, or a one-element fp32 tensor on the
        step's device that the step reads at run time: a value written into it in place is read by the next step, captured
        or not (fit_temperature(out=...)).  Not with ``normalized``.
        ``scaling``: a LogitScaling that maps every sample's logits, z <- a * z + b, before the exchange, in the
        temperature's place (bbb_mc_logit_scale, one more kernel per step): every output is then that of
        p_bar = mean_s softmax(a * z_s + b).  Its parameters are read at run time (fit_scaling(out=...) writes them in
        place).  Not with ``temperature`` or ``normalized``."""
        if want_information and not want_uncertainty:
            raise L.EngineError("MCForward: want_information needs want_uncertainty")
        Fn._require_cuda(example_x, "MCForward")
        lib = L.lib()
        if metrics is not None:
            if not with_labels:
                raise L.EngineError("MCForward: metrics needs with_labels")
            _check_tensor(metrics, "MCForward: metrics", dtype=torch.float64, device=example_x.device)
            n = int(lib.bbb_mc_metrics_bytes()) // 8
            if metrics.numel() < n:
                raise L.EngineError(f"MCForward: metrics holds {metrics.numel()} float64 elements, < {n} (mc.new_metrics)")
        self.metrics = self._metrics = metrics      # _metrics: the accumulator the exchange adds to
        self.net, self.group = net, group
        self.dist, self.world, self.rank = _dist_info(group)
        dev = self.dev = example_x.device
        self.num_ens = int(num_ens)
        self.C = int(num_classes if num_classes is not None else net.num_classes)
        # the logs the steps append to (_CursorLog._log), in the order their kernels are enqueued
        self._logs = [lg for lg in (logit_bank, score_log, prob_bank, conformal) if lg is not None]
        for lg in self._logs:
            lg._bind(self)
        # a step without labels logs label -1 into a logit bank, which the host must know of (LogitBank._unlabelled)
        self._unlabelled_bank = logit_bank if not with_labels else None
        self.temperature, self.scaling = _logit_map(temperature, scaling, example_x.device, normalized, self.C,
                                                    "MCForward")
        if self.world > 16:
            raise L.EngineError("MCForward: at most 16 ranks (one node)")
        self.sample_shards, self.group_index, self.block = shard_layout(self.world, self.rank, batch_shards)
        self.batch_shards = int(batch_shards)
        self.ids = local_samples(self.num_ens, self.sample_shards, self.group_index)
        self.B = int(example_x.shape[0])
        if self.batch_shards > self.B:
            raise L.EngineError(f"MCForward: batch_shards={self.batch_shards} > batch {self.B} (a row block would be empty)")
        self.rows = row_block(self.B, self.batch_shards, self.block)     # this rank's images [b0, b1)
        self.nb = self.rows[1] - self.rows[0]
        self.flags = (L.MC_MOMENTS if want_uncertainty else 0) | (L.MC_NORMALIZED if normalized else 0) | \
            (L.MC_INFO if want_information else 0)
        self.want_uncertainty, self.with_labels = want_uncertainty, with_labels
        self.train_size, self.beta = float(train_size), float(beta)
        # every rank must draw sample j from the same (seed, stream): share rank 0's seed unless one is given
        self.seed = int(seed if seed is not None else _from_rank0(Fn.current_seed(), group))
        B, Cc = self.B, self.C
        f32 = dict(dtype=torch.float32, device=dev)
        self.inputs = list(static_inputs) if static_inputs else [example_x.clone()]
        assert all(t.is_cuda and t.shape == example_x.shape and t.is_contiguous() for t in self.inputs)
        self.x = self.inputs[0]
        self.first_replay = int(first_replay)
        self.overlap = bool(overlap) and graph
        self.inflight = max(1, min(int(inflight), 8)) if self.overlap else 1
        self.nbuf = max(2, self.inflight) if self.overlap else 1
        nbuf = self.nbuf
        self.labels_all = torch.zeros(nbuf, B, dtype=torch.int64, device=dev) if with_labels else None
        self.labels = self.labels_all[0] if with_labels else None
        self.logits_all = torch.zeros(nbuf, max(1, len(self.ids)), self.nb, Cc, **f32)
        self.logits = self.logits_all[0]
        self.kl_one_all = torch.zeros(nbuf, **f32)
        self.kl_one = self.kl_one_all[0]
        self.kl_terms_all = torch.zeros(nbuf, 64, **f32)
        self.out = {"log_outputs": torch.empty(B, Cc, **f32), "kl": torch.empty((), **f32)}
        if want_uncertainty:
            for k in ("pred", "epistemic", "aleatoric"):
                self.out[k] = torch.empty(B, Cc, **f32)
            self.out["entropy"] = torch.empty(B, **f32)
        if want_information:
            self.out["expected_entropy"] = torch.empty(B, **f32)
            self.out["mutual_info"] = torch.empty(B, **f32)
        if with_labels:
            self.out["head"] = torch.empty(4, **f32)
        self.state = torch.zeros(int(lib.bbb_mc_state_bytes()), dtype=torch.uint8, device=dev)
        nbytes = int(lib.bbb_mc_buffer_bytes(B, Cc, self.flags, self.sample_shards))   # one slot per sample group
        # a sample bank on several ranks: every step gathers the logits of all S samples onto every rank, with a receive
        # buffer, a state and an [S, B, C] array per buffer parity of its own (None on one rank: nothing is gathered)
        gather = self.world > 1 and any(isinstance(lg, _SampleBank) for lg in self._logs)
        self._gather_state = self.gathered_all = None
        self._imported, self._own = [], []
        if self.world == 1:
            self._buf = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
            ptrs = [self._buf.data_ptr()]
        else:
            ptrs, *gptrs = self._open_peers(nbytes, *([int(lib.bbb_mc_gather_bytes(self.num_ens, B, Cc))] if gather
                                                       else []))
        self.peers = (C.c_void_p * self.world)(*ptrs)
        if gather:
            self._gather_peers = (C.c_void_p * self.world)(*gptrs[0])
            self._gather_state = torch.zeros(int(lib.bbb_mc_state_bytes()), dtype=torch.uint8, device=dev)
            self.gathered_all = torch.zeros(nbuf, self.num_ens, B, Cc, **f32)
        self.base = torch.zeros(1, dtype=torch.int64, device=dev)
        # The local samples FOLD into the batch -- one pass of the fused chain over S_local*B rows (what
        # uncertainty_estimation.py:38-41 does by repeating the input), each row drawing from its own sample's Philox
        # stream; the KL is computed once.  LRT samples differ only in their per-activation noise; a BBB layer prepares one
        # weight draw per sample and each row tile multiplies by its sample's draw.  Nets whose layers are all LRT or all
        # BBB fold when the engine accepts the folded chain (BBB: B a multiple of 128); the rest run sample by sample.
        self.fold_steps = None
        from . import fused
        from .modules import _BayesLayer
        kids = list(net.children())
        layers = [m_ for m_ in kids if isinstance(m_, _BayesLayer)]
        one_variant = bool(layers) and len({m_._variant for m_ in layers}) == 1 and getattr(net, "fuse", True)
        # Row blocks: everything below runs on this rank's nb rows; a group's local samples are g, g + Rs, .. (stream
        # stride Rs << 40).
        if fold and len(self.ids) > 1 and one_variant:
            self.fold = (self.nb, self.sample_shards << 40)
            with Fn.first_image(self.rows[0]):
                self.fold_steps = fused.plan(kids, (len(self.ids) * self.nb,) + tuple(example_x.shape[1:]), self.fold)
        # Nets the fused chain does not take (BBBLeNet, BBB3Conv3FC) fold on the per-layer path instead: groups of G
        # consecutive local samples, one pass of the tensor-core layer kernels over G x B rows each (Fn.layer_fold), with
        # the aten activations / pools between them -- per-image ops, so every output equals the sample loop's bit for bit.
        groups = None
        if self.fold_steps is None and fold and len(self.ids) > 1:
            groups = self._plan_layer_fold(net, kids, example_x, fold_group, fold_budget)
        self._set_passes(groups, example_x)
        self.graph, self.graphs = None, []
        self.cache_prep = bool(cache_prep)
        self._prep, self._prep_graph, self._prep_key = None, None, None     # set by _capture (fused.PrepCache)
        self._prep_watch = None
        self._prep_pending = set()                # buffer parities whose next step must wait for the last re-prep
        self.prep_replays = 0                     # replays of the prep graph (one per parameter version after the first)
        self.prep_kernels = 0                     # kernels of the prep graph
        self._prior_guard = None                   # set by _capture (modules.PriorGuard)
        self.result_stream = None                 # overlap mode: the stream the results are complete on
        self.replays = 0
        self.kernels_per_step = None
        if graph:
            self._capture()

    def _plan_layer_fold(self, net, kids, example_x, fold_group, budget):
        """The groups of the per-layer fold (layer_fold_groups), or None: the net runs on the fused chain unfolded (it
        then keeps the fused fold or the sample loop), a child is not a per-image op, or the engine would refuse a
        Bayesian layer's folded call (bbb_forward_supported: e.g. math='fp32', or a BBB layer whose 128-row tiles would
        straddle two samples)."""
        from . import fused
        from .modules import ModuleWrapper, _default_fuse
        if not kids or type(net).forward is not ModuleWrapper.forward:
            return None
        shape = (self.nb,) + tuple(example_x.shape[1:])
        if getattr(net, "fuse", _default_fuse()) and fused.plan(kids, shape) is not None:
            return None
        chain = _per_image_chain(kids, shape)
        if chain is None:
            return None
        layers, pass_bytes, big = chain
        groups = layer_fold_groups(len(self.ids), pass_bytes, big, budget, fold_group)
        if groups is None:
            return None
        fold = (self.nb, self.sample_shards << 40)
        for n in sorted({n for _, n in groups}):
            for m, xs in layers:
                if not _fold_forward_supported(m, xs, n, fold, self.rows[0]):
                    return None
        return groups

    def _set_passes(self, groups, example_x):
        """This rank's passes: (first local sample s0, sample count n) -- the fused fold's one pass over every local
        sample, the per-layer fold's ``groups``, or one pass per sample.  ``layer_fold`` = (G, number of groups) when the
        per-layer fold runs, else None."""
        self._groups, self.layer_fold = groups, None
        if self.fold_steps is not None:
            self.passes = [(0, len(self.ids))]
        elif groups is not None:
            self.passes = list(groups)
            G = max(n for _, n in groups)
            self.layer_fold = (G, len(groups))
            # the first layer's input: x repeated G times, one buffer per concurrently running step
            self.xrep_all = [torch.empty((G * self.nb,) + tuple(example_x.shape[1:]), dtype=example_x.dtype,
                                         device=self.dev) for _ in range(self.nbuf)]
        else:
            self.passes = [(k, 1) for k in range(len(self.ids))]

    def _pass_inputs(self, x, par=0, grad=False):
        """(s0, n, input, fold context) of every pass over this rank's row block ``x``.  Per-layer fold group (s0, n):
        local samples s0 .. s0+n-1 in one pass over x repeated n times; row block k is global sample ids[s0] + k * Rs
        (stream stride Rs << 40, as in the fused fold) and its logits are those of local sample s0 + k."""
        if self._groups is not None:
            xr, G = self.xrep_all[par], self.layer_fold[0]
            with torch.no_grad():
                xr.view((G,) + tuple(x.shape)).copy_(x.unsqueeze(0).expand((G,) + tuple(x.shape)))
        for s0, n in self.passes:
            if self._groups is None:
                yield s0, n, x, contextlib.nullcontext()
            else:
                yield s0, n, xr[:n * self.nb], Fn.layer_fold(self.nb, self.sample_shards << 40, grad=grad)

    # -- operand tiles and KL prepared once per parameter version (cache_prep) ---------------------------------------
    def _plan_prep(self, example_x):
        """The PrepCache of this engine's fused chain -- the LRT fold's, or the chain a sample's net(x) runs -- or None
        (no fused chain, or a layer that is not LRT)."""
        from . import fused
        from .modules import ModuleWrapper, _default_fuse
        if self.fold_steps is not None:
            steps, fold = self.fold_steps, self.fold
        elif (self._groups is None and type(self.net).forward is ModuleWrapper.forward
              and getattr(self.net, "fuse", _default_fuse())):
            with Fn.first_image(self.rows[0]):
                steps, fold = fused.plan(list(self.net.children()), (self.nb,) + tuple(example_x.shape[1:])), None
        else:
            return None
        return fused.PrepCache(steps, fold, self.dev) if fused.PrepCache.eligible(steps) else None

    def _prep_version(self):
        """The version counters of the tensors the prep graph reads: the layers' parameters, prior and mask buffers (the part of
        _BayesLayer._versions a replay can see -- the KL settings and the addresses are baked into the graphs, and a
        prior that is set anew is refused by PriorGuard).  About 2 us of host time for BBBAlexNet, where the whole
        _versions() tuple takes ten times that."""
        if self._prep_watch is None:
            from .modules import _MASK_BUFFERS, _PRIOR_BUFFERS
            self._prep_watch = [t for m in self._prep.layers for t in (m.W_mu, m.W_rho, m.bias_mu, m.bias_rho)
                                + tuple(m._buffers.get(n) for n in _PRIOR_BUFFERS + _MASK_BUFFERS) if t is not None]
        return [t._version for t in self._prep_watch]

    def _fill_prep(self):
        with torch.no_grad(), Fn.first_image(self.rows[0]):
            self._prep.fill()

    def _reprep(self):
        """Replay the prep graph: after the current stream's work so far (in-place updates the caller enqueued) and after
        every step that may still read the tiles or the KL; the steps enqueued from now on wait for it."""
        cur = torch.cuda.current_stream(self.dev)
        if self.overlap:
            ps = self._prep_stream
            ps.wait_stream(cur)
            for ev, seen in zip(self._exch_done, self._exch_seen):     # the last step of each buffer parity: its
                if seen:                                                 # exchange follows its chain
                    ps.wait_event(ev)
            with torch.cuda.stream(ps):
                self._prep_graph.replay()
            self._prep_done.record(ps)
            self._prep_pending = set(range(self.nbuf))
        else:
            self._prep_graph.replay()              # stream order: behind the steps before, in front of this one
        self.prep_replays += 1

    # -- peer-mapped receive buffers (CUDA IPC; handles travel over torch.distributed) -----------------------
    def _open_peers(self, *sizes):
        """One receive buffer of each size in ``sizes`` on every rank, mapped into every peer: per buffer, the list of
        every rank's pointer (the local one at [rank])."""
        lib = L.lib()
        torch.cuda.synchronize(self.dev)
        with torch.cuda.device(self.dev):
            mine = []
            for nbytes in sizes:
                own = C.c_void_p()
                L.check(lib.bbb_comm_alloc(C.c_size_t(nbytes), C.byref(own)), "bbb_comm_alloc")
                self._own.append(own.value)
                handle = (C.c_ubyte * 64)()
                L.check(lib.bbb_comm_export(C.c_void_p(own.value), handle), "bbb_comm_export")
                mine.append(bytes(handle))
            handles = [None] * self.world
            self.dist.all_gather_object(handles, mine, group=self.group)
            bufs = []
            for i, own in enumerate(self._own):
                ptrs = []
                for q, h in enumerate(handles):
                    if q == self.rank:
                        ptrs.append(own)
                        continue
                    peer = C.c_void_p()
                    L.check(lib.bbb_comm_import((C.c_ubyte * 64).from_buffer_copy(h[i]), C.byref(peer)),
                            f"bbb_comm_import (rank {q})")
                    self._imported.append(peer.value)
                    ptrs.append(peer.value)
                bufs.append(ptrs)
        self.dist.barrier(group=self.group)
        return bufs

    def timeouts(self) -> int:
        """Exchange and gather waits that gave up because a peer never delivered (results of those steps are invalid)."""
        states = [self.state] + ([self._gather_state] if self._gather_state is not None else [])
        return sum(int(st[8:12].view(torch.int32).item()) for st in states)

    def close(self):
        """Unmap the peers' buffers and free the local ones (after every rank is done with them)."""
        lib = L.lib()
        if self.world > 1 and self._own:
            torch.cuda.synchronize(self.dev)
            self.dist.barrier(group=self.group)
            for p in self._imported:
                lib.bbb_comm_unimport(C.c_void_p(p))
            for p in self._own:
                lib.bbb_comm_free(C.c_void_p(p))
            self._imported, self._own = [], []

    # -- one step ----------------------------------------------------------------------------------------------
    def _step(self, x, base=None, advance=False):
        """This rank's samples through the engine, then the exchange kernel."""
        kl_ptr, n_kl = self._chain(x, base, advance)
        self._exchange(kl_ptr, n_kl)
        return self.out

    def _mean_kl(self, kls, par=0):
        """Nets with mixture-prior layers: every sample has its own KL estimate.  ``kls``: the local samples' KLs in
        local order (0-dim tensors, or vectors of folded samples).  Their mean goes where the exchange reads one sample's
        KL, which it multiplies by the local sample count.  The sum is taken over one [n_local] vector on every path, so
        folded and sample-loop steps agree bit for bit."""
        v = torch.cat([torch.as_tensor(k, dtype=torch.float32, device=self.dev).detach().reshape(-1) for k in kls])
        one = self.kl_one_all[par:par + 1]
        one.copy_((v.sum() / v.numel()).reshape(1))
        return Fn._ptr(one), 1

    def _kl_arg(self, kls, terms=False, par=0):
        """The (pointer, count) of the floats whose sum is one sample's KL, from the passes' KLs ``kls`` (local order):
        with mixture-prior layers the mean of the per-sample estimates (_mean_kl).  Otherwise every sample has the same
        KL, which a pass computes once: the first pass's per-layer scalars when a fused chain handed them over un-summed
        (``terms``), else its scalar."""
        from .modules import has_mixture
        if has_mixture(self.net):
            return self._mean_kl(kls, par)
        if terms:
            self._kl_terms = kls[0]                      # kept alive: a captured exchange reads it
            return Fn._ptr(kls[0]), kls[0].numel()
        one = self.kl_one_all[par:par + 1]
        one.copy_(torch.as_tensor(kls[0], dtype=torch.float32, device=self.dev).detach().reshape(1))
        return Fn._ptr(one), 1

    def _chain(self, x, base=None, advance=False, par=0):
        """This rank's samples through the engine into the sample buffer ``par``.  A fused chain writes its logits
        straight into it and hands over its per-layer KL scalars un-summed (fused.direct_output).  Returns the (pointer,
        count) of the floats whose sum is one sample's KL."""
        from . import fused
        from .graph import _STRIDE
        logits_buf = self.logits_all[par]
        kl_buf = self.kl_terms_all[par] if self.overlap else None
        b0, nb = self.rows[0], self.nb
        x = x[b0:b0 + nb]                                 # this rank's row block (a view: NCHW rows are contiguous)
        with torch.no_grad(), Fn.workspace_slot(par if self.inflight > 1 else Fn.current_workspace_slot()), \
                Fn.first_image(b0), fused.use_prep(self._prep):
            # The Philox base moves at the HEAD of a captured step, BEFORE the prep streams fork: with this one-thread
            # kernel as the single root of the graph every GEMM kernel of the chain is launched programmatically behind
            # its predecessor; with the fork in front of it (prep kernels as further root nodes) or with no plain kernel
            # at the head, the programmatic edges of the whole chain are lost and every GEMM waits for its predecessor.
            # With the operands prepared ahead (self._prep) there is no prep in the step: the first GEMM kernel follows
            # this one directly.
            if advance:
                Fn.noise_advance(base, _STRIDE * self.inflight)
            kls, terms = [], False
            for s0, n, xin, fold_ctx in self._pass_inputs(x, par):
                out = logits_buf[s0:s0 + n].view(n * nb, self.C)
                with Fn.stream_base(base), Fn.mc_sample(self.ids[s0], self.seed), fold_ctx:
                    if self.fold_steps is not None:
                        _, kl = fused._run(self.fold_steps, xin, True, out, True, None, fold=self.fold, kls_out=kl_buf)
                        taken = True
                    else:                                 # (the fused chain never takes a per-layer fold's pass)
                        with fused.direct_output(out, kl_buf if s0 == 0 else None) as hook:
                            logits, kl = self.net(xin)
                        taken = hook.used
                if not taken:
                    out.copy_(logits.reshape(n * nb, self.C))
                if s0 == 0:
                    terms = taken
                kls.append(kl)
            if not self.ids and self.group_index == 0:
                raise L.EngineError("MCForward: sample group 0 must own a sample")
            return self._kl_arg(kls, terms, par) if kls else (None, 0)

    def _exchange(self, kl_ptr, n_kl, advance_base=None, par=0):
        """The one kernel behind the samples: combine + exchange + heads (bbb_mc_exchange_sharded; with an evaluation
        accumulator bbb_mc_exchange_metrics)."""
        from .graph import _STRIDE
        o = self.out
        lib = L.lib()
        if self._gather_state is not None:
            L.check(lib.bbb_mc_logit_gather(Fn._ptr(self.logits_all[par]) if self.ids else None, len(self.ids),
                                            self.num_ens, self.B, self.C, self.rank, self.world, self.batch_shards,
                                            self._gather_peers, Fn._ptr(self._gather_state),
                                            Fn._ptr(self.gathered_all[par]), Fn._stream(self.dev)), "bbb_mc_logit_gather")
        for lg in self._logs:
            if lg.before_temper:
                lg._log(self, par)
        if self.ids:
            self._map(self.logits_all[par])
        args = (
            Fn._ptr(self.logits_all[par]), len(self.ids), self.num_ens, self.B, self.C, kl_ptr, n_kl, self.flags,
            Fn._ptr(self._labels_of(par)), C.c_float(self.train_size), C.c_float(self.beta), self.rank, self.world, self.peers,
            Fn._ptr(self.state), Fn._ptr(o["log_outputs"]), Fn._ptr(o["kl"]), Fn._ptr(o.get("pred")),
            Fn._ptr(o.get("epistemic")), Fn._ptr(o.get("aleatoric")), Fn._ptr(o.get("entropy")), Fn._ptr(o.get("head")),
            Fn._ptr(advance_base), C.c_uint64(_STRIDE if advance_base is not None else 0),
            Fn._ptr(o.get("expected_entropy")), Fn._ptr(o.get("mutual_info")))
        if self._metrics is not None:
            L.check(lib.bbb_mc_exchange_metrics(*args, self.batch_shards, Fn._ptr(self._metrics), Fn._stream(self.dev)),
                    "bbb_mc_exchange_metrics")
        else:
            L.check(lib.bbb_mc_exchange_sharded(*args, self.batch_shards, Fn._stream(self.dev)), "bbb_mc_exchange_sharded")
        for lg in self._logs:
            if not lg.before_temper:
                lg._log(self, par)

    def _labels_of(self, par):
        """The labels of buffer parity ``par``, or None without ``with_labels``."""
        return self.labels_all[par] if self.labels_all is not None else None

    def _map(self, z):
        """The temperature or the scaling, in place on per-sample logits ``z`` (bbb_mc_temper / bbb_mc_logit_scale on
        the step's stream); nothing without either."""
        if self.scaling is not None:
            self.scaling._launch(z, Fn._stream(self.dev))
        elif self.temperature is not None:
            L.check(L.lib().bbb_mc_temper(Fn._ptr(z), z.numel(), Fn._ptr(self.temperature), Fn._stream(self.dev)),
                    "bbb_mc_temper")

    def _bank_logits(self, par, mapped=False):
        """The per-sample logits [S, B, C] of buffer parity ``par`` a sample bank logs: on one rank the step's own (the
        map has run on them once the temper slot is passed), on several the gathered ones, raw -- or, with ``mapped``,
        after the step's map, applied here.  The map works element by element or row by row, so mapping the gathered
        logits gives the bits of gathering the mapped ones."""
        if self._gather_state is None:
            return self.logits_all[par]
        z = self.gathered_all[par]
        if mapped:
            self._map(z)
        return z

    def _capture(self, warmup: int = 2):
        from .graph import _STRIDE
        from .modules import PriorGuard
        dev = self.dev
        self._prior_guard = PriorGuard(self.net)   # the layers' prior buffers as the graphs read them
        # several steps in flight: the tap-GEMM layers take their 128-column tiles wherever Cout allows (throughput over the
        # latency of one step; the choice is made at launch = capture time, include/bbb_b200.h bbb_set_wide_tiles)
        prev_wide = L.lib().bbb_set_wide_tiles(1 if self.inflight > 1 else 0)
        # Engines cached on a net (mc_forward, evaluate) form a reference cycle with it.  If the cyclic collector freed a
        # dropped one in the middle of this capture, destroying its CUDA graphs would invalidate the capture: collect
        # before, and keep the collector off while capturing.
        import gc
        gc.collect()
        gc_on = gc.isenabled()
        gc.disable()
        try:
            self._capture_graphs(warmup)
        finally:
            if gc_on:
                gc.enable()
            L.lib().bbb_set_wide_tiles(prev_wide)

    def _capture_graphs(self, warmup):
        from .graph import _STRIDE
        dev = self.dev
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        live, live_logs = self._metrics, self._logs
        if live is not None:
            self._metrics = torch.zeros_like(live)      # the warm-up steps do not count
        self._logs = [lg._empty() for lg in live_logs]   # nor are they logged (a log of no capacity drops them)
        self._prep = self._plan_prep(self.x) if self.cache_prep else None
        with torch.cuda.stream(side):
            if self._prep is not None:              # the first prep, which the warm-up steps already read
                self._prep_key = self._prep_version()
                self._fill_prep()
            for _ in range(warmup):                 # eager: creates plans / workspaces; every rank runs the same exchanges
                self._step(self.x, self.base)
            for p_ in range(1, self.inflight):      # the other in-flight steps' own layer workspaces
                self._exchange(*self._chain(self.x, self.base, par=p_), par=p_)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self._metrics, self._logs = live, live_logs
        # GEMM chain on a HIGH-priority stream, parameter preps on the (default-priority) side streams: when both have CTAs
        # pending, the chain's go first -- the preps of later layers no longer keep the first GEMM's CTAs off the SMs
        cap = torch.cuda.Stream(device=dev, priority=-1)
        # A folded pass of the per-layer path holds up to fold_budget bytes of activations, which a captured graph keeps in
        # its memory pool: the chain graphs that never run at the same time (one per resident input, same buffer parity)
        # share one pool instead of one each.
        pools = {}

        def pool_kw(par):
            return {"pool": pools.get(par)} if self._groups is not None else {}

        def keep_pool(par, g):
            if self._groups is not None:
                pools.setdefault(par, g.pool())
        if self._prep is not None:
            self._prep_graph = torch.cuda.CUDAGraph()
            n0 = L.launch_count()
            with torch.cuda.graph(self._prep_graph, stream=cap):
                self._fill_prep()
            self.prep_kernels = L.launch_count() - n0
            self._prep_stream = torch.cuda.Stream(device=dev, priority=-1)
            self._prep_done = torch.cuda.Event()
        if self.overlap:
            # two graphs per step: the layer chain (per resident input and buffer parity) and the exchange kernel (per
            # parity); __call__ replays the second on its own stream so that it runs beside the next step's chain
            nb = self.nbuf
            self.chain_graphs, self.exch_graphs = [[] for _ in range(nb)], []
            self.base2 = torch.zeros(nb, dtype=torch.int64, device=dev)
            self._bases = [self.base2[p_:p_ + 1] for p_ in range(nb)] if self.inflight > 1 else [self.base] * nb
            for par in range(nb):
                for xin in self.inputs:
                    g = torch.cuda.CUDAGraph()
                    n0 = L.launch_count()
                    with torch.cuda.graph(g, stream=cap, **pool_kw(par)):
                        kl_ptr, n_kl = self._chain(xin, self._bases[par], advance=True, par=par)
                    keep_pool(par, g)
                    n_chain = L.launch_count() - n0
                    self.chain_graphs[par].append(g)
                g = torch.cuda.CUDAGraph()
                n0 = L.launch_count()
                with torch.cuda.graph(g, stream=cap):
                    self._exchange(kl_ptr, n_kl, par=par)
                n_exch = L.launch_count() - n0
                self.exch_graphs.append(g)
            self.kernels_per_step = n_chain + n_exch
            self.graphs = self.chain_graphs[0]
            # the exchange kernel is tiny and latency-critical (peers wait for it): highest priority the device offers
            lo = getattr(torch.cuda.Stream, "priority_range", lambda: (-1, 0))()
            self.result_stream = torch.cuda.Stream(device=dev, priority=min(lo))
            self._chain_done = [torch.cuda.Event() for _ in range(nb)]
            self._exch_done = [torch.cuda.Event() for _ in range(nb)]
            self._exch_seen = [False] * nb          # has a step of buffer parity p been enqueued (its exchange event recorded)
            self._in_ready = [torch.cuda.Event() for _ in range(nb)]
            self.chain_streams = [torch.cuda.Stream(device=dev, priority=-1) for _ in range(nb)] if self.inflight > 1 else None
            # torch creates an event at its first record: create them all now (nothing is pending), so that every step is
            # enqueued by one native call on their raw handles (bbb_mc_graph_step) -- the host work of a step is then a
            # small fraction of its ~0.1 ms on the device, where the runtime calls made one by one from Python were not
            events = self._chain_done + self._exch_done + self._in_ready + \
                ([self._prep_done] if self._prep is not None else [])
            for ev in events:
                ev.record(cap)
            rs_raw = self.result_stream.cuda_stream
            # per (parity, input slot): run stream (None = the caller's current stream), in_ready, chain graph, chain
            # event, result stream, exchange graph, exchange event
            self._step_handles = [[(self.chain_streams[p_].cuda_stream if self.chain_streams else None,
                                    self._in_ready[p_].cuda_event, g_.raw_cuda_graph_exec(), self._chain_done[p_].cuda_event,
                                    rs_raw, self.exch_graphs[p_].raw_cuda_graph_exec(), self._exch_done[p_].cuda_event)
                                   for g_ in self.chain_graphs[p_]] for p_ in range(nb)]
            # replay r draws noise block first_replay + r: with k counters, counter p starts k blocks back and moves by k
            for p_ in range(nb):
                self.base2[p_] = (self.first_replay + p_ - nb) * _STRIDE
        for xin in (() if self.overlap else self.inputs):
            g = torch.cuda.CUDAGraph()
            n0 = L.launch_count()
            with torch.cuda.graph(g, stream=cap, **pool_kw(0)):
                self._step(xin, self.base, advance=True)
            keep_pool(0, g)
            self.kernels_per_step = L.launch_count() - n0          # engine kernels captured in one step
            self.graphs.append(g)
        self.graph = self.graphs[0]
        self.base.fill_((self.first_replay - 1) * _STRIDE)

    def __call__(self, x: Optional[torch.Tensor] = None, labels: Optional[torch.Tensor] = None, slot: int = 0):
        if labels is not None and self.labels is None:
            raise L.EngineError("MCForward was built without with_labels=True")
        if self._unlabelled_bank is not None:
            self._unlabelled_bank._unlabelled = True   # this step logs label -1
        if self._prior_guard is not None:
            self._prior_guard.check("MCForward")
        if self._prep_graph is not None:
            key = self._prep_version()
            if key != self._prep_key:
                self._reprep()
                self._prep_key = key
        if self.overlap:
            # Step `par` (even / odd / .. steps on their own streams when several are in flight) runs behind the caller's
            # work so far, behind the exchange of the last step of the same parity (which read buffers `par`) and, for the
            # first step of `par` since a re-prep, behind the prep.  Its exchange follows on result_stream.
            par = self.replays % self.nbuf
            h = self._step_handles[par][slot]
            wait_a = self._exch_done[par].cuda_event if self._exch_seen[par] else None
            wait_b = self._prep_done.cuda_event if par in self._prep_pending else None
            self._prep_pending.discard(par)
            cur_raw = torch._C._cuda_getCurrentRawStream(self.dev.index)
            if labels is not None or x is not None:       # the copies go on the step's stream, behind its waits
                cur = torch.cuda.current_stream(self.dev)
                run = self.chain_streams[par] if self.inflight > 1 else cur
                if run is not cur:
                    self._in_ready[par].record(cur)
                    run.wait_event(self._in_ready[par])
                for ev in (self._exch_done[par] if wait_a else None, self._prep_done if wait_b else None):
                    if ev is not None:
                        run.wait_event(ev)
                with torch.cuda.stream(run):
                    if labels is not None:
                        self.labels_all[par].copy_(labels, non_blocking=True)
                    if x is not None:
                        self.inputs[slot].copy_(x, non_blocking=True)
                cur_raw, wait_a, wait_b = run.cuda_stream, None, None
            L.check(L.lib().bbb_mc_graph_step(cur_raw, h[0] if h[0] is not None else cur_raw, h[1], wait_a, wait_b,
                                              h[2], h[3], h[4], h[5], h[6]), "bbb_mc_graph_step")
            self._exch_seen[par] = True
            self._last = par
            self.replays += 1
            return self.out
        if labels is not None:
            self.labels.copy_(labels, non_blocking=True)
        if self.graph is not None:
            if x is not None:
                self.inputs[slot].copy_(x, non_blocking=True)
            self.graphs[slot].replay()
            self.replays += 1
            return self.out
        return self._step(self.inputs[slot] if x is None else x.to(self.dev))

    def wait(self):
        """Make the current stream wait for the last step's results (a no-op unless built with ``overlap=True``)."""
        if self.overlap and self.replays and self._exch_seen[self._last]:
            # exchanges run in step order on one stream and each follows its chain: the last one covers everything before
            torch.cuda.current_stream(self.dev).wait_event(self._exch_done[self._last])
        return self.out

    def input_consumed(self):
        """Event after which the input of the LAST step may be rewritten (its layer chain has read it); None = stream order
        of the current stream already says so."""
        return self._chain_done[self._last] if (self.overlap and self.replays) else None


def chan_merge(counts, means, m2s):
    """Merge per-group (count, mean, M2 = sum (x - mean)^2) in the order given with Chan's update
    M2 = M2a + M2b + d^2 na nb / (na + nb), d = mean_b - mean_a; groups with count 0 are skipped.  Returns (mean, M2)
    of all the samples.  The variance stays a centred sum: no E[x^2] - mean^2, which cancels when the samples agree."""
    n, mean, m2 = 0, None, None
    for nq, mq, m2q in zip(counts, means, m2s):
        if nq == 0:
            continue
        if mean is None:
            n, mean, m2 = nq, mq.clone(), m2q.clone()
            continue
        nn = n + nq
        d = mq - mean
        mean = mean + d * (nq / nn)
        m2 = m2 + m2q + d * d * (n * nq / nn)
        n = nn
    return mean, m2


def _generic_mc_forward(forward_fn: Callable, x: torch.Tensor, num_ens: int, group=None, want_uncertainty: bool = False,
                        information: bool = False, batch_shards: int = 1):
    """Backend-agnostic restatement (any device, any torch.distributed backend): the exact (max, sum-exp) partials of
    logmeanexp per rank and ONE all-gather; returns (log_outputs, kl[, (pred, epistemic, aleatoric, entropy)]) --
    with ``information`` the tuple also holds expected_entropy and mutual_info (each rank's sum of H[p_hat_s] over its
    samples travels as one more [B] plane of the same all-gather).  ``batch_shards``: as MCForward -- rank (g, k) calls
    ``forward_fn`` on its row block x[b0:b1] (under Fn.first_image(b0)), the groups are merged in ascending order and
    each group's KL is counted once (block 0)."""
    dist, world, rank = _dist_info(group)
    rs, g, k = shard_layout(world, rank, batch_shards)
    rb = world // rs
    B = int(x.shape[0])
    if rb > B:
        raise L.EngineError(f"mc_forward: batch_shards={rb} > batch {B} (a row block would be empty)")
    b0, b1 = row_block(B, rb, k)
    ids = local_samples(num_ens, rs, g)
    parts, shape, dev = None, None, x.device
    with Fn.first_image(b0):
        for j in ids:
            logits, kl = forward_fn(x[b0:b1], j)
            logits = logits.float()
            shape, dev = logits.shape, logits.device
            lsm = torch.log_softmax(logits, dim=1)
            p = lsm.exp()
            klv = torch.as_tensor(kl, dtype=torch.float32, device=dev).reshape(1)
            if information:
                h = -torch.where(p > 0, p * lsm, torch.zeros_like(p)).sum(1)   # H[p_hat_j], 0 log 0 = 0
            if parts is None:                         # planes 2, 3: Welford mean and M2 = sum (p - mean)^2 of p_hat
                parts = [lsm.clone(), torch.ones_like(lsm), p.clone(), torch.zeros_like(p), logits.clone(), klv.clone()]
                if information:
                    parts.append(h)
                n = 1
            else:
                m = torch.maximum(parts[0], lsm)
                parts[1] = parts[1] * (parts[0] - m).exp() + (lsm - m).exp()
                parts[0] = m
                n += 1
                d = p - parts[2]
                parts[2] += d / n; parts[3] += d * (p - parts[2]); parts[4] += logits; parts[5] += klv
                if information:
                    parts[6] += h
    if world > 1:
        metas = [None] * world
        dist.all_gather_object(metas, tuple(shape) if shape is not None else None, group=group)
        ncls = next(s_[1] for s_ in metas if s_ is not None)
    else:
        ncls = shape[1]
    nb, P = b1 - b0, -(-B // rb)                      # rows of this block; rows of the longest block
    shape = (nb, ncls)
    if parts is None:                                 # a rank with no sample (num_ens < Rs) still joins the collective
        z = torch.zeros(shape, dtype=torch.float32, device=dev)
        parts = [torch.full(shape, -float("inf"), device=dev), z, z.clone(), z.clone(), z.clone(), torch.zeros(1, device=dev)]
        if information:
            parts.append(torch.zeros(shape[0], device=dev))
    if nb < P:                                        # ragged blocks: every rank sends the longest block's size
        pad = lambda t: torch.cat([t, t.new_zeros((P - nb,) + tuple(t.shape[1:]))])
        parts = [t if i == 5 else pad(t) for i, t in enumerate(parts)]
    vec = torch.cat([t.reshape(-1) for t in parts])
    if world > 1:
        allv = [torch.empty_like(vec) for _ in range(world)]
        dist.all_gather(allv, vec, group=group)       # the ONE collective of the forward path
    else:
        allv = [vec]
    n, full = P * ncls, (B, ncls)

    def plane(i, width=ncls, off=None):
        """[Rs] list of plane i of every sample group over all B rows (rank r fills rows row_block(.., r // Rs))."""
        off = i * n if off is None else off
        out = [torch.empty((B, width) if width > 1 else (B,), dtype=vec.dtype, device=vec.device) for _ in range(rs)]
        for r, v in enumerate(allv):
            c0, c1 = row_block(B, rb, r // rs)
            out[r % rs][c0:c1] = v[off:off + (c1 - c0) * width].view(out[r % rs][c0:c1].shape)
        return out
    S = float(num_ens)
    ms = torch.stack(plane(0))
    as_ = torch.stack(plane(1))
    M = ms.max(0).values
    tot = (as_ * torch.where(as_ > 0, (ms - M).exp(), torch.zeros_like(ms))).sum(0)
    log_outputs = (M + torch.log(tot / S)).view(full)          # == logmeanexp_j log_softmax_j (utils.py:14-22), finite
    kl = sum(v[5 * n] for r, v in enumerate(allv) if r // rs == 0) / S      # main_bayesian.py:51; one block per group
    if not want_uncertainty:
        return log_outputs, kl
    counts = [len(local_samples(num_ens, rs, q)) for q in range(rs)]
    p_bar, m2 = chan_merge(counts, plane(2), plane(3))
    p_bar, m2 = p_bar.view(full), m2.view(full)
    pred = (sum(plane(4)) / S).view(full)
    epistemic = m2 / S                                # diag((p-pbar)^T (p-pbar))/T, centred (uncertainty_estimation.py:89-91)
    aleatoric = p_bar * (1.0 - p_bar) - epistemic     # diag(diag(pbar) - p^T p / T) = pbar - E[p^2]  (:94-95)
    entropy = -(p_bar * torch.log(p_bar.clamp_min(1e-38))).sum(1)      # H[pbar]; no reference (SURVEY D3)
    if not information:
        return log_outputs, kl, (pred, epistemic, aleatoric, entropy)
    expected_entropy = sum(plane(6, 1, 5 * n + 1)) / S      # E_j H[p_hat_j], group order
    return log_outputs, kl, (pred, epistemic, aleatoric, entropy, expected_entropy, entropy - expected_entropy)


def mc_forward(net_or_fn, x: torch.Tensor, num_ens: int, group=None, want_uncertainty: bool = False,
               normalized: bool = False, labels: Optional[torch.Tensor] = None, train_size: float = 1.0,
               beta: float = 0.0, seed: Optional[int] = None, information: bool = False, batch_shards: int = 1):
    """(log_outputs [B,C], kl) like main_bayesian.py:46-53 -- plus (pred, epistemic, aleatoric, entropy) like
    uncertainty_estimation.py:70-96 with ``want_uncertainty`` and the ELBO head [loss, nll, acc, beta*kl] when
    ``labels`` are given.  ``information`` (needs ``want_uncertainty``) extends that tuple to (pred, epistemic, aleatoric,
    entropy, expected_entropy, mutual_info).  ``net_or_fn``: a net built on the engine with CUDA input -> the device path
    (MCForward, cached on the net per shape/options); any ``forward_fn(x, sample_id) -> (logits, kl)`` -> the generic
    path.  ``batch_shards``: split the batch into that many row blocks as well (MCForward); 1 = samples only."""
    from .modules import ModuleWrapper
    if information and not want_uncertainty:
        raise L.EngineError("mc_forward: information needs want_uncertainty")
    if isinstance(net_or_fn, ModuleWrapper) and x.is_cuda:
        net = net_or_fn
        key = (tuple(x.shape), int(num_ens), bool(want_uncertainty), bool(normalized), labels is not None,
               float(train_size), float(beta), seed, id(group), bool(information), int(batch_shards))
        cache = _engine_cache(net, "_mc_engines")
        eng = cache.get(key)
        if eng is None:
            eng = cache[key] = MCForward(net, x, num_ens, group, want_uncertainty, normalized, labels is not None,
                                         train_size, beta, seed, want_information=information,
                                         batch_shards=batch_shards)
        out = eng(x, labels)
        res = [out["log_outputs"], out["kl"]]
        if want_uncertainty:
            res.append(tuple(out[k] for k in ("pred", "epistemic", "aleatoric", "entropy") +
                             (("expected_entropy", "mutual_info") if information else ())))
        if labels is not None:
            res.append(out["head"])
        return tuple(res)
    return _generic_mc_forward(net_or_fn, x, num_ens, group, want_uncertainty, information, batch_shards)


def _engine_cache(net, name):
    """The engine cache `name` kept on the net (mc_forward: "_mc_engines", evaluate: "_mc_eval").  Both are dropped when a
    layer's prior was set, cleared, re-allocated or moved since their engines were captured (modules.PriorGuard), so
    the next call captures engines that read the layers' current priors."""
    from .modules import PriorGuard
    guard = net.__dict__.get("_mc_prior_guard")
    if guard is None or not guard.ok():
        net.__dict__.pop("_mc_engines", None)
        net.__dict__.pop("_mc_eval", None)
        net.__dict__["_mc_prior_guard"] = PriorGuard(net)
    return net.__dict__.setdefault(name, {})


def new_metrics(device) -> torch.Tensor:
    """A zeroed evaluation accumulator for ``MCForward(metrics=...)`` (bbb_mc_metrics_bytes of float64 words)."""
    return torch.zeros(int(L.lib().bbb_mc_metrics_bytes()) // 8, dtype=torch.float64, device=device)


def read_metrics(t: torch.Tensor) -> dict:
    """One host read of an evaluation accumulator (layout: include/bbb_b200.h, bbb_mc_exchange_metrics).

    ``steps``, ``images``; validate_model's inputs ``sum_nll_step`` / ``sum_acc_step`` (sums of the per-batch means) and
    ``klsum`` (sum_j kl_j of one step, the mean over steps); over all images ``nll``, ``accuracy``, ``brier`` (mean
    sum_c (p_bar_c - [c == y])^2) and ``ece`` (sum_m |correct_m - conf_m| / images over the MC_CAL_BINS equal-width
    confidence bins); per bin ``bin_count``, ``bin_confidence`` and ``bin_accuracy`` (means; nan for an empty bin) -- a
    reliability diagram."""
    nb = L.MC_CAL_BINS
    a = t[:8 + 3 * nb].cpu().tolist()
    steps, images = a[0], a[1]
    div = lambda x, n: x / n if n else float("nan")
    cnt, conf, cor = a[8:8 + nb], a[8 + nb:8 + 2 * nb], a[8 + 2 * nb:8 + 3 * nb]
    return {"steps": int(steps), "images": int(images), "sum_nll_step": a[2], "sum_acc_step": a[3],
            "klsum": div(a[4], steps), "nll": div(a[5], images), "accuracy": div(a[6], images), "brier": div(a[7], images),
            "ece": div(sum(abs(cor[m] - conf[m]) for m in range(nb)), images),
            "bin_count": [int(c) for c in cnt], "bin_confidence": [div(conf[m], cnt[m]) for m in range(nb)],
            "bin_accuracy": [div(cor[m], cnt[m]) for m in range(nb)]}


class _CursorLog:
    """What a data-set-long device log shares: the two-word cursor of bbb_mc_score_log / bbb_mc_prob_log (next index,
    images dropped) and its host reads.

    A log the Monte-Carlo step appends to -- MCForward's keyword ``_keyword`` -- also implements the step's hooks:
    ``_bind(step)`` refuses an engine being built that it cannot log, ``_empty()`` is a log of no capacity with the same
    options (what the engine's warm-up steps append to), and ``_log(step, par)`` enqueues the append from the step's
    buffers of parity ``par``: in front of the temper when ``before_temper`` (the log holds the raw logits), else
    behind the exchange."""

    _keyword = None
    before_temper = False

    def _bind(self, step):
        if self.device != step.dev:
            raise L.EngineError(f"MCForward: {self._keyword} is on {self.device}, the step on {step.dev}")

    def _init_cursor(self, device, capacity: int, what: str):
        capacity = int(capacity)
        if capacity < 0:
            raise ValueError(f"{what}: capacity must be >= 0 (got {capacity})")
        self.device = torch.device(device)
        if self.device.type == "cuda" and self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.capacity = capacity
        self._cursor = torch.zeros(2, dtype=torch.int64, device=self.device)     # next index, images dropped

    def reset(self):
        """Start the log again (stream-ordered: after the work enqueued on the current stream so far)."""
        self._cursor.zero_()

    def _counts(self):
        nxt, dropped = self._cursor.tolist()
        return min(nxt, self.capacity), dropped

    def __len__(self):
        """Entries held (a host read of the cursor)."""
        return self._counts()[0]

    @property
    def dropped(self) -> int:
        """Images that did not fit (a host read of the cursor)."""
        return self._counts()[1]

    def _held(self, what: str) -> int:
        """Entries held; raises EngineError if images were dropped."""
        n, dropped = self._counts()
        if dropped:
            raise L.EngineError(f"{what}: {dropped} images did not fit (capacity {self.capacity}, "
                                f"{n + dropped} logged)")
        return n


class ScoreLog(_CursorLog):
    """A data-set-long log of per-image scores on the device, appended to by the Monte-Carlo step (bbb_mc_score_log):
    ``MCForward(..., score_log=log)`` and ``evaluate(..., score_log=log)`` add one entry per image, in step order, with
    no host read; ``read()`` returns the entries once the data set is done.

    Entry i holds ``confidence`` = max_c p_bar (exp of the largest log_output; the first maximal class is ``pred``),
    ``entropy`` = H[p_bar], ``mutual_info`` and ``expected_entropy`` (the BALD decomposition), ``epistemic`` = sum_c of
    the epistemic variance, ``correct`` = 1.0 / 0.0 (pred == label), and ``pred`` (int32).  A score the step does not
    compute (no ``want_uncertainty`` / ``want_information`` / labels) is NaN.  ``capacity`` entries fit; images past
    them are counted, not written, and ``read()`` refuses a log that dropped any."""

    PLANES = ("confidence", "entropy", "mutual_info", "expected_entropy", "epistemic", "correct")
    _keyword = "score_log"

    def __init__(self, device, capacity: int):
        self._init_cursor(device, capacity, "ScoreLog")
        assert len(self.PLANES) == L.MC_SCORE_PLANES
        # (one column at least: an empty tensor has no address, and the kernel takes the log's pointers even when
        # nothing fits)
        self._planes = torch.zeros(L.MC_SCORE_PLANES, max(1, capacity), dtype=torch.float32, device=self.device)
        self._pred = torch.zeros(max(1, capacity), dtype=torch.int32, device=self.device)

    def _empty(self):
        return ScoreLog(self.device, 0)

    def _log(self, step, par):
        o = step.out
        self.append(o["log_outputs"], o.get("entropy"), o.get("expected_entropy"), o.get("mutual_info"),
                    o.get("epistemic"), step._labels_of(par))

    def read(self) -> dict:
        """The entries logged so far: {plane name: float32 [n], "pred": int32 [n]}, copies on the log's device.  Raises
        EngineError if images were dropped.  Steps in flight must be complete first (``MCForward.wait()``)."""
        n = self._held("ScoreLog")
        out = {k: self._planes[i, :n].clone() for i, k in enumerate(self.PLANES)}
        out["pred"] = self._pred[:n].clone()
        return out

    def append(self, log_outputs, entropy=None, expected_entropy=None, mutual_info=None, epistemic=None, labels=None):
        """Append one step's images (bbb_mc_score_log on the current stream): log_outputs [B, C] and the optional
        [B] / [B, C] uncertainty outputs and int64 labels [B] of the same step, fp32 contiguous on the log's device."""
        Fn._require_cuda(self._cursor, "ScoreLog.append")
        B, Cc = log_outputs.shape
        for t, shape, dt in ((log_outputs, (B, Cc), torch.float32), (entropy, (B,), torch.float32),
                             (expected_entropy, (B,), torch.float32), (mutual_info, (B,), torch.float32),
                             (epistemic, (B, Cc), torch.float32), (labels, (B,), torch.int64)):
            if t is not None:
                _check_tensor(t, "ScoreLog.append", shape, dt, self.device)
        L.check(L.lib().bbb_mc_score_log(Fn._ptr(log_outputs), Fn._ptr(entropy), Fn._ptr(expected_entropy),
                                         Fn._ptr(mutual_info), Fn._ptr(epistemic), Fn._ptr(labels), B, Cc,
                                         Fn._ptr(self._planes), Fn._ptr(self._pred), self.capacity,
                                         Fn._ptr(self._cursor), Fn._stream(self.device)), "bbb_mc_score_log")


def evaluate(net, loader, num_ens: int, train_size: float, beta_type=0.1, epoch=None, num_epochs=None, group=None,
             seed: Optional[int] = None, inflight: int = 4, batch_shards: int = 1, normalized: bool = False,
             score_log: Optional[ScoreLog] = None, prob_bank: Optional["ProbBank"] = None,
             conformal: Optional["ConformalLog"] = None, logit_bank: Optional["LogitBank"] = None,
             temperature=None, scaling: Optional["LogitScaling"] = None) -> dict:
    """main_bayesian.validate_model over ``loader`` (batches of (inputs, labels)) on the engine, with calibration.

    Returns read_metrics' dict plus ``valid_loss`` and ``valid_acc`` as validate_model computes them: the mean over
    batches of nll_loss * train_size + beta_i * kl, with beta_i = get_beta(i - 1, len(loader), ...) for batch i (0-based)
    and kl = sum_j kl_j (not divided by num_ens); the mean over batches of the batch accuracy.

    Every batch runs through an in-flight engine (``overlap=True, inflight``), one per batch shape, all adding to one
    device accumulator; the host reads it once, at the end.  Inputs and labels go into rotating device slots (the
    engine's static_inputs), each rewritten only after the step that last read it has consumed it; host batches that are
    not pinned are first copied into pinned slots, so the host can run up to ``max(2, inflight)`` batches ahead.  The
    engines and the accumulator are kept on the net, as mc_forward keeps its engines, for the next call with the same
    options (the next epoch); each call draws fresh noise.  Every rank must iterate the same loader (as MCForward
    requires).

    ``normalized``: p_hat_s is the softplus-normalised row (uncertainty_estimation.py:73-77), not the softmax.
    ``score_log``: a ScoreLog every image is appended to, in loader order (after what it already holds: ``reset()`` it
    to start over).  The engines then also compute the uncertainty and information outputs; the returned figures are
    the same bits as without a log.  Engines are kept per log object: reuse a log from epoch to epoch.
    ``prob_bank``: a ProbBank every image's per-sample probability rows are appended to, in loader order, as the score
    log is (on several ranks the bank's ``group`` must be ``group``: every rank then holds all of it); the returned figures
    keep their bits.
    ``conformal``: a ConformalLog every image's conformity score and prediction set are appended to, in loader order,
    as the score log is; the returned figures keep their bits.  Engines are kept per log object.
    ``logit_bank``: a LogitBank every image's raw per-sample logits and label are appended to, in loader order (as
    ``prob_bank`` on several ranks; calibrate_temperature fills one); the returned figures keep their bits.
    ``temperature``: MCForward's -- every figure, log and bank behind the exchange is that of the tempered predictive.
    Engines are kept per temperature tensor (a float: per value), and read a value written into the tensor in place.
    ``scaling``: MCForward's, kept and read in place as a temperature tensor is."""
    dev = next(net.parameters()).device
    logs = dict(score_log=score_log, prob_bank=prob_bank, conformal=conformal, logit_bank=logit_bank)
    key = (int(num_ens), float(train_size), seed, id(group), int(inflight), int(batch_shards), bool(normalized),
           *(None if lg is None else id(lg) for lg in logs.values()), _map_key(temperature), _map_key(scaling))
    ev = _engine_cache(net, "_mc_eval").get(key)
    if ev is None:
        # (the entry holds the logs and the maps its key names by id, so that no other object takes their id)
        ev = net.__dict__["_mc_eval"][key] = {"acc": new_metrics(dev), "engines": {}, "seed": seed,
                                              "logs": [lg for lg in logs.values() if lg is not None],
                                              "maps": (temperature, scaling)}
    ev["acc"].zero_()

    def build(slots, first_replay):
        return MCForward(net, slots[0], num_ens, group, with_labels=True, train_size=train_size, seed=ev["seed"],
                         static_inputs=slots, first_replay=first_replay, overlap=True, inflight=inflight,
                         batch_shards=batch_shards, metrics=ev["acc"], normalized=normalized,
                         want_uncertainty=score_log is not None, want_information=score_log is not None,
                         temperature=temperature, scaling=scaling, **logs)
    n = _run_loader(ev, loader, dev, max(2, int(inflight)), build)
    if not n:
        raise ValueError("evaluate: the loader yielded no batch")
    m = read_metrics(ev["acc"])
    beta_sum = sum(get_beta(i - 1, n, beta_type, epoch, num_epochs) for i in range(n))
    m["valid_loss"] = (float(train_size) * m["sum_nll_step"] + beta_sum * m["klsum"]) / n
    m["valid_acc"] = m["sum_acc_step"] / n
    return m


def _run_loader(entry, loader, dev, nslots, build, **call_kw):
    """The loader loop of evaluate and route: every batch (x, y) through the in-flight step of its shape in the cache
    ``entry`` (an MCForward or ExpertStep, made by ``build(slots, first_replay)`` over ``nslots`` rotating input slots
    when the shape first comes), as ``step(labels=, slot=, **call_kw)``.  Returns the number of batches, with the
    current stream behind the last step."""
    engines, cur = entry["engines"], torch.cuda.current_stream(dev)
    last, n = None, 0
    for x, y in loader:
        shape = (tuple(x.shape), x.dtype)
        e = engines.get(shape)
        if e is None:
            slots = [torch.zeros(x.shape, dtype=x.dtype, device=dev) for _ in range(nslots)]
            # the k-th step built draws noise blocks k * 2^16, k * 2^16 + 1, ...: steps do not share noise
            eng = build(slots, len(engines) << 16)
            entry["seed"] = eng.seed            # every step draws from the same seed
            e = engines[shape] = {"eng": eng, "slots": slots, "consumed": [None] * nslots, "steps": 0,
                                  "labels": [torch.zeros(x.shape[0], dtype=torch.int64, device=dev) for _ in range(nslots)],
                                  "pinned": [None] * nslots}
        eng = e["eng"]
        if last is not None and last is not eng:
            last.wait()                         # the accumulator and the logs take the steps one after another
        s = e["steps"] % nslots
        x, y = _pinned(e, s, x, y)
        if e["consumed"][s] is not None:
            # the step that last read slot s has consumed it.  The event is the engine's per-parity chain event, which a
            # later step of the same parity may have recorded again: waiting on it can only wait longer.
            cur.wait_event(e["consumed"][s])
        e["slots"][s].copy_(x, non_blocking=True)
        e["labels"][s].copy_(y, non_blocking=True)  # the step copies them on its own stream: they must outlive the call
        if e["pinned"][s] is not None:
            e["pinned"][s][2].record(cur)       # the pinned slot may be refilled once these copies are done
        eng(labels=e["labels"][s], slot=s, **call_kw)
        e["consumed"][s] = eng.input_consumed()
        e["steps"] += 1
        last, n = eng, n + 1
    if last is not None:
        last.wait()
    return n


def _kept_log(net, store: dict, key, loader, make, fits=lambda log: True):
    """The log that detect_ood, acquire, conformal or calibrate_temperature keeps for the net in ``store[key]``, reset
    and sized for ``loader``: ``make(capacity)`` makes a new one when there is none yet, or the one kept holds fewer
    entries than the loader has images, is on another device than the net or does not pass ``fits``.  evaluate's
    engines that append to the old log go with it."""
    dev = next(net.parameters()).device
    n = _loader_images(loader)
    log = store.get(key)
    if log is None or log.capacity < n or log.device != dev or not fits(log):
        if log is not None:
            cache = net.__dict__.get("_mc_eval", {})
            for k in [k for k, e in cache.items() if any(lg is log for lg in e["logs"])]:
                del cache[k]
        log = store[key] = make(n)
    log.reset()
    return log


def _pinned(e, s, x, y):
    """(x, y), with host tensors that are not pinned copied into pinned slot s of engine entry e (after the previous
    copies out of that slot have finished), so that the copies to the device do not hold up the host."""
    if (x.is_cuda or x.is_pinned()) and (y.is_cuda or y.is_pinned()):
        return x, y
    if e["pinned"][s] is None:
        e["pinned"][s] = (torch.empty(x.shape, dtype=x.dtype).pin_memory(),
                          torch.empty(y.shape, dtype=y.dtype).pin_memory(), torch.cuda.Event())
    hx, hy, done = e["pinned"][s]
    done.synchronize()
    if not (x.is_cuda or x.is_pinned()):
        hx.copy_(x)
        x = hx
    if not (y.is_cuda or y.is_pinned()):
        hy.copy_(y)
        y = hy
    return x, y


def engine_forward_fn(net, seed: Optional[int] = None, offset: int = 0) -> Callable:
    """forward_fn for a net built on the engine: draws Monte-Carlo sample j (and leaves the training stream untouched).
    ``seed`` / ``offset``: Fn.mc_sample's; an engine's replay r draws sample j at offset (first_replay + r) << 20."""
    def fn(x, j):
        with Fn.mc_sample(j, seed, offset), torch.no_grad():
            return net(x)
    return fn


# Below this log p_bar[b, y_b] (p_bar < 1e-26) MCTrainStep forms the loss gradient's softmax / p_bar ratio in log space.
# Above it both factors are far from fp32 underflow: any loss of precision of softmax_j[b, y_b] then moves the ratio by
# less than 1e-18.
_LOG_P_DIRECT_MIN = -60.0


def train_fold_groups(net, x_shape, n_local: int, stride: int, first_image: int = 0, fold_group: Optional[int] = None,
                      budget: int = LAYER_FOLD_BUDGET):
    """How MCTrainStep(fold=True) groups a rank's ``n_local`` samples on a row block of ``x_shape`` (rows, C, H, W):
    layer_fold_groups, or None for the sample loop.  None unless every Bayesian layer is LRT and every child treats
    each image on its own.  G is the largest group size -- up to the budget's or ``fold_group``, the int32 element cap and
    n_local -- at which the engine accepts every layer's folded forward (bbb_forward_supported) and every contraction of
    its backward (Fn.tc_backward_refusal; e.g. a linear layer's weight gradient takes at most so many rows).  A math mode
    without tensor cores folds neither.  Unlike MCForward's per-layer fold this does not defer to the fused chain, which
    never runs under autograd.  Host-only: no GPU work."""
    from .modules import ModuleWrapper
    kids = list(net.children())
    if not kids or type(net).forward is not ModuleWrapper.forward:
        return None
    chain = _per_image_chain(kids, tuple(x_shape))
    if chain is None:
        return None
    layers, pass_bytes, big = chain
    if not layers or any(m._variant != L.VARIANT_LRT for m, _ in layers):
        return None
    fold = (int(x_shape[0]), int(stride))
    groups = layer_fold_groups(n_local, pass_bytes, big, budget, fold_group)
    while groups is not None and not all(_train_fold_accepted(layers, n, fold, first_image) for n in {n for _, n in groups}):
        groups = layer_fold_groups(n_local, pass_bytes, big, fold_group=max(n for _, n in groups) - 1)
    return groups


def _fold_forward_supported(m, xs, n, fold, first_image):
    """Does the engine take Bayesian layer m's forward of n samples folded into the batch, one sample's input of shape
    ``xs`` (bbb_forward_supported)?"""
    cfg = m._cfg(True)
    d = Fn.make_desc((n * xs[0],) + tuple(xs[1:]), tuple(m.W_mu.shape), cfg["conv"], cfg["variant"], True,
                     m.bias_mu is not None, cfg["prior_mu"], cfg["prior_sigma"], cfg["math"], cfg["kl_convention"],
                     cfg["act"], fold=fold, first_image=first_image)
    return L.lib().bbb_forward_supported(C.byref(d)) == 0


def _train_fold_accepted(layers, n, fold, first_image):
    """Does the engine take a training pass of n folded samples: every layer's forward and backward?"""
    for i, (m, xs) in enumerate(layers):
        if not _fold_forward_supported(m, xs, n, fold, first_image):
            return False
        # the first layer's input is data (no input gradient); a later layer's input comes out of a layer
        if Fn._fold_grad_refusal(m._cfg(True), (n * xs[0],) + tuple(xs[1:]), tuple(m.W_mu.shape), i > 0) is not None:
            return False
    return True


def train_fold_kl_weights(groups, beta: float, num_ens: int):
    """The gradient each group's KL term gets in a folded training step: every sample has the same KL, which a folded
    pass computes once, so a group of n samples carries n * beta / S (the sample loop gives each sample beta / S)."""
    return [n * float(beta) / float(num_ens) for _, n in groups]


class MCTrainStep(MCForward):
    """One SHARDED training step with main_bayesian.train_model's semantics (main_bayesian.py:38-58): every rank runs
    its share of the ``num_ens`` weight samples WITH autograd (layer forward kernels + the engine's backward kernels),
    the exchange kernel combines them into log_outputs / kl / the ELBO (metrics.py:12-14) on every rank, each rank
    back-propagates d loss / d logits_j of ITS samples -- which needs only the combined log_outputs:
        d loss / d logits_j[b,:] = -(train_size / B) * softmax_j[b,y_b] / (S * p_bar[b,y_b]) * (onehot(y_b) - softmax_j[b,:])
    -- plus beta/S of its samples' KL terms, and ONE all-reduce sums the parameter gradients (SURVEY.md 8e "Backward
    sharding").  The caller owns the optimizer: ``out = step(x, labels, beta); optimizer.step()``.

    Noise: sample j of step t draws Philox streams 2^63 + (j << 40) + t * 2^20 + layer, so R ranks == 1 rank.

    ``batch_shards=Rb`` (MCForward): rank (g, k) back-propagates its samples on its row block only -- d loss / d logits
    keeps the global B (train_size / B) and uses the combined log_outputs rows of the block, the beta/S KL gradient is
    added by the block-0 rank of each group -- and the same all-reduce sums the gradients.  With num_ens = 1 (the
    reference's default) and Rb = world this is a data-parallel step.

    ``fold=True`` folds the local samples into grouped passes, forward and backward: groups of G consecutive local
    samples (layer_fold_groups; ``fold_group`` caps G) each run ONE forward and ONE backward of the per-layer
    tensor-core kernels over G x rows images (Fn.layer_fold(grad=True)) instead of G of each.  It folds when every
    Bayesian layer is LRT, the math mode is a tensor-core one, every child treats each image on its own, and the engine
    accepts every layer's folded forward and every contraction of its backward at the group's row count; otherwise the
    step runs the sample loop.  ``layer_fold`` = (G, number of groups), or None for the sample loop.  The per-sample
    logits, log_outputs, kl and head are bitwise those of the sample loop; the gradients differ only in the order their
    sums are taken.  The input x gets no gradient in a folded step (a pass reads x repeated G times, a copy).  Memory: the budget (LAYER_FOLD_BUDGET) bounds the activations of one pass, not the step's -- the
    loss gradient needs p_bar, which depends on every sample, so the autograd graph of every group lives until the
    exchange, and the step holds as much as the sample loop does."""

    def __init__(self, net, example_x, num_ens, train_size, group=None, seed=None, batch_shards: int = 1,
                 fold: bool = False, fold_group: Optional[int] = None, score_log=None, prob_bank=None, conformal=None,
                 logit_bank=None, temperature=None, scaling=None):
        for given, why in ((temperature, "temper: a temperature is fitted after training (fit_temperature) and "
                                         "applied by MCForward or evaluate()"),
                           (scaling, "scale logits: a scaling is fitted after training (fit_scaling) and applied by "
                                     "MCForward or evaluate()"),
                           (logit_bank, "fill a logit_bank: fill it from MCForward or evaluate()"),
                           (conformal, "log conformal scores: log them from MCForward or evaluate()"),
                           (score_log, "log scores: log them from MCForward or evaluate()"),
                           (prob_bank, "fill a prob_bank: fill it from MCForward or evaluate()")):
            if given is not None:
                raise L.EngineError(f"MCTrainStep does not {why}")
        super().__init__(net, example_x, num_ens, group=group, with_labels=True, train_size=train_size, seed=seed,
                         graph=False, fold=False, batch_shards=batch_shards)
        self.params = [p for p in net.parameters() if p.requires_grad]
        self.steps = 0
        if fold and len(self.ids) > 1:
            self._set_passes(train_fold_groups(net, (self.nb,) + tuple(example_x.shape[1:]), len(self.ids),
                                               self.sample_shards << 40, self.rows[0], fold_group), example_x)

    def __call__(self, x, labels, beta: float = 0.0):
        from .graph import _STRIDE
        from .modules import has_mixture
        self.beta = float(beta)
        self.labels.copy_(labels, non_blocking=True)
        for p in self.params:
            p.grad = None
        logits, kls = [], []
        b0, b1 = self.rows
        # logits[i] holds the n samples of pass i, one nb-row block each; autograd on: per-layer kernels (no fused chain)
        for s0, n, xin, fold_ctx in self._pass_inputs(x[b0:b1], grad=True):
            with Fn.mc_sample(self.ids[s0], self.seed, offset=self.steps * _STRIDE), Fn.first_image(b0), fold_ctx:
                lg, kl = self.net(xin)
            logits.append(lg)
            kls.append(kl)
            self.logits[s0:s0 + n].view(n * self.nb, self.C).copy_(lg.detach().reshape(n * self.nb, self.C))
        mixture = has_mixture(self.net)        # per-sample KL estimates: kls[i] is [n] for a folded group of n samples
        self._exchange(*(self._kl_arg(kls) if kls else (None, 0)))
        o = self.out
        if self.ids:
            S = float(self.num_ens)
            idx = self.labels[b0:b1].view(-1, 1)
            log_p_bar_y = o["log_outputs"][b0:b1].gather(1, idx)            # log p_bar[b, y_b] of the block's rows
            p_bar_y = log_p_bar_y.exp()
            # softmax_j[b,y_b] / (S p_bar[b,y_b]) is a ratio in [0, 1], but both factors underflow fp32 (0 / 0 = NaN) once
            # the label's log-probability falls below about -100.  Rows with log p_bar below _LOG_P_DIRECT_MIN take the
            # ratio in log space; the others keep the direct quotient, exact to fp32 rounding there.
            in_range = log_p_bar_y > _LOG_P_DIRECT_MIN
            grads = []
            for lg_all in logits:
                lg_dtype, lg_all = lg_all.dtype, lg_all.detach().float()
                blocks = []
                for r0 in range(0, lg_all.shape[0], self.nb):              # one sample per block of nb rows
                    lg = lg_all[r0:r0 + self.nb]
                    sm = torch.softmax(lg, dim=1)
                    w = torch.where(in_range, sm.gather(1, idx) / (S * p_bar_y),
                                    (torch.log_softmax(lg, dim=1).gather(1, idx) - log_p_bar_y - math.log(S)).exp())
                    onehot = torch.zeros_like(sm).scatter_(1, idx, 1.0)
                    blocks.append((-(self.train_size / self.B)) * w * (onehot - sm))
                # bf16 logits (bf16 activations) take their gradient in bf16, as autograd would cast it
                grads.append((blocks[0] if len(blocks) == 1 else torch.cat(blocks)).to(lg_dtype))
            # the KL does not depend on the rows: one block per sample group adds its gradient, n * beta / S for a
            # folded group of n samples (with mixture-prior layers its KL is the n samples' estimates: beta / S each)
            wkl = train_fold_kl_weights(self._groups, self.beta, self.num_ens) \
                if self._groups is not None and not mixture else [self.beta / S] * len(kls)
            kl_t = [(k_, w_) for k_, w_ in zip(kls, wkl) if torch.is_tensor(k_) and k_.requires_grad] \
                if self.block == 0 else []
            kl_g = [torch.full_like(k_, w_) for k_, w_ in kl_t]
            kl_t = [k_ for k_, _ in kl_t]
            torch.autograd.backward(logits + kl_t, grads + kl_g)
        if self.world > 1:                                                  # ONE collective: the summed parameter gradients
            for p in self.params:
                if p.grad is None:
                    p.grad = torch.zeros_like(p)
            flat = torch.cat([p.grad.reshape(-1) for p in self.params])
            self.dist.all_reduce(flat, group=self.group)
            off = 0
            for p in self.params:
                n = p.numel()
                p.grad.copy_(flat[off:off + n].view_as(p))
                off += n
        self.steps += 1
        return o


# --------------------------------------------------------------------------------------------------------------------
# Ranking metrics over a score log: out-of-distribution detection and selective prediction.  Larger score = more likely
# out-of-distribution / wrong.  They run once per data set, in float64 torch ops on the scores' device.
# --------------------------------------------------------------------------------------------------------------------
OOD_SCORES = ("confidence", "entropy", "mutual_info", "expected_entropy", "epistemic")
SELECTIVE_COVERAGES = (0.5, 0.8, 0.9, 0.95, 0.99)


def _scores64(s, what):
    s = torch.as_tensor(s).detach().reshape(-1).to(torch.float64)
    if s.numel() == 0:
        raise ValueError(f"{what}: empty score set")
    if bool(torch.isnan(s).any()):
        raise ValueError(f"{what}: NaN score")
    return s


def _auroc(neg, pos):
    """P(pos > neg) + 1/2 P(pos = neg) over all pairs, from the midranks of the pooled scores (Mann-Whitney U)."""
    v, order = torch.sort(torch.cat([neg, pos]))
    _, inv, counts = torch.unique_consecutive(v, return_inverse=True, return_counts=True)
    ends = counts.cumsum(0).to(torch.float64)
    mid = ends - (counts.to(torch.float64) - 1.0) / 2.0          # mean of the 1-based ranks end - count + 1 .. end
    n_neg, n_pos = neg.numel(), pos.numel()
    r_pos = mid[inv][order >= n_neg].sum()
    return float((r_pos - n_pos * (n_pos + 1) / 2.0) / (float(n_pos) * float(n_neg)))


def _flagged(s, pos):
    """At the distinct thresholds t_1 > t_2 > ... of s, flagging s >= t_k: (positives flagged, negatives flagged)."""
    v, order = torch.sort(s, descending=True)
    _, counts = torch.unique_consecutive(v, return_counts=True)
    ends = counts.cumsum(0) - 1
    p = pos[order].to(torch.float64)
    return p.cumsum(0)[ends], (1.0 - p).cumsum(0)[ends]


def _average_precision(s, pos):
    """sum_k (R_k - R_{k-1}) P_k over the distinct thresholds, R_0 = 0 (sklearn's average_precision_score)."""
    tp, fp = _flagged(s, pos)
    recall = tp / tp[-1]
    return float((torch.diff(recall, prepend=recall.new_zeros(1)) * (tp / (tp + fp))).sum())


def ood_metrics(s_in, s_out) -> dict:
    """Out-of-distribution detection from the scores of an in-distribution set ``s_in`` and an OOD set ``s_out``
    (larger = more likely OOD; OOD is the positive class): ``auroc``, ``aupr_out`` (average precision, OOD positive),
    ``aupr_in`` (the in-distribution set positive, scores negated) and ``fpr_at_95_tpr`` (the least false-positive
    rate over thresholds whose true-positive rate is >= 0.95).  NaN scores or an empty set raise ValueError."""
    s_in, s_out = _scores64(s_in, "ood_metrics: s_in"), _scores64(s_out, "ood_metrics: s_out")
    s_out = s_out.to(s_in.device)
    s = torch.cat([s_in, s_out])
    out = torch.cat([torch.zeros_like(s_in, dtype=torch.bool), torch.ones_like(s_out, dtype=torch.bool)])
    tp, fp = _flagged(s, out)
    tpr, fpr = tp / s_out.numel(), fp / s_in.numel()
    return {"auroc": _auroc(s_in, s_out), "aupr_out": _average_precision(s, out),
            "aupr_in": _average_precision(-s, ~out), "fpr_at_95_tpr": float(fpr[tpr >= 0.95].min()),
            "n_in": s_in.numel(), "n_out": s_out.numel()}


def selective_metrics(score, correct) -> dict:
    """Selective prediction (Geifman et al. 2019) and misclassification detection (Hendrycks & Gimpel 2017) from a
    per-image ``score`` (larger = more likely wrong) and ``correct`` (1 / 0).

    ``coverage`` / ``risk``: the risk-coverage curve at the distinct thresholds in ascending order, accepting score <= t
    (float64 tensors); ``aurc`` = sum_k (cov_k - cov_{k-1}) risk_k; ``eaurc`` = aurc minus the AURC of the ideal order
    (every correct image first, no ties: (1/n) sum_{k=1..n} max(0, k - n_correct) / k); ``auroc`` with the wrong
    predictions positive (NaN when all or none are correct); ``accuracy``; ``accuracy_at`` {c: accuracy of the
    ceil(c * n) lowest scores (ties by index)} for c in SELECTIVE_COVERAGES.  NaN or an empty set raise ValueError."""
    from fractions import Fraction
    s = _scores64(score, "selective_metrics: score")
    ok = _scores64(correct, "selective_metrics: correct").to(s.device)
    if ok.numel() != s.numel():
        raise ValueError(f"selective_metrics: {s.numel()} scores but {ok.numel()} correct flags")
    if not bool(((ok == 0) | (ok == 1)).all()):
        raise ValueError("selective_metrics: correct must be 0 or 1")
    n = s.numel()
    v, order = torch.sort(s, stable=True)
    _, counts = torch.unique_consecutive(v, return_counts=True)
    ends = counts.cumsum(0) - 1
    wrong = (1.0 - ok[order]).cumsum(0)[ends]
    accepted = (ends + 1).to(torch.float64)
    cov, risk = accepted / n, wrong / accepted
    aurc = float((torch.diff(cov, prepend=cov.new_zeros(1)) * risk).sum())
    n_ok = int(ok.sum())
    k = torch.arange(1, n + 1, dtype=torch.float64, device=s.device)
    ideal = float(((k - n_ok).clamp_min(0.0) / k).sum() / n)
    bad = ok == 0
    auroc = _auroc(s[~bad], s[bad]) if 0 < n_ok < n else float("nan")
    at = {}
    for c in SELECTIVE_COVERAGES:
        m = max(1, math.ceil(Fraction(repr(c)) * n))
        at[c] = float(ok[order[:m]].mean())
    return {"coverage": cov, "risk": risk, "aurc": aurc, "eaurc": aurc - ideal, "auroc": auroc,
            "accuracy": n_ok / n, "accuracy_at": at, "n": n}


def _score(log: dict, name: str):
    """The score ``name`` of a ScoreLog.read() dict, larger = more likely OOD / wrong: -confidence (not 1 - conf,
    which loses the bits near 1), the others as logged."""
    if name not in OOD_SCORES:
        raise ValueError(f"unknown score {name!r}: one of {OOD_SCORES}")
    return -log["confidence"] if name == "confidence" else log[name]


def _loader_images(loader):
    """Images a loader yields: len(loader.dataset), else the batches of a sized sequence counted."""
    ds = getattr(loader, "dataset", None)
    if ds is not None:
        return len(ds)
    if hasattr(loader, "__len__") and hasattr(loader, "__getitem__"):
        return sum(int(b[0].shape[0]) for b in loader)
    raise ValueError("detect_ood: a loader without .dataset must be a sequence of (x, y) batches")


def detect_ood(net, in_loader, out_loader, num_ens: int, score: Optional[str] = "mutual_info", normalized: bool = False,
               **evaluate_kwargs) -> dict:
    """Out-of-distribution detection over whole data sets (uncertainty_estimation.py's MNIST vs notMNIST comparison):
    ``evaluate`` over ``in_loader`` and ``out_loader`` (batches of (x, y); the OOD set's labels are not used), each
    into a ScoreLog, and the ranking metrics of their scores.

    Returns ``in`` (evaluate's dict on the in-distribution set), ``ood`` (ood_metrics of ``score``, or {name:
    ood_metrics} for every name of OOD_SCORES with ``score=None``), ``selective`` (selective_metrics on the
    in-distribution set, per score in the same way) and ``logs`` ({"in": ..., "out": ...}, ScoreLog.read() dicts).
    ``evaluate_kwargs`` go to evaluate (``train_size`` defaults to 1.0).  The two logs are kept on the net, as evaluate
    keeps its engines, and reused by the next call."""
    names = OOD_SCORES if score is None else (score,)
    if any(nm not in OOD_SCORES for nm in names):
        raise ValueError(f"detect_ood: unknown score {score!r}: one of {OOD_SCORES}, or None for all")
    dev = next(net.parameters()).device
    kw = dict(evaluate_kwargs)
    train_size = kw.pop("train_size", 1.0)
    logs, res = net.__dict__.setdefault("_ood_logs", {}), {}
    for role, loader in (("in", in_loader), ("out", out_loader)):
        log = _kept_log(net, logs, role, loader, lambda n: ScoreLog(dev, n))
        res[role] = evaluate(net, loader, num_ens, train_size, normalized=normalized, score_log=log, **kw)
    got = {role: logs[role].read() for role in ("in", "out")}
    ood = {nm: ood_metrics(_score(got["in"], nm), _score(got["out"], nm)) for nm in names}
    sel = {nm: selective_metrics(_score(got["in"], nm), got["in"]["correct"]) for nm in names}
    return {"in": res["in"], "ood": ood if score is None else ood[score],
            "selective": sel if score is None else sel[score], "logs": got}


# --------------------------------------------------------------------------------------------------------------------
# Active learning: a pool-long bank of every sample's probabilities, and BALD / BatchBALD (Kirsch et al. 2019)
# selection on the device.
# --------------------------------------------------------------------------------------------------------------------
def bank_pads(num_ens: int, num_classes: int):
    """(S_pad, C_pad) of a probability bank: S rounded up to 8 (the tf32 wgmma K step), C to the next power of two."""
    return -(-int(num_ens) // 8) * 8, 1 << (int(num_classes) - 1).bit_length()


class _SampleBank(_CursorLog):
    """What ProbBank and LogitBank share: entries of all S samples x C classes of an image, taken from the step's
    per-sample logits.  A rank of a sharded step holds only its own samples, so a bank binds to a step on several ranks
    only when it was made with that step's ``group``: the step then gathers every rank's logits onto every rank
    (bbb_mc_logit_gather), and each rank's bank holds all of them.  The group also carries the bank's collectives
    (batchbald's seed)."""

    def _init_bank(self, device, capacity, num_ens, num_classes, group):
        self._init_cursor(device, capacity, type(self).__name__)
        self.num_ens, self.num_classes, self.group = num_ens, num_classes, group

    def _bind(self, step):
        if step.world > 1:
            dist, n, _ = _dist_info(self.group) if self.group is not None else (None, 1, 0)
            if n == 1:
                raise L.EngineError(f"MCForward: a {self._keyword} needs one rank (the group has {step.world}): a rank "
                                    "holds only its own samples")
            world = dist.group.WORLD if dist is not None else None      # the step's group=None
            if self.group is not (step.group if step.group is not None else world):
                raise L.EngineError(f"MCForward: the {self._keyword} was made with another group than the step's: every "
                                    "step that fills a bank must run over the bank's ranks")
        super()._bind(step)
        self._require(step.num_ens, step.C, "MCForward")

    def _empty(self):
        return type(self)(self.device, 0, self.num_ens, self.num_classes, group=self.group)

    def _require(self, num_ens, num_classes, what):
        if (int(num_ens), int(num_classes)) != (self.num_ens, self.num_classes):
            raise L.EngineError(f"{what}: the {self._keyword} holds {self.num_ens} samples x {self.num_classes} "
                                f"classes, the step makes {num_ens} x {num_classes}")

    def _check_logits(self, logits):
        """Refuse anything but per-sample logits [S, B, C] of this bank: fp32, contiguous, on its device."""
        what = f"{type(self).__name__}.append"
        Fn._require_cuda(self._cursor, what)
        B = max(1, logits.shape[1]) if logits.dim() == 3 else 1        # an empty batch is refused
        _check_tensor(logits, f"{what}: expected contiguous float32 logits [S, B, C]",
                      (self.num_ens, B, self.num_classes), torch.float32, self.device)


class ProbBank(_SampleBank):
    """A device-resident bank of every Monte-Carlo sample's probability row for each image of a pool, appended to by the
    step (bbb_mc_prob_log): ``MCForward(..., prob_bank=bank)`` and ``evaluate(..., prob_bank=bank)`` add one entry per
    image, in step order, with no host read.  It is what BatchBALD scores (``batchbald``, ``bald``, ``acquire``).

    Entry i holds the S rows p_hat_s (the exchange's softmax, or softplus-normalised row with ``normalized``), rounded to
    tf32, in ``bank[i][c][s]`` order with S padded to S_pad and C to C_pad (bank_pads; the padding is zero), and
    ``expected_entropy`` = (1/S) sum_s H[p_hat_s] in float64.  ``capacity`` entries fit; images past them are counted,
    not written, and ``read()`` refuses a bank that dropped any.

    ``group``: the torch.distributed group of the steps that fill it (None: one rank).  Every rank then receives every
    step's full [S, B, C] logits and holds the whole bank, with the one-rank bank's bits."""

    _keyword = "prob_bank"

    def __init__(self, device, capacity: int, num_ens: int, num_classes: int, group=None):
        num_ens, num_classes = int(num_ens), int(num_classes)
        if not 1 <= num_ens <= L.BANK_MAX_SAMPLES:
            raise ValueError(f"ProbBank: num_ens must be in [1, {L.BANK_MAX_SAMPLES}] (got {num_ens})")
        if not 2 <= num_classes <= L.BANK_MAX_CLASSES:
            raise ValueError(f"ProbBank: num_classes must be in [2, {L.BANK_MAX_CLASSES}] (got {num_classes})")
        self._init_bank(device, capacity, num_ens, num_classes, group)
        self.S_pad, self.C_pad = bank_pads(num_ens, num_classes)
        # (one entry at least: the kernel takes the bank's pointers even when nothing fits)
        self._probs = torch.zeros(max(1, self.capacity), self.C_pad, self.S_pad, dtype=torch.float32, device=self.device)
        self._ee = torch.zeros(max(1, self.capacity), dtype=torch.float64, device=self.device)

    def _launch(self, logits, B, normalized):
        L.check(L.lib().bbb_mc_prob_log(Fn._ptr(logits), self.num_ens, int(B), self.num_classes, int(bool(normalized)),
                                        Fn._ptr(self._probs), Fn._ptr(self._ee), self.capacity, Fn._ptr(self._cursor),
                                        Fn._stream(self.device)), "bbb_mc_prob_log")

    def _log(self, step, par):
        self._launch(step._bank_logits(par, mapped=True), step.B, bool(step.flags & L.MC_NORMALIZED))

    def append(self, logits, normalized: bool = False):
        """Append the images of per-sample logits [S, B, C] (fp32 contiguous on the bank's device; bbb_mc_prob_log on
        the current stream): probabilities from anywhere else."""
        self._check_logits(logits)
        self._launch(logits, logits.shape[1], normalized)

    def read(self) -> dict:
        """The entries so far: {"probs": float32 [n, S, C], "expected_entropy": float64 [n]}, copies on the bank's
        device.  Raises EngineError if images were dropped.  Steps in flight must be complete first."""
        n = self._held("ProbBank")
        return {"probs": self._probs[:n, :self.num_classes, :self.num_ens].transpose(1, 2).contiguous(),
                "expected_entropy": self._ee[:n].clone()}


def batchbald_plan(num_classes: int, k: int, num_configs: int):
    """(M, exact) of each of the k greedy rounds: round n (n labels chosen) enumerates the C^n configurations of their
    labels while C^n <= num_configs, and draws num_configs of them after that."""
    out = []
    for n in range(int(k)):
        exact = int(num_classes) ** n <= int(num_configs)
        out.append((int(num_classes) ** n if exact else int(num_configs), exact))
    return out


def _tf32(x64):
    """float64 -> the nearest tf32 value (ties away from zero, as cvt.rna) in float32 words; x >= 0 and finite."""
    b = x64.to(torch.float32).view(torch.int32)
    return ((b + 0x1000) & ~0x1FFF).view(torch.float32)


def _draw(w, gen, n=None):
    """Inverse-CDF draws from non-negative weights: one index per row of w [R, K] ([R] int64), or with w [K] n indices
    of the one distribution ([n] int64; one cumulative sum of K words, whatever n is)."""
    cdf = w.cumsum(-1)
    shape = (w.shape[0], 1) if w.dim() == 2 else (n,)
    u = torch.rand(shape, dtype=torch.float64, device=w.device, generator=gen) * cdf[..., -1:]
    idx = torch.searchsorted(cdf, u, right=True).clamp_(max=w.shape[-1] - 1)
    return idx[:, 0] if w.dim() == 2 else idx


def _check_selection(bank, k, num_configs=1):
    n = bank._held("batch selection")
    if not 1 <= int(k) <= n:
        raise ValueError(f"select {k} of a pool of {n}: k must be in [1, {n}]")
    if not 1 <= int(num_configs) <= 1 << 20:
        raise ValueError(f"num_configs must be in [1, 2^20] (got {num_configs})")
    Fn._require_cuda(bank._cursor, "batch selection")
    return n


class _Scorer:
    """bbb_joint_entropy over the first n entries of a bank, with the Pt / omega / mask / output buffers of the rounds."""

    def __init__(self, bank, n, m_max):
        dev = bank.device
        self.bank, self.n = bank, n
        self.pt = torch.zeros(-(-m_max // 64) * 64, bank.S_pad, dtype=torch.float32, device=dev)
        self.omega = torch.zeros(m_max, dtype=torch.float64, device=dev)
        self.mask = torch.zeros(n, dtype=torch.uint8, device=dev)
        self.out = torch.empty(n, dtype=torch.float64, device=dev)

    def __call__(self, pt64, omega64):
        """out[i] for the configurations pt64 [M, S] (normalised columns) and omega64 [M], both float64."""
        b, M = self.bank, pt64.shape[0]
        self.pt[:M, :b.num_ens].copy_(_tf32(pt64))
        self.pt[M:].zero_()
        self.omega[:M].copy_(omega64)
        L.check(L.lib().bbb_joint_entropy(Fn._ptr(self.pt), Fn._ptr(self.omega), Fn._ptr(self.mask), Fn._ptr(b._probs),
                                          self.n, b.num_ens, b.num_classes, M, Fn._ptr(self.out), None, 0,
                                          Fn._stream(b.device)), "bbb_joint_entropy")
        return self.out


def bald(bank: ProbBank, k: int) -> dict:
    """BALD top-k: the k candidates of largest mutual information, scored by round 0 of ``batchbald`` (the same kernel).
    Returns ``indices`` (int64 [k], by decreasing score) and ``scores`` (float64 [k]) on the host."""
    n = _check_selection(bank, k)
    S = bank.num_ens
    f64 = dict(dtype=torch.float64, device=bank.device)
    mi = _Scorer(bank, n, 1)(torch.full((1, S), 1.0 / S, **f64), torch.ones(1, **f64)) - bank._ee[:n]
    s, i = torch.topk(mi, int(k))
    return {"indices": i.cpu(), "scores": s.cpu()}


def batchbald(bank: ProbBank, k: int, num_configs: int = 10000, seed: Optional[int] = None, trace: bool = False) -> dict:
    """Greedy BatchBALD (Kirsch et al. 2019) over the entries of ``bank``: round n picks the candidate i of largest
        a(A u {i}) = H(y_A, y_i) - sum_{j in A} E_s H[p_hat_s(y_j)] - E_s H[p_hat_s(y_i)],
    with H(y_A, y_i) = sum_m omega_m h_m(i) + const from bbb_joint_entropy over configurations m of the labels y_A:
    enumerated while C^n <= num_configs (omega_m = P(y_A = m), const = -sum omega log omega), else num_configs of them
    drawn -- the first time from the exact joint, then extended ancestrally, y_a(m) ~ Q_a[m, .] -- with omega = 1/M
    and const = -(1/M) sum_m log P(y_A(m)).  Pt's column m is P(s | y_A = m); the update between rounds runs in float64
    torch ops on the device and the k rounds are enqueued with no host read; ``seed`` seeds the draws (same seed, same
    bits).  ``seed=None`` draws one; on a bank made with a group of several ranks, rank 0's draw, so that every rank
    selects the same images.

    Returns ``indices`` (int64 [k]) and ``scores`` (float64 [k], a(A) after each pick) on the host, and ``exact`` (per
    round: enumerated?).  ``trace=True`` adds ``trace``: per round a dict of the device tensors ``scores`` (every
    candidate; chosen ones -inf), ``pt`` (the tf32 Pt the kernel read, [M, S]), ``omega``, ``const`` and ``configs`` (the
    label configurations [M, n])."""
    n = _check_selection(bank, k, num_configs)
    picks, scores, plan, rounds = _batchbald_rounds(bank, n, int(k), int(num_configs), seed, trace)
    res = {"indices": picks.cpu(), "scores": scores.cpu(), "exact": [e for _, e in plan]}
    if trace:
        res["trace"] = rounds
    return res


def _selection_seed(bank, seed):
    """The seed of batchbald's draws: ``seed``, or a fresh draw -- rank 0's on a bank made with a group, so that every
    rank of it selects the same images."""
    if seed is not None:
        return int(seed)
    seed = int(torch.randint(1 << 62, (1,)).item())
    return int(_from_rank0(seed, bank.group)) if bank.group is not None else seed


def _batchbald_rounds(bank, n, k, num_configs, seed, trace):
    """The k rounds of batchbald over the first n entries, enqueued on the current stream with no host read: (picks,
    scores) as device tensors, the plan and the trace."""
    dev, S, Cc = bank.device, bank.num_ens, bank.num_classes
    plan = batchbald_plan(Cc, k, num_configs)
    score = _Scorer(bank, n, max(M for M, _ in plan))
    f64 = dict(dtype=torch.float64, device=dev)
    gen = torch.Generator(device=dev)
    gen.manual_seed(_selection_seed(bank, seed))
    eh = bank._ee[:n]
    pt, omega, const = torch.full((1, S), 1.0 / S, **f64), torch.ones(1, **f64), torch.zeros((), **f64)
    configs = torch.zeros(1, 0, dtype=torch.int64, device=dev)
    log_p = None
    eh_sum = torch.zeros((), **f64)
    picks = torch.zeros(k, dtype=torch.int64, device=dev)
    scores = torch.zeros(k, **f64)
    rounds, p_a = [], None
    for r, (M, exact) in enumerate(plan):
        if r > 0:
            q_a = pt @ p_a.T                                         # [M_prev, C]: P(y_a = c | y_A = m)
            M_prev = pt.shape[0]
            if exact:
                col = (pt[:, None, :] * p_a[None, :, :]).reshape(M_prev * Cc, S)
                q = q_a.reshape(-1, 1)
                pt = torch.where(q > 0, col / torch.where(q > 0, q, 1.0), 0.0)
                omega = (omega[:, None] * q_a).reshape(-1)
                const = -torch.special.xlogy(omega, omega).sum()
                configs = torch.cat([configs.repeat_interleave(Cc, 0),
                                     torch.arange(Cc, device=dev).repeat(M_prev)[:, None]], 1)
            else:
                if log_p is None:                                     # first sampled round: from the exact joint
                    joint = (omega[:, None] * q_a).reshape(-1)       # [M_prev * C]
                    idx = _draw(joint, gen, M)
                    m_i, c_i = idx // Cc, idx % Cc
                    log_p = torch.log(joint.gather(0, idx))
                else:                                                 # ancestral: y_a(m) ~ Q_a[m, .]
                    m_i, c_i = torch.arange(M, device=dev), _draw(q_a, gen)
                    log_p = log_p + torch.log(q_a.gather(1, c_i[:, None])[:, 0])
                q = q_a[m_i].gather(1, c_i[:, None])
                pt = pt[m_i] * p_a.index_select(0, c_i) / q
                configs = torch.cat([configs[m_i], c_i[:, None]], 1)
                omega = torch.full((M,), 1.0 / M, **f64)
                const = -log_p.sum() / M
        out = score(pt, omega)
        a = out + const - eh_sum - eh
        pick = torch.argmax(a).view(1)
        picks[r:r + 1].copy_(pick)
        scores[r:r + 1].copy_(a.index_select(0, pick))
        score.mask.index_fill_(0, pick, 1)
        eh_sum = eh_sum + eh.index_select(0, pick)[0]
        p_a = bank._probs.index_select(0, pick)[0, :Cc, :S].to(torch.float64)       # the stored (tf32) rows
        if trace:
            rounds.append({"scores": a.clone(), "pt": score.pt[:M, :S].clone(), "omega": omega.clone(),
                           "const": const.clone(), "configs": configs.clone(), "exact": exact, "M": M})
    return picks, scores, plan, rounds


def acquire(net, pool_loader, k: int, num_ens: int, method: str = "batchbald", num_configs: int = 10000,
            **evaluate_kwargs) -> dict:
    """One active-learning acquisition (Gal et al. 2017, Kirsch et al. 2019): ``evaluate`` over ``pool_loader``
    (batches of (x, y); the labels are not used) into a ProbBank sized from the loader, then ``batchbald`` or ``bald``
    selects k pool images.  Returns the selection's dict (``indices`` are positions in loader order) plus
    ``evaluate`` (evaluate's figures).  ``evaluate_kwargs`` go to evaluate (``train_size`` defaults to 1.0); its
    ``seed`` also seeds the sampled configurations.  The bank is kept on the net, as detect_ood keeps its logs; it is
    made with evaluate's ``group``, so on several ranks every rank holds the whole pool's bank and selects the same
    images (with ``seed=None``, rank 0's draw)."""
    if method not in ("batchbald", "bald"):
        raise ValueError(f"acquire: method must be 'batchbald' or 'bald' (got {method!r})")
    dev = next(net.parameters()).device
    kw = dict(evaluate_kwargs)
    train_size = kw.pop("train_size", 1.0)
    group = kw.get("group")
    bank = _kept_log(net, net.__dict__, "_al_bank", pool_loader,
                     lambda n: ProbBank(dev, n, num_ens, net.num_classes, group=group),
                     lambda b: (b.num_ens, b.num_classes) == (int(num_ens), int(net.num_classes)) and b.group is group)
    m = evaluate(net, pool_loader, num_ens, train_size, prob_bank=bank, **kw)
    sel = batchbald(bank, k, num_configs, seed=kw.get("seed")) if method == "batchbald" else bald(bank, k)
    sel["evaluate"] = m
    return sel


# --------------------------------------------------------------------------------------------------------------------
# Split conformal prediction (Vovk et al. 2005): a coverage threshold calibrated on held-out labelled images, and
# prediction sets that hold the true label with probability >= 1 - alpha, on the device.
# --------------------------------------------------------------------------------------------------------------------
CONFORMAL_METHODS = {"lac": L.CONFORMAL_LAC, "aps": L.CONFORMAL_APS, "raps": L.CONFORMAL_RAPS}
SIZE_BINS = (("0", 0, 0), ("1", 1, 1), ("2-3", 2, 3), ("4-10", 4, 10), ("11+", 11, None))


class ConformalLog(_CursorLog):
    """A data-set-long log of conformity scores and prediction sets on the device, appended to by the Monte-Carlo step
    (bbb_mc_conformal_log): ``MCForward(..., conformal=log)`` and ``evaluate(..., conformal=log)`` add one entry per
    image, in step order, with no host read.

    Entry i holds ``score`` = E_y, the conformity score of the label (float64; NaN without a label), the prediction set
    {c : E_c <= q_hat_c} at the log's threshold (``sets``, ``size``), ``covered`` (y in the set: 1 / 0, -1 without a
    label) and ``label`` (-1 without one).  E_c is ``method``'s score: "lac" 1 - p_c, "aps" the probability mass of
    the classes ranked above c plus ``u`` p_c (``randomized``; p_c otherwise), "raps" the APS score plus ``lam`` *
    max(0, rank + 1 - ``k_reg``) (include/bbb_b200.h).  ``u`` is drawn from (``seed``, ``stream``, i): logs that must
    be independent (a calibration set and a test set) take different streams.  Until ``set_threshold`` the log has no
    threshold (size = covered = -1, empty sets): a calibration log needs none.  ``capacity`` entries fit; images past
    them are counted, not written, and ``read()`` refuses a log that dropped any."""

    _keyword = "conformal"

    def __init__(self, device, capacity: int, num_classes: int, method: str = "aps", randomized: bool = True,
                 lam: float = 0.0, k_reg: int = 0, seed: Optional[int] = None, stream: int = 0):
        num_classes, lam, k_reg = int(num_classes), float(lam), int(k_reg)
        if method not in CONFORMAL_METHODS:
            raise ValueError(f"ConformalLog: method must be one of {tuple(CONFORMAL_METHODS)} (got {method!r})")
        if not 2 <= num_classes <= L.CONFORMAL_MAX_CLASSES:
            raise ValueError(f"ConformalLog: num_classes must be in [2, {L.CONFORMAL_MAX_CLASSES}] (got {num_classes})")
        if not (math.isfinite(lam) and lam >= 0.0):
            raise ValueError(f"ConformalLog: lam must be finite and >= 0 (got {lam})")
        if k_reg < 0:
            raise ValueError(f"ConformalLog: k_reg must be >= 0 (got {k_reg})")
        if not 0 <= int(stream) < 1 << 64:
            raise ValueError(f"ConformalLog: stream must be in [0, 2^64) (got {stream})")
        self._init_cursor(device, capacity, "ConformalLog")
        self.num_classes, self.method, self.randomized, self.lam, self.k_reg = num_classes, method, bool(randomized), \
            lam, k_reg
        self.seed = int(Fn.current_seed() if seed is None else seed) & ((1 << 64) - 1)
        self.stream = int(stream)
        self.words = (num_classes + 31) // 32
        # (one entry at least: the kernel takes the log's pointers even when nothing fits)
        n = max(1, self.capacity)
        self._score = torch.full((n,), float("nan"), dtype=torch.float64, device=self.device)
        self._size, self._covered, self._label = (torch.zeros(n, dtype=torch.int32, device=self.device) for _ in range(3))
        self._sets = torch.zeros(n, self.words, dtype=torch.int32, device=self.device)      # uint32 words
        # the threshold, per class (a scalar is written to every class): NaN = none yet; read by the kernel at run time
        self._qhat = torch.full((num_classes,), float("nan"), dtype=torch.float64, device=self.device)
        self._threshold = None

    def _options(self):
        return dict(method=self.method, randomized=self.randomized, lam=self.lam, k_reg=self.k_reg, seed=self.seed,
                    stream=self.stream)

    def _empty(self):
        """A log of no capacity with the same options (what an engine's warm-up steps append to)."""
        return ConformalLog(self.device, 0, self.num_classes, **self._options())

    def _bind(self, step):
        super()._bind(step)
        if step.C != self.num_classes:
            raise L.EngineError(f"MCForward: the conformal log holds {self.num_classes} classes, the step makes "
                                f"{step.C}")

    def _log(self, step, par):
        self._launch(step.out["log_outputs"], step._labels_of(par))

    def _launch(self, log_outputs, labels):
        L.check(L.lib().bbb_mc_conformal_log(
            Fn._ptr(log_outputs), Fn._ptr(labels), int(log_outputs.shape[0]), self.num_classes,
            CONFORMAL_METHODS[self.method], int(self.randomized), C.c_double(self.lam), self.k_reg,
            C.c_uint64(self.seed), C.c_uint64(self.stream), Fn._ptr(self._qhat), 1, Fn._ptr(self._score),
            Fn._ptr(self._size), Fn._ptr(self._covered), Fn._ptr(self._label), Fn._ptr(self._sets), self.capacity,
            Fn._ptr(self._cursor), Fn._stream(self.device)), "bbb_mc_conformal_log")

    def append(self, log_outputs, labels=None):
        """Append one step's images (bbb_mc_conformal_log on the current stream): log p_bar [B, C] fp32 and optional
        int64 labels [B], contiguous on the log's device."""
        Fn._require_cuda(self._cursor, "ConformalLog.append")
        B = max(1, int(log_outputs.shape[0])) if log_outputs.dim() == 2 else 1     # an empty batch is refused
        for t, shape, dt in ((log_outputs, (B, self.num_classes), torch.float32), (labels, (B,), torch.int64)):
            if t is not None:
                _check_tensor(t, "ConformalLog.append", shape, dt, self.device)
        self._launch(log_outputs, labels)

    def read(self) -> dict:
        """The entries logged so far: {"score": float64 [n], "size", "covered", "label": int32 [n], "sets": bool
        [n, C]}, on the log's device.  Raises EngineError if images were dropped.  Steps in flight must be complete
        first (``MCForward.wait()``)."""
        n = self._held("ConformalLog")
        bit = torch.arange(32, dtype=torch.int32, device=self.device)
        sets = ((self._sets[:n, :, None] >> bit) & 1).reshape(n, self.words * 32)[:, :self.num_classes].bool()
        return {"score": self._score[:n].clone(), "size": self._size[:n].clone(), "covered": self._covered[:n].clone(),
                "label": self._label[:n].clone(), "sets": sets}

    def set_threshold(self, q):
        """Set q_hat, in place (stream-ordered on the current stream; engines captured with this log read it from the
        next step on): a scalar, or [num_classes] class-conditional thresholds (``calibrate(mondrian=True)``).  NaN
        clears it."""
        q = torch.as_tensor(q, dtype=torch.float64).detach().reshape(-1)
        if q.numel() not in (1, self.num_classes):
            raise ValueError(f"ConformalLog.set_threshold: one value or {self.num_classes} (got {q.numel()})")
        self._qhat.copy_(q.to(self.device).expand(self.num_classes))
        self._threshold = q.to(self.device).clone().reshape(() if q.numel() == 1 else (self.num_classes,))

    @property
    def threshold(self):
        """The threshold last set (float64 scalar or [num_classes] tensor on the log's device), or None."""
        return self._threshold

    def calibrate(self, alpha: float, mondrian: bool = False) -> torch.Tensor:
        """q_hat from the scores logged so far (conformal_quantile; every entry needs a label): one value, or with
        ``mondrian`` one per class from that class's images (class-conditional coverage).  The log is not changed."""
        r = self.read()
        if bool((r["label"] < 0).any()):
            raise ValueError("ConformalLog.calibrate: every calibration image needs a label")
        return conformal_quantile(r["score"], alpha, r["label"] if mondrian else None, num_classes=self.num_classes)


def _conformal_rank(n: int, alpha) -> int:
    """ceil((n + 1)(1 - alpha)), exactly (alpha as its shortest decimal)."""
    from fractions import Fraction
    a = Fraction(repr(float(alpha)))
    return -(-(n + 1) * (a.denominator - a.numerator) // a.denominator)


def conformal_quantile(scores, alpha: float, classes=None, num_classes: Optional[int] = None) -> torch.Tensor:
    """The split-conformal threshold: the ceil((n + 1)(1 - alpha))-th smallest of the n ``scores``, +inf when that rank
    exceeds n (too few calibration images for 1 - alpha).  Sets {c : E_c <= q_hat} then cover the label of a new
    exchangeable image with probability >= 1 - alpha.  With ``classes`` (one label per score) the rule is applied to
    each class's scores and the result is [num_classes] (default: the largest class + 1); a class without images gets
    +inf.  float64 on the scores' device.  NaN scores or alpha outside (0, 1) raise ValueError."""
    alpha = float(alpha)
    if not 0.0 < alpha < 1.0:
        raise ValueError(f"conformal_quantile: alpha must be in (0, 1) (got {alpha})")
    s = torch.as_tensor(scores).detach().reshape(-1).to(torch.float64)
    if bool(torch.isnan(s).any()):
        raise ValueError("conformal_quantile: NaN score (an image without a label?)")
    inf = float("inf")
    if classes is None:
        n, k = s.numel(), _conformal_rank(s.numel(), alpha)
        return torch.sort(s).values[k - 1] if k <= n else torch.tensor(inf, dtype=torch.float64, device=s.device)
    cls = torch.as_tensor(classes).detach().reshape(-1).to(device=s.device, dtype=torch.int64)
    if cls.numel() != s.numel():
        raise ValueError(f"conformal_quantile: {s.numel()} scores but {cls.numel()} classes")
    if num_classes is None:
        if cls.numel() == 0:
            raise ValueError("conformal_quantile: num_classes is needed without scores")
        num_classes = int(cls.max()) + 1
    if cls.numel() and (int(cls.min()) < 0 or int(cls.max()) >= num_classes):
        raise ValueError(f"conformal_quantile: classes must be in [0, {num_classes})")
    counts = torch.bincount(cls, minlength=num_classes)
    ks = torch.tensor([_conformal_rank(n, alpha) for n in counts.tolist()], dtype=torch.int64, device=s.device)
    q = torch.full((num_classes,), inf, dtype=torch.float64, device=s.device)
    if s.numel():
        o = torch.argsort(s, stable=True)
        ordered = s[o][torch.argsort(cls[o], stable=True)]         # by class, then by score
        starts = counts.cumsum(0) - counts
        ok = ks <= counts
        q = torch.where(ok, ordered[(starts + ks - 1).clamp(0, s.numel() - 1)], q)
    return q


def conformal_metrics(log_or_read) -> dict:
    """Figures of a thresholded ConformalLog (or its ``read()`` dict): ``coverage`` (the fraction of labelled images
    whose label is in the set), ``mean_size``, ``size_histogram`` (int64 [C + 1]: images per set size),
    ``empty_fraction``, ``class_coverage`` (float64 [C], NaN for a class without images), ``class_count``,
    ``min_class_coverage`` and ``size_stratified`` ({bin: {"count", "coverage"}} over set sizes 0, 1, 2-3, 4-10, 11+;
    coverage NaN for an empty bin).  Coverage figures are over the labelled images (NaN if there are none).  A log
    without a threshold raises ValueError."""
    r = log_or_read.read() if isinstance(log_or_read, ConformalLog) else log_or_read
    size, covered, label = r["size"].long(), r["covered"].long(), r["label"].long()
    n, ncls = size.numel(), int(r["sets"].shape[1])
    if n == 0:
        raise ValueError("conformal_metrics: no images")
    if bool((size < 0).any()):
        raise ValueError("conformal_metrics: the log had no threshold (set_threshold) when these images were logged")
    lab = covered >= 0
    cov = covered[lab].double()
    nan = float("nan")
    coverage = float(cov.mean()) if cov.numel() else nan
    count = torch.bincount(label[lab], minlength=ncls)
    hit = torch.bincount(label[lab], weights=cov, minlength=ncls)
    per = torch.where(count > 0, hit / count.clamp_min(1).double(), torch.full_like(hit, nan))
    strata = {}
    for name, lo, hi in SIZE_BINS:
        m = (size >= lo) & ((size <= hi) if hi is not None else True)
        ml = m & lab
        strata[name] = {"count": int(m.sum()),
                        "coverage": float(covered[ml].double().mean()) if bool(ml.any()) else nan}
    return {"n": n, "coverage": coverage, "mean_size": float(size.double().mean()),
            "size_histogram": torch.bincount(size, minlength=ncls + 1), "empty_fraction": float((size == 0).double().mean()),
            "class_coverage": per, "class_count": count,
            "min_class_coverage": float(per[count > 0].min()) if bool((count > 0).any()) else nan,
            "size_stratified": strata}


def conformal(net, cal_loader, test_loader, num_ens: int, alpha: float = 0.1, method: str = "aps",
              randomized: bool = True, lam: float = 0.0, k_reg: int = 0, mondrian: bool = False,
              **evaluate_kwargs) -> dict:
    """Split conformal prediction over whole data sets: ``evaluate`` over ``cal_loader`` (batches of (x, y)) into a
    ConformalLog, q_hat = its ``calibrate(alpha, mondrian)``, then ``evaluate`` over ``test_loader`` into a second log
    that holds q_hat, so every test image gets its prediction set on the device as its step runs.

    Returns ``qhat``, ``test`` (conformal_metrics of the test log, plus ``evaluate``: evaluate's figures on the test
    set), ``calibration`` ({"n", "alpha", "rank", "method", "mondrian"}; rank = ceil((n + 1)(1 - alpha))), ``in``
    (evaluate's figures on the calibration set) and ``logs`` ({"calibration": ..., "test": ...}, read() dicts).  The
    two logs draw APS's ``u`` from two streams of one seed (evaluate's ``seed`` when given).  ``evaluate_kwargs`` go to
    evaluate (``train_size`` defaults to 1.0).  The logs are kept on the net, as detect_ood keeps its logs."""
    dev = next(net.parameters()).device
    kw = dict(evaluate_kwargs)
    train_size = kw.pop("train_size", 1.0)
    opts = dict(method=method, randomized=bool(randomized), lam=float(lam), k_reg=int(k_reg),
                seed=int(kw["seed"] if kw.get("seed") is not None else Fn.current_seed()) & ((1 << 64) - 1))
    logs, res = net.__dict__.setdefault("_conformal_logs", {}), {}
    for stream, (role, loader) in enumerate((("calibration", cal_loader), ("test", test_loader))):
        log = _kept_log(
            net, logs, role, loader, lambda n: ConformalLog(dev, n, net.num_classes, stream=stream, **opts),
            lambda lg: lg.num_classes == int(net.num_classes) and lg._options() == dict(opts, stream=stream))
        if role == "test":
            log.set_threshold(qhat)
        res[role] = evaluate(net, loader, num_ens, train_size, conformal=log, **kw)
        if role == "calibration":
            qhat = log.calibrate(alpha, mondrian)
    got = {role: logs[role].read() for role in ("calibration", "test")}
    test = conformal_metrics(got["test"])
    test["evaluate"] = res["test"]
    n_cal = got["calibration"]["score"].numel()
    return {"qhat": qhat, "test": test, "in": res["calibration"], "logs": got,
            "calibration": {"n": n_cal, "alpha": float(alpha), "rank": _conformal_rank(n_cal, alpha), "method": method,
                            "mondrian": bool(mondrian)}}


# --------------------------------------------------------------------------------------------------------------------
# Task experts: route each image to the expert least uncertain about it (the reference's Split-MNIST mixture,
# Mixtures/utils_mixture.py:119-187), behind the experts' own Monte-Carlo steps.
# --------------------------------------------------------------------------------------------------------------------
ROUTE_SCORES = ("epistemic", "aleatoric", "both", "mutual_info", "confidence")     # BBB_ROUTE_*, in enum order
_ROUTE_ACC_WORDS = 6 + 2 * L.ROUTE_MAX_EXPERTS


def new_route_metrics(device) -> torch.Tensor:
    """A zeroed routing accumulator for ``ExpertStep(metrics=...)`` (bbb_mc_route_bytes of float64 words)."""
    return torch.zeros(int(L.lib().bbb_mc_route_bytes()) // 8, dtype=torch.float64, device=device)


def read_route_metrics(t: torch.Tensor, num_experts: int) -> dict:
    """One host read of a routing accumulator (layout: include/bbb_b200.h, bbb_mc_route).

    ``steps``, ``images``; ``accuracy`` (routed global class == label), ``local_accuracy`` (the reference's figure: the
    mean over batches of the batch's local accuracy, in which a wrong expert counts as correct when its local class
    matches), ``routing_accuracy`` (routed to the label's task), ``selected`` (the fraction of images sent to each
    expert), ``total_score`` (each expert's score summed over every image) and ``invalid`` (labels outside every
    expert's class range, counted wrong)."""
    K = int(num_experts)
    a = t[:_ROUTE_ACC_WORDS].cpu().tolist()
    steps, images = int(a[0]), int(a[1])
    div = lambda x, n: x / n if n else float("nan")
    sel = a[6:6 + K]
    return {"steps": steps, "images": images, "local_accuracy": div(a[2], steps), "accuracy": div(a[3], images),
            "routing_accuracy": div(a[4], images), "invalid": int(a[5]), "selected": [div(s, images) for s in sel],
            "selected_count": [int(s) for s in sel],
            "total_score": a[6 + L.ROUTE_MAX_EXPERTS:6 + L.ROUTE_MAX_EXPERTS + K]}


class RouteLog(_CursorLog):
    """A data-set-long log of routing decisions on the device, appended to by ``ExpertStep(log=...)`` / ``route`` at
    the score log's device cursor: per image the routed ``expert``, its ``local`` class, the global class ``pred``
    (int32) and every expert's ``scores`` (fp32 [K]).  ``capacity`` entries fit; images past them are counted, not
    written, and ``read()`` refuses a log that dropped any."""

    def __init__(self, device, capacity: int, num_experts: int):
        self._init_cursor(device, capacity, "RouteLog")
        K = int(num_experts)
        if not 2 <= K <= L.ROUTE_MAX_EXPERTS:
            raise ValueError(f"RouteLog: num_experts must be in [2, {L.ROUTE_MAX_EXPERTS}] (got {K})")
        self.num_experts = K
        n = max(1, self.capacity)           # an empty tensor has no address
        self._ints = torch.zeros(3, n, dtype=torch.int32, device=self.device)
        self._scores = torch.zeros(n, K, dtype=torch.float32, device=self.device)

    def read(self) -> dict:
        """The entries logged so far, copies on the log's device: ``expert``, ``local``, ``pred`` int32 [n] and
        ``scores`` float32 [n, K].  Raises EngineError if images were dropped.  Steps in flight must be complete first
        (``ExpertStep.wait()``)."""
        n = self._held("RouteLog")
        return {"expert": self._ints[0, :n].clone(), "local": self._ints[1, :n].clone(),
                "pred": self._ints[2, :n].clone(), "scores": self._scores[:n].clone()}


def _route_offsets(offsets, K, C):
    if offsets is None:
        return [e * C for e in range(K)]
    offs = [int(o) for o in offsets]
    if len(offs) != K or any(o < 0 or o + C > _INT32_MAX for o in offs):
        raise ValueError(f"offsets: {K} class offsets >= 0 expected (got {list(offsets)})")
    return offs


def _route_score(score):
    if score not in ROUTE_SCORES:
        raise ValueError(f"unknown routing score {score!r}: one of {ROUTE_SCORES}")
    return ROUTE_SCORES.index(score)


def _route_launcher(outs, score, offsets, metrics, log, result):
    """Checks the planes and buffers of a routing launch once; returns launch(labels, task), which enqueues
    bbb_mc_route on the current stream (labels: int64 [B] or None; task: -1 or an expert)."""
    kind = _route_score(score)
    K = len(outs)
    if not 2 <= K <= L.ROUTE_MAX_EXPERTS:
        raise L.EngineError(f"route: {K} experts; 2 to {L.ROUTE_MAX_EXPERTS} are routed")
    p0 = outs[0]["pred"]
    B, Cc = p0.shape
    dev = p0.device
    need = {"pred", {L.ROUTE_EPISTEMIC: "epistemic", L.ROUTE_ALEATORIC: "aleatoric", L.ROUTE_BOTH: "epistemic",
                     L.ROUTE_MUTUAL_INFO: "mutual_info", L.ROUTE_CONFIDENCE: "log_outputs"}[kind]}
    if kind == L.ROUTE_BOTH:
        need.add("aleatoric")
    table = (L.RouteExpert * K)()
    for e, o in enumerate(outs):
        for name in ("pred", "epistemic", "aleatoric", "log_outputs", "mutual_info"):
            t = o.get(name)
            shape = (B,) if name == "mutual_info" else (B, Cc)
            if t is None:
                if name in need:
                    raise L.EngineError(f"route: expert {e} has no {name!r} plane (score {score!r})")
                continue
            _check_tensor(t, f"route: expert {e}'s {name!r}", shape, torch.float32, dev)
            setattr(table[e], name, t.data_ptr())
    offs = (C.c_int32 * K)(*_route_offsets(offsets, K, Cc))
    if metrics is not None:
        _check_tensor(metrics, "route: metrics", dtype=torch.float64, device=dev)
        if metrics.numel() * 8 < int(L.lib().bbb_mc_route_bytes()):
            raise L.EngineError(f"route: metrics holds {metrics.numel()} float64 elements, fewer than new_route_metrics")
    if log is not None and (log.device != dev or log.num_experts != K):
        raise L.EngineError(f"route: the log holds {log.num_experts} experts on {log.device}, the step {K} on {dev}")
    for k, shape in (("expert", (B,)), ("local", (B,)), ("pred", (B,)), ("scores", (B, K))):
        _check_tensor(result[k], f"route: result {k!r}", shape, torch.float32 if k == "scores" else torch.int32, dev)
    lg = log is not None
    fixed = (Fn._ptr(result["expert"]), Fn._ptr(result["local"]), Fn._ptr(result["pred"]), Fn._ptr(result["scores"]))
    logs = (Fn._ptr(log._ints[0] if lg else None), Fn._ptr(log._ints[1] if lg else None),
            Fn._ptr(log._ints[2] if lg else None), Fn._ptr(log._scores if lg else None), log.capacity if lg else 0,
            Fn._ptr(log._cursor if lg else None))
    fn = L.lib().bbb_mc_route

    def launch(labels, task):
        if labels is not None:
            _check_tensor(labels, "route: labels", (B,), torch.int64, dev)
        L.check(fn(table, offs, K, B, Cc, kind, Fn._ptr(labels), task, *fixed,
                   Fn._ptr(metrics if labels is not None else None), *logs, Fn._stream(dev)), "bbb_mc_route")
    return launch


def _route_result(B, K, dev):
    i32 = dict(dtype=torch.int32, device=dev)
    return {"expert": torch.empty(B, **i32), "local": torch.empty(B, **i32), "pred": torch.empty(B, **i32),
            "scores": torch.empty(B, K, dtype=torch.float32, device=dev)}


def _route_task(task, K):
    t_ = -1 if task is None else int(task)
    if not -1 <= t_ < K:
        raise ValueError(f"route: task must be None or in [0, {K}) (got {task})")
    return t_


def route_batch(outs, score: str = "epistemic", offsets=None, labels: Optional[torch.Tensor] = None,
                task: Optional[int] = None, metrics: Optional[torch.Tensor] = None,
                log: Optional[RouteLog] = None) -> dict:
    """Route one batch between K experts (bbb_mc_route, on the current stream): ``outs`` are the experts' exchange
    outputs (``MCForward.out`` dicts with ``want_uncertainty``: pred, epistemic, aleatoric, log_outputs [B, C], and
    mutual_info [B] for ``score="mutual_info"``).  Returns ``expert``, ``local``, ``pred`` (int32 [B]) and ``scores``
    (fp32 [B, K]).  ``labels`` (int64 [B]): global classes, or with ``task=t`` the local classes of expert t; with
    labels the step is added to ``metrics`` (new_route_metrics).  ``log``: a RouteLog the images are appended to.
    ``offsets``: each expert's first global class (default e * C)."""
    _route_score(score)
    t_ = _route_task(task, len(outs))
    B = int(outs[0]["pred"].shape[0])
    result = _route_result(B, len(outs), outs[0]["pred"].device)
    _route_launcher(outs, score, offsets, metrics, log, result)(labels, t_)
    return result


def _check_experts(experts, device, score, offsets, group):
    """Host checks of ExpertStep / route: (K, C, offsets)."""
    _route_score(score)
    K = len(experts)
    if not 2 <= K <= L.ROUTE_MAX_EXPERTS:
        raise L.EngineError(f"ExpertStep: {K} experts; 2 to {L.ROUTE_MAX_EXPERTS} are routed")
    ncls = {int(net.num_classes) for net in experts}
    if len(ncls) != 1:
        raise L.EngineError(f"ExpertStep: the experts make different numbers of classes {sorted(ncls)}")
    Cc = ncls.pop()
    offs = _route_offsets(offsets, K, Cc)
    if _dist_info(group)[1] > 1:
        raise L.EngineError("ExpertStep: one rank only (experts on several GPUs are not supported)")
    devs = {next(net.parameters()).device for net in experts} | {torch.device(device)}
    if len(devs) != 1:
        raise L.EngineError(f"ExpertStep: the experts and the input must be on one device (got {sorted(map(str, devs))})")
    return K, Cc, offs


class ExpertStep:
    """``res = ExpertStep(experts, example_x, num_ens, score=...)(x, labels=None, task=None, slot=k)`` -- one Monte-Carlo
    step of every task expert and the routing between them (the reference's predict_using_uncertainty_separate_models,
    Mixtures/utils_mixture.py:119-162, for K experts; ``score="confidence"`` is the baseline of :165-187 on p_bar).

    Each expert gets its own in-flight MCForward (``overlap=True``, ``want_uncertainty=True``, ``want_information`` for
    ``score="mutual_info"``, the same ``normalized``, ``seed``, ``first_replay`` and input slots), so it folds, caches
    preps and runs on the fused chain or the per-layer path exactly as it would alone, with the same output bits.  The
    K steps of a batch are independent and run concurrently; the routing kernel (bbb_mc_route) runs on a stream of its
    own behind the K exchanges.  Before an expert's next step its exchange waits for the last routing, which reads the
    expert's ``out``: the layer chains of batch t+1 overlap the routing of batch t, but no exchange of t+1 overwrites
    planes the routing of t still reads.  No host synchronisation per batch.

    Returns ``expert`` (the routed expert), ``pred`` (its global class offsets[e*] + local), ``local_pred`` (int32 [B])
    and ``scores`` (fp32 [B, K]), the same tensors every call, complete on the routing stream (``wait()``), plus
    ``experts``: the K experts' own ``out`` dicts.  ``labels`` (int64 [B]; global classes, or with ``task=t`` the local
    classes of expert t) add the step to ``metrics`` (new_route_metrics); ``log``: a RouteLog every step appends to.
    ``temperatures``: one per expert (MCForward's ``temperature``; None: that expert is not tempered), so experts
    calibrated one by one route on comparable uncertainty scores.  ``scalings``: one LogitScaling (or None) per expert,
    as ``temperatures``; an expert takes a temperature or a scaling, not both.
    ``offsets``: each expert's first global class (default e * C).  Inference only, one rank only.  As with MCForward,
    two engines over the same layers share the layers' workspaces: ``wait()`` for one before stepping the other."""

    def __init__(self, experts, example_x: torch.Tensor, num_ens: int, score: str = "epistemic",
                 normalized: bool = False, offsets=None, group=None, seed: Optional[int] = None, static_inputs=None,
                 first_replay: int = 0, inflight: int = 1, metrics: Optional[torch.Tensor] = None,
                 log: Optional[RouteLog] = None, temperatures=None, scalings=None):
        experts = list(experts)
        self.K, self.C, self.offsets = _check_experts(experts, example_x.device, score, offsets, group)
        temps = _expert_temperatures(temperatures, self.K, "temperatures")
        scals = _expert_temperatures(scalings, self.K, "scalings")
        Fn._require_cuda(example_x, "ExpertStep")
        if log is not None and (log.device != example_x.device or log.num_experts != self.K):
            raise L.EngineError(f"ExpertStep: the log holds {log.num_experts} experts on {log.device}, the step "
                                f"{self.K} on {example_x.device}")
        self.score, self.metrics, self.log = score, metrics, log
        self.dev = example_x.device
        self.B = int(example_x.shape[0])
        self.seed = int(seed if seed is not None else Fn.current_seed())
        self.inputs = list(static_inputs) if static_inputs else [example_x.clone()]
        self.engines = [MCForward(net, self.inputs[0], num_ens, want_uncertainty=True, normalized=normalized,
                                  seed=self.seed, static_inputs=self.inputs, first_replay=first_replay, overlap=True,
                                  inflight=inflight, want_information=score == "mutual_info", temperature=t,
                                  scaling=sc)
                        for net, t, sc in zip(experts, temps, scals)]
        self.nbuf = self.engines[0].nbuf
        res = _route_result(self.B, self.K, self.dev)
        self._launch = _route_launcher([e.out for e in self.engines], score, self.offsets, metrics, log, res)
        self.out = {"expert": res["expert"], "pred": res["pred"], "local_pred": res["local"],
                    "scores": res["scores"], "experts": [e.out for e in self.engines]}
        self._labels = torch.zeros(self.B, dtype=torch.int64, device=self.dev)
        lo = getattr(torch.cuda.Stream, "priority_range", lambda: (-1, 0))()
        self.route_stream = torch.cuda.Stream(device=self.dev, priority=min(lo))
        self._join_stream = torch.cuda.Stream(device=self.dev)
        # one stream per expert: the K layer chains of a batch run side by side (with inflight > 1 each engine also
        # has its own chain streams behind this one)
        self._streams = [torch.cuda.Stream(device=self.dev, priority=-1) for _ in self.engines]
        self._in_ready, self._route_done, self._labels_read = torch.cuda.Event(), torch.cuda.Event(), torch.cuda.Event()
        self._consumed = [torch.cuda.Event() for _ in range(self.nbuf)]
        self.steps = 0

    def __call__(self, x: Optional[torch.Tensor] = None, labels: Optional[torch.Tensor] = None,
                 task: Optional[int] = None, slot: int = 0) -> dict:
        t_ = _route_task(task, self.K)
        if labels is not None and tuple(labels.shape) != (self.B,):
            raise ValueError(f"ExpertStep: labels must have shape ({self.B},), got {tuple(labels.shape)}")
        cur = torch.cuda.current_stream(self.dev)
        if x is not None:
            # the experts read the slot in place: the last step's chains must have read it first
            for eng in self.engines:
                ev = eng.input_consumed()
                if ev is not None:
                    cur.wait_event(ev)
            self.inputs[slot].copy_(x, non_blocking=True)
        self._in_ready.record(cur)
        for eng, st in zip(self.engines, self._streams):
            if self.steps:                  # the exchange overwrites the out planes the last routing reads
                eng.result_stream.wait_event(self._route_done)
            st.wait_event(self._in_ready)
            with torch.cuda.stream(st):
                eng(slot=slot)
        rs = self.route_stream
        rs.wait_event(self._in_ready)
        with torch.cuda.stream(rs):
            if labels is not None:          # copied before the routing waits: the caller may rewrite them once consumed
                self._labels.copy_(labels, non_blocking=True)
                if labels.is_cuda:
                    labels.record_stream(rs)
            self._labels_read.record(rs)
            for eng in self.engines:
                rs.wait_event(eng._exch_done[eng._last])
            self._launch(self._labels if labels is not None else None, t_)
        self._route_done.record(rs)
        consumed = self._consumed[self.steps % self.nbuf]
        for eng in self.engines:
            self._join_stream.wait_event(eng.input_consumed())
        self._join_stream.wait_event(self._labels_read)
        consumed.record(self._join_stream)
        self._last_consumed = consumed
        self.steps += 1
        return self.out

    def wait(self):
        """Make the current stream wait for the last step's routing (and so for every expert's outputs)."""
        if self.steps:
            torch.cuda.current_stream(self.dev).wait_event(self._route_done)
        return self.out

    def input_consumed(self):
        """Event after which the input slot and labels of the LAST step may be rewritten: the join of the K experts'
        chains (and of the routing stream's copy of the labels)."""
        return self._last_consumed if self.steps else None


def route(experts, loader, num_ens: int, score: str = "epistemic", normalized: bool = False,
          task: Optional[int] = None, log: bool = True, inflight: int = 4, seed: Optional[int] = None,
          offsets=None, temperatures=None, scalings=None) -> dict:
    """predict_using_uncertainty_separate_models (Mixtures/utils_mixture.py:119-162) over ``loader`` (batches of
    (inputs, labels)) for K task experts, on the device: every batch through an ExpertStep, one per batch shape, all
    adding to one routing accumulator that the host reads once, at the end.  Inputs and labels go into rotating device
    slots (pinned host slots for host batches that are not pinned), as in ``evaluate``; the steps and the accumulator
    are kept on the first expert per option key, so the next call rebuilds nothing and draws fresh noise.

    ``labels``: global classes (expert e holds [offsets[e], offsets[e] + C), default e * C), or with ``task=t`` the
    local classes of expert t (the reference's Split-MNIST loaders of task t).  Returns ``accuracy`` (global),
    ``local_accuracy`` (the reference's figure), ``routing_accuracy``, ``selected`` (the fraction sent to each expert),
    ``total_score`` (per expert), ``steps`` / ``images``, and with ``log`` ``per_image``: ``expert``, ``pred`` and
    ``scores`` on the device, in loader order.  ``temperatures`` / ``scalings``: ExpertStep's, one per expert.  Raises
    ValueError at the end if a label was outside every range."""
    experts = list(experts)
    dev = next(experts[0].parameters()).device
    K = _check_experts(experts, dev, score, offsets, None)[0]
    _route_task(task, K)
    if dev.type != "cuda":
        raise L.EngineError(f"route: the experts are on {dev}; the engine runs on CUDA (sm_90a) only")
    n_img = _loader_images(loader) if log else 0
    temps = _expert_temperatures(temperatures, K, "temperatures")
    scals = _expert_temperatures(scalings, K, "scalings")
    key = (tuple(id(e) for e in experts), int(num_ens), score, bool(normalized), int(inflight), seed,
           None if offsets is None else tuple(int(o) for o in offsets),
           tuple(_map_key(t) for t in temps), tuple(_map_key(sc) for sc in scals))
    cache = _engine_cache(experts[0], "_mc_route")
    ent = cache.get(key)
    if ent is not None and not all(eng._prior_guard.ok() for e in ent["engines"].values()
                                   for eng in e["eng"].engines):
        ent = None                          # an expert's prior or mask changed since its graphs were captured
    if ent is None:
        ent = cache[key] = {"acc": new_route_metrics(dev), "engines": {}, "seed": seed, "log": None,
                            "maps": (temps, scals)}
    if log and (ent["log"] is None or ent["log"].capacity < n_img):
        ent["log"] = RouteLog(dev, n_img, K)
        ent["engines"].clear()              # the steps append to the log they were built with
    rlog = ent["log"] if log else None
    ent["acc"].zero_()
    if rlog is not None:
        rlog.reset()

    def build(slots, first_replay):
        return ExpertStep(experts, slots[0], num_ens, score=score, normalized=normalized, offsets=offsets,
                          seed=ent["seed"], static_inputs=slots, first_replay=first_replay, inflight=inflight,
                          metrics=ent["acc"], log=rlog, temperatures=temps, scalings=scals)
    if not _run_loader(ent, loader, dev, max(2, int(inflight)), build, task=task):
        raise ValueError("route: the loader yielded no batch")
    m = read_route_metrics(ent["acc"], K)
    if m["invalid"]:
        raise ValueError(f"route: {m['invalid']} labels are outside every expert's class range"
                         + (f" (task={task}: local classes 0..{experts[0].num_classes - 1})" if task is not None else ""))
    if rlog is not None:
        got = rlog.read()
        m["per_image"] = {"expert": got["expert"], "pred": got["pred"], "scores": got["scores"]}
    return m


# --------------------------------------------------------------------------------------------------------------------
# Temperature scaling (Guo et al. 2017) of the Monte-Carlo predictive, on each sample's logits before the softmax and
# the average over samples (Laves et al. 2019): p_bar_T = mean_s softmax(z_s / T).  A calibration bank of raw
# per-sample logits, a grid search for T on the device, and the temper in front of the exchange.
# --------------------------------------------------------------------------------------------------------------------
def _logit_map(temperature, scaling, device, normalized, num_classes, what):
    """MCForward's ``temperature`` and ``scaling``, the two maps of the one slot in front of the exchange: (the
    one-element fp32 device tensor the temper reads or None, the LogitScaling or None), at most one of them given."""
    if scaling is None:
        return _temperature_tensor(temperature, device, normalized, what), None
    if normalized:
        raise ValueError(f"{what}: a scaling maps the logits of the softmax predictive; the softplus-normalised one "
                         "(normalized=True) takes none")
    if temperature is not None:
        raise ValueError(f"{what}: a temperature or a scaling, not both (fit_scaling(init_temperature=T) starts a "
                         "scaling from T)")
    if not isinstance(scaling, LogitScaling):
        raise TypeError(f"{what}: scaling must be a LogitScaling, got {type(scaling).__name__}")
    if scaling.device != torch.device(device) or scaling.num_classes != int(num_classes):
        raise L.EngineError(f"{what}: the scaling holds {scaling.num_classes} classes on {scaling.device}, the step "
                            f"{num_classes} on {device}")
    return None, scaling


def _map_key(v):
    """The engine-cache key of a temperature or a scaling: by object for a tensor or a LogitScaling (the engines read
    it at run time), by value for a float."""
    if v is None:
        return None
    if isinstance(v, (torch.Tensor, LogitScaling)):
        return (type(v).__name__, id(v))
    return float(v)


def _temperature_tensor(t, device, normalized, what):
    """MCForward's ``temperature`` as the one-element fp32 device tensor the temper reads (a tensor is used as given)."""
    if t is None:
        return None
    if normalized:
        raise ValueError(f"{what}: a temperature tempers the softmax predictive; the softplus-normalised one "
                         "(normalized=True) takes none")
    device = torch.device(device)
    if isinstance(t, torch.Tensor):
        _check_tensor(t, f"{what}: temperature", dtype=torch.float32, device=device)
        if t.numel() != 1:
            raise L.EngineError(f"{what}: temperature must be a one-element float32 tensor, got shape {tuple(t.shape)}")
        return t
    v = float(t)
    if not (math.isfinite(v) and v > 0.0):
        raise ValueError(f"{what}: temperature must be finite and > 0 (got {v})")
    return torch.full((1,), v, dtype=torch.float32, device=device)


def _expert_temperatures(values, K, what="temperatures"):
    if values is None:
        return [None] * K
    values = list(values)
    if len(values) != K:
        raise ValueError(f"ExpertStep: {len(values)} {what} for {K} experts (one per expert, None: none)")
    return values


class LogitBank(_SampleBank):
    """A device-resident bank of every Monte-Carlo sample's raw logits and the label of each image of a calibration set,
    appended to by the step (bbb_mc_logit_log): ``MCForward(..., logit_bank=bank)`` and ``evaluate(..., logit_bank=bank)``
    add one entry per image, in step order, with no host read.  It is what ``fit_temperature`` fits T on.

    Entry i holds the S logit rows z_s [S, C] of its image as the net produced them, fp32 bit for bit -- before any
    temperature, so a bank filled under any temperature fits the same T -- and its int64 label (-1 for a step without
    labels, which the fit refuses).  Unlike ProbBank (tf32 probabilities, which lose the small ones a temperature > 1
    raises) it keeps the logits themselves.  ``capacity`` entries fit; images past them are counted, not written, and
    ``read()`` and the fit refuse a bank that dropped any.  ``group``: as ProbBank's."""

    _keyword = "logit_bank"
    before_temper = True

    def __init__(self, device, capacity: int, num_ens: int, num_classes: int, group=None):
        num_ens, num_classes = int(num_ens), int(num_classes)
        if not 1 <= num_ens <= L.LOGIT_BANK_MAX_SAMPLES:
            raise ValueError(f"LogitBank: num_ens must be in [1, {L.LOGIT_BANK_MAX_SAMPLES}] (got {num_ens})")
        if not 2 <= num_classes <= L.LOGIT_BANK_MAX_CLASSES:
            raise ValueError(f"LogitBank: num_classes must be in [2, {L.LOGIT_BANK_MAX_CLASSES}] (got {num_classes})")
        if int(capacity) >= 1 << 31:
            raise ValueError(f"LogitBank: capacity must be < 2^31 (got {capacity})")
        self._init_bank(device, capacity, num_ens, num_classes, group)
        # (one entry at least: the kernel takes the bank's pointers even when nothing fits)
        self._logits = torch.zeros(max(1, self.capacity), num_ens, num_classes, dtype=torch.float32, device=self.device)
        self._labels = torch.full((max(1, self.capacity),), -1, dtype=torch.int64, device=self.device)
        # a step without labels has been appended since the last reset: append() and MCForward's steps say so (a
        # captured step's kernel runs without the host seeing it)
        self._unlabelled = False

    def reset(self):
        super().reset()
        self._unlabelled = False

    def _launch(self, logits, labels, B):
        L.check(L.lib().bbb_mc_logit_log(Fn._ptr(logits), Fn._ptr(labels), self.num_ens, int(B), self.num_classes,
                                         Fn._ptr(self._logits), Fn._ptr(self._labels), self.capacity,
                                         Fn._ptr(self._cursor), Fn._stream(self.device)), "bbb_mc_logit_log")

    def _log(self, step, par):
        self._launch(step._bank_logits(par), step._labels_of(par), step.B)

    def append(self, logits, labels=None):
        """Append the images of per-sample logits [S, B, C] (fp32 contiguous on the bank's device) and their int64 labels
        [B] (bbb_mc_logit_log on the current stream): logits from anywhere else."""
        self._check_logits(logits)
        B = logits.shape[1]
        if labels is not None:
            _check_tensor(labels, "LogitBank.append: labels", (B,), torch.int64, self.device)
        self._unlabelled |= labels is None
        self._launch(logits, labels, B)

    def read(self) -> dict:
        """The entries so far: {"logits": float32 [n, S, C], "labels": int64 [n]}, copies on the bank's device.  Raises
        EngineError if images were dropped.  Steps in flight must be complete first."""
        n = self._held("LogitBank")
        return {"logits": self._logits[:n].clone(), "labels": self._labels[:n].clone()}


def _check_search(t_min, t_max, grid, rounds):
    t_min, t_max = float(t_min), float(t_max)
    if not (0.0 < t_min < t_max and math.isfinite(t_max)):
        raise ValueError(f"temperature search: need 0 < t_min < t_max < inf (got {t_min}, {t_max})")
    if int(grid) != grid or not 3 <= int(grid) <= L.TEMPERATURE_MAX_POINTS - 1:
        raise ValueError(f"temperature search: grid must be an integer in [3, {L.TEMPERATURE_MAX_POINTS - 1}] "
                         f"(got {grid})")
    if int(rounds) != rounds or int(rounds) < 1:
        raise ValueError(f"temperature search: rounds must be an integer >= 1 (got {rounds})")
    return t_min, t_max, int(grid), int(rounds)


def temperature_grid(t_min: float = 0.05, t_max: float = 20.0, grid: int = 32, prev=None, argmin=None) -> list:
    """One round of the temperature search on tau = ln T (pure host): round 0 (``prev`` None) is ``grid`` points
    equally spaced on [ln t_min, ln t_max]; the round after a grid ``prev`` whose first minimal NLL is point ``argmin``
    spans [prev[max(argmin - 1, 0)], prev[min(argmin + 1, grid - 1)]] with ``grid`` points.  Point k is
    lo + ((hi - lo) * k) / (grid - 1) in IEEE double, as bbb_temperature_nll forms the next round on the device, so
    both plan the same bits.  Every round narrows the spacing by 2 / (grid - 1)."""
    _, _, grid, _ = _check_search(t_min, t_max, grid, 1)
    if prev is None:
        lo, hi = math.log(float(t_min)), math.log(float(t_max))
    else:
        prev = [float(v) for v in prev]
        if len(prev) != grid:
            raise ValueError(f"temperature_grid: prev holds {len(prev)} points, grid is {grid}")
        if argmin is None or int(argmin) != argmin or not 0 <= int(argmin) < grid:
            raise ValueError(f"temperature_grid: argmin must be an index into prev (got {argmin})")
        a = int(argmin)
        lo, hi = prev[max(a - 1, 0)], prev[min(a + 1, grid - 1)]
    return [lo + (hi - lo) * k / (grid - 1) for k in range(grid)]


class TemperatureFit:
    """What fit_temperature enqueued: ``temperature`` (one-element fp32 device tensor, the fitted T), and on ``read()``
    -- the one host synchronisation -- the floats."""

    def __init__(self, bank, temperature, fit, taus, nlls, grid, trace):
        self.temperature, self._fit, self._taus, self._nlls = temperature, fit, taus, nlls
        self._bank, self._grid, self._trace = bank, grid, trace

    def read(self) -> dict:
        """{"temperature", "nll" (the bank's NLL at it), "nll_at_one" (at T = 1), "at_bound" (round 0's minimum was an
        end of [t_min, t_max]: widen the range), "tau" (ln T)}, and with ``trace`` "trace": one {"tau", "nll"} per round
        (round 0 with T = 1 last).  Raises ValueError when there is no fit -- an empty bank, one that dropped images, or
        one that holds an image logged without a label or with a label outside [0, C) -- and ``temperature`` then keeps
        the value it had before the fit.  Read after the fit, not after later appends to the bank."""
        v = torch.cat([self._fit, self.temperature.to(torch.float64)]).tolist()
        if any(math.isnan(x) for x in v[:4]):
            raise ValueError(f"fit_temperature: no fit -- {self._why()}")
        out = {"temperature": v[4], "nll": v[1], "nll_at_one": v[0], "at_bound": bool(v[2]), "tau": v[3]}
        if self._trace:
            taus, nlls = self._taus.tolist(), self._nlls.tolist()
            out["trace"] = [{"tau": taus[r][:self._grid + (r == 0)], "nll": nlls[r][:self._grid + (r == 0)]}
                            for r in range(len(taus))]
        return out

    def _why(self):
        return _no_fit_reason(self._bank)


def _no_fit_reason(bank):
    """Why the device found no fit on a LogitBank (host reads of the bank)."""
    n, dropped = bank._counts()
    if dropped:
        return f"the bank dropped {dropped} images (capacity {bank.capacity})"
    if n == 0:
        return "the bank is empty"
    y = bank._labels[:n]
    if bool((y < 0).any()):
        return f"{int((y < 0).sum())} images were logged without a label (a step with_labels=False)"
    if bool((y >= bank.num_classes).any()):
        return f"a label is outside [0, {bank.num_classes})"
    return "the bank's logits give no finite NLL (NaN or infinite logits?)"


def fit_temperature(bank: LogitBank, t_min: float = 0.05, t_max: float = 20.0, grid: int = 32, rounds: int = 4,
                    out: Optional[torch.Tensor] = None, trace: bool = False) -> TemperatureFit:
    """The temperature that minimises the bank's NLL of the tempered predictive,
        l(T) = -(1/n) sum_i log( (1/S) sum_s softmax(z_is / T)[y_i] ),
    by a grid search on tau = ln T, enqueued on the current stream with no host read: ``rounds`` passes of
    bbb_temperature_nll over the bank, each evaluating ``grid`` points (temperature_grid; round 0 also T = 1) and
    writing the next round's grid on the device.  The result is never worse than T = 1 on the bank.

    Returns a TemperatureFit: ``.temperature`` is the fitted T as a one-element fp32 device tensor -- written in place
    into ``out`` when given, so engines that temper with ``out`` (MCForward / evaluate ``temperature=out``) read the new
    value at their next step; without ``out`` it starts at 1 -- and ``.read()`` gives the floats.  A fit the device
    cannot make (an empty bank, one that dropped images, or one that holds an image without a valid label) leaves
    ``.temperature`` as it was, and ``.read()`` raises.  A bank known on the host to hold images without labels (appended
    without them, or by a step with_labels=False) is refused here already."""
    t_min, t_max, grid, rounds = _check_search(t_min, t_max, grid, rounds)
    if not isinstance(bank, LogitBank):
        raise TypeError(f"fit_temperature: expected a LogitBank, got {type(bank).__name__}")
    Fn._require_cuda(bank._cursor, "fit_temperature")
    if bank.capacity < 1:
        raise ValueError("fit_temperature: the bank has no capacity")
    if bank._unlabelled:
        raise ValueError("fit_temperature: the bank holds images logged without labels (a step with_labels=False)")
    dev = bank.device
    if out is None:
        out = torch.ones(1, dtype=torch.float32, device=dev)
    _temperature_tensor(out, dev, False, "fit_temperature(out=...)")
    f64 = dict(dtype=torch.float64, device=dev)
    taus = torch.zeros(rounds, grid + 1, **f64)               # round 0's point `grid` is tau = 0 (T = 1)
    plan = torch.tensor(temperature_grid(t_min, t_max, grid), dtype=torch.float64).pin_memory()
    taus[0, :grid].copy_(plan, non_blocking=True)
    nlls = torch.full((rounds, grid + 1), float("nan"), **f64)
    fit = torch.full((4,), float("nan"), **f64)
    lib = L.lib()
    nbytes = int(lib.bbb_temperature_workspace_bytes(bank.capacity, grid + 1))
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    for r in range(rounds):
        flags = (L.TEMPERATURE_FIRST if r == 0 else 0) | (L.TEMPERATURE_LAST if r == rounds - 1 else 0)
        L.check(lib.bbb_temperature_nll(
            Fn._ptr(bank._logits), Fn._ptr(bank._labels), Fn._ptr(bank._cursor), bank.capacity, bank.num_ens,
            bank.num_classes, Fn._ptr(taus[r]), grid + (r == 0), grid, flags, Fn._ptr(nlls[r]),
            Fn._ptr(taus[r + 1]) if r + 1 < rounds else None, Fn._ptr(fit), Fn._ptr(out), Fn._ptr(ws), nbytes,
            Fn._stream(dev)), "bbb_temperature_nll")
    return TemperatureFit(bank, out, fit, taus, nlls, grid, trace)


def calibrate_temperature(net, cal_loader, num_ens: int, t_min: float = 0.05, t_max: float = 20.0, grid: int = 32,
                          rounds: int = 4, out: Optional[torch.Tensor] = None, trace: bool = False,
                          **evaluate_kwargs) -> dict:
    """Temperature scaling over a whole calibration set: ``evaluate`` over ``cal_loader`` (batches of (x, y), held out
    from training) into a LogitBank, then fit_temperature on it.  Returns ``temperature`` (the one-element fp32 device
    tensor; ``out`` when given), ``fit`` (TemperatureFit.read()) and ``evaluate`` (evaluate's figures on the calibration
    set, untempered unless ``temperature`` is among ``evaluate_kwargs``).  The intended use:

        cal = mc.calibrate_temperature(net, cal_loader, num_ens)
        test = mc.evaluate(net, test_loader, num_ens, train_size, temperature=cal["temperature"])   # test ECE, NLL

    and the same ``temperature=`` to detect_ood, conformal or acquire (through their evaluate keywords), MCForward, or
    ExpertStep / route (one per expert).  ``evaluate_kwargs`` go to evaluate (``train_size`` defaults to 1.0).  The
    bank is kept on the net, as detect_ood keeps its logs, and reused by the next call; it is made with evaluate's
    ``group``, so on several ranks every rank fits the same T on the whole calibration set."""
    dev = next(net.parameters()).device
    kw = dict(evaluate_kwargs)
    train_size = kw.pop("train_size", 1.0)
    S, Cc = int(num_ens), int(net.num_classes)
    group = kw.get("group")
    bank = _kept_log(net, net.__dict__.setdefault("_temperature_banks", {}), "calibration", cal_loader,
                     lambda n: LogitBank(dev, n, S, Cc, group=group),
                     lambda b: (b.num_ens, b.num_classes) == (S, Cc) and b.group is group)
    m = evaluate(net, cal_loader, num_ens, train_size, logit_bank=bank, **kw)
    fit = fit_temperature(bank, t_min, t_max, grid, rounds, out=out, trace=trace)
    return {"temperature": fit.temperature, "fit": fit.read(), "evaluate": m}


# --------------------------------------------------------------------------------------------------------------------
# Vector and matrix scaling (Guo et al. 2017) of the Monte-Carlo predictive, in the temperature's place:
# p_bar = mean_s softmax(f(z_s)), f(z) = a * z + b or W z + b, fitted by full-batch Adam on a LogitBank on the device.
# --------------------------------------------------------------------------------------------------------------------
SCALING_KINDS = {"vector": L.SCALING_VECTOR, "matrix": L.SCALING_MATRIX}


def _check_kind(kind, what, num_classes=None):
    if kind not in SCALING_KINDS:
        raise ValueError(f"{what}: kind must be 'vector' or 'matrix' (got {kind!r})")
    if kind == "matrix" and num_classes is not None and int(num_classes) > L.SCALING_MATRIX_MAX_CLASSES:
        raise ValueError(f"{what}: matrix scaling takes at most {L.SCALING_MATRIX_MAX_CLASSES} classes "
                         f"(got {num_classes})")
    return SCALING_KINDS[kind]


class LogitScaling:
    """The parameters of vector or matrix scaling on the device.  ``params`` is fp32: vector [2, C], ``a = params[0]``
    (the per-class scales) and ``b = params[1]``; matrix [C + 1, C], ``W = params[:C]`` (row j maps to class j, C <= 128)
    and ``b = params[C]``.  It starts at the identity (a = 1 or W = I, b = 0), which gives the untransformed predictive
    bit for bit.  Engines given it (MCForward / evaluate ``scaling=``, ExpertStep / route ``scalings=``) read the
    parameters at run time, so a fit written in place (fit_scaling(out=...)) or parameters set in place under no_grad
    are read by their next step."""

    def __init__(self, device, num_classes: int, kind: str = "vector"):
        self._kind = _check_kind(kind, "LogitScaling", num_classes)
        num_classes = int(num_classes)
        if not 2 <= num_classes <= L.LOGIT_BANK_MAX_CLASSES:
            raise ValueError(f"LogitScaling: num_classes must be in [2, {L.LOGIT_BANK_MAX_CLASSES}] (got {num_classes})")
        self.kind, self.num_classes = kind, num_classes
        rows = num_classes + 1 if kind == "matrix" else 2
        self.params = torch.zeros(rows, num_classes, dtype=torch.float32, device=device)
        self.device = self.params.device
        self.reset()

    @property
    def a(self):
        if self.kind != "vector":
            raise AttributeError("LogitScaling.a: a matrix scaling has W")
        return self.params[0]

    @property
    def W(self):
        if self.kind != "matrix":
            raise AttributeError("LogitScaling.W: a vector scaling has a")
        return self.params[:self.num_classes]

    @property
    def b(self):
        return self.params[-1]

    def reset(self):
        """Back to the identity, in place."""
        self.params.zero_()
        if self.kind == "matrix":
            self.W.fill_diagonal_(1.0)
        else:
            self.a.fill_(1.0)
        return self

    def _launch(self, z, stream):
        L.check(L.lib().bbb_mc_logit_scale(Fn._ptr(z), z.numel() // self.num_classes, self.num_classes, self._kind,
                                           Fn._ptr(self.params), stream), "bbb_mc_logit_scale")

    def apply_(self, z):
        """z <- f(z) in place on fp32 logits [..., C] (contiguous, on the device; bbb_mc_logit_scale on the current
        stream): vector, the bits of torch's ``z * a + b``; matrix, each output an fmaf chain over the classes in order,
        then + b."""
        _check_tensor(z, "LogitScaling.apply_: logits", dtype=torch.float32, device=self.device)
        if z.dim() < 1 or z.shape[-1] != self.num_classes or z.numel() == 0:
            raise L.EngineError(f"LogitScaling.apply_: expected non-empty logits [..., {self.num_classes}], got "
                                f"{tuple(z.shape)}")
        self._launch(z, Fn._stream(self.device))
        return z


class ScalingFit:
    """What fit_scaling enqueued: ``scaling`` (the LogitScaling holding the fitted parameters), and on ``read()`` --
    the one host synchronisation -- the floats."""

    def __init__(self, bank, scaling, fit, iters):
        self.scaling, self._bank, self._fit, self._iters = scaling, bank, fit, iters

    def read(self) -> dict:
        """{"nll" (the bank's objective at the fitted parameters: its NLL, plus the penalties when l2_offdiag or l2_bias
        > 0), "nll_start" (at the starting point), "nll_last" (at the last iterate), "iters", and "a" or "W" (lists; W
        row by row) and "b"}.  The result is the best iterate, never worse than the start.  Raises ValueError when
        there is no fit -- an empty bank, one that dropped images, one that holds an image without a valid label, or
        a non-finite objective -- and ``scaling`` then keeps the parameters it had before the fit."""
        v = torch.cat([self._fit, self.scaling.params.flatten().to(torch.float64)]).tolist()
        if not (math.isfinite(v[0]) and math.isfinite(v[1])):
            raise ValueError(f"fit_scaling: no fit -- {_no_fit_reason(self._bank)}")
        C = self.scaling.num_classes
        p = v[3:]
        out = {"nll": v[1], "nll_start": v[0], "nll_last": v[2], "iters": self._iters, "b": p[-C:]}
        if self.scaling.kind == "matrix":
            out["W"] = [p[j * C:(j + 1) * C] for j in range(C)]
        else:
            out["a"] = p[:C]
        return out


def scaling_schedule(lr: float, iters: int) -> list:
    """The step sizes of fit_scaling's Adam passes (pure host): a cosine decay from ``lr`` to 0 over ``iters`` steps,
    lr_t = lr (1 + cos(pi t / iters)) / 2 for t = 0 .. iters - 1."""
    return [float(lr) * 0.5 * (1.0 + math.cos(math.pi * t / iters)) for t in range(int(iters))]


def fit_scaling(bank: LogitBank, kind: str = "vector", *, iters: int = 300, lr: float = 0.1, l2_offdiag: float = 0.0,
                l2_bias: float = 0.0, init_temperature=None, out: Optional[LogitScaling] = None) -> ScalingFit:
    """The map f -- vector a * z + b, or matrix W z + b (C <= 128) -- that minimises the bank's objective
        J = -(1/n) sum_i log( (1/S) sum_s softmax(f(z_is))[y_i] )
            + l2_offdiag * sum_{j != k} W_jk^2 / (C (C - 1)) + l2_bias * sum_c b_c^2 / C
    (the matrix penalties are ODIR, Kull et al. 2019; l2_offdiag is for matrix scaling only), by ``iters`` full-batch
    Adam steps (scaling_schedule's step sizes; beta 0.9 / 0.999) from the identity -- or from a = 1 / T or W = I / T,
    b = 0 with ``init_temperature`` T (a float or a one-element fp32 device tensor, e.g. a TemperatureFit's, read on
    the device) -- enqueued on the current stream with no host read: ``iters + 1`` passes of bbb_scaling_nll_grad over
    the bank, each the objective, its gradient and the step (matrix: both contractions on tf32 wgmma); the last pass
    evaluates the last iterate.  The best iterate is kept on the device, so the result is never worse on the bank than
    the start.

    Returns a ScalingFit: ``.scaling`` holds the result -- ``out`` when given, written in place, so engines that scale
    with it read the new parameters at their next step; a new LogitScaling otherwise -- and ``.read()`` gives the
    floats.  A fit the device cannot make (an empty bank, one that dropped images, an image without a valid label, a
    non-finite objective) leaves ``.scaling`` as it was, and ``.read()`` raises.  A bank on several ranks (``group``) holds
    every sample on every rank, so every rank fits the same bits.  The arguments after
    ``kind`` are keyword-only."""
    if not isinstance(bank, LogitBank):
        raise TypeError(f"fit_scaling: expected a LogitBank, got {type(bank).__name__}")
    k = _check_kind(kind, "fit_scaling", bank.num_classes)
    if int(iters) != iters or int(iters) < 0:
        raise ValueError(f"fit_scaling: iters must be an integer >= 0 (got {iters})")
    lr, l2_offdiag, l2_bias = float(lr), float(l2_offdiag), float(l2_bias)
    if not (math.isfinite(lr) and lr >= 0.0):
        raise ValueError(f"fit_scaling: lr must be finite and >= 0 (got {lr})")
    if not (math.isfinite(l2_bias) and l2_bias >= 0.0):
        raise ValueError(f"fit_scaling: l2_bias must be finite and >= 0 (got {l2_bias})")
    if not (math.isfinite(l2_offdiag) and l2_offdiag >= 0.0) or (kind == "vector" and l2_offdiag != 0.0):
        raise ValueError(f"fit_scaling: l2_offdiag must be finite and >= 0, and 0 for vector scaling (got {l2_offdiag})")
    Fn._require_cuda(bank._cursor, "fit_scaling")
    if bank.capacity < 1:
        raise ValueError("fit_scaling: the bank has no capacity")
    if bank._unlabelled:
        raise ValueError("fit_scaling: the bank holds images logged without labels (a step with_labels=False)")
    dev, C, S, iters = bank.device, bank.num_classes, bank.num_ens, int(iters)
    if out is None:
        out = LogitScaling(dev, C, kind)
    elif not isinstance(out, LogitScaling) or out.device != dev or out.num_classes != C or out.kind != kind:
        raise L.EngineError(f"fit_scaling(out=...): expected a {kind} LogitScaling of {C} classes on {dev}")
    P = out.params.numel()
    state = torch.zeros(3, P, dtype=torch.float64, device=dev)          # Adam's double iterate and moments
    start = state[0, :P - C].view(C, C).diagonal() if kind == "matrix" else state[0, :C]
    start.fill_(1.0)
    if init_temperature is not None:
        T = _temperature_tensor(init_temperature, dev, False, "fit_scaling(init_temperature=...)")
        start.copy_((1.0 / T.to(torch.float64)).expand_as(start))
    theta = state[0].to(torch.float32)
    best = theta.clone()
    fit = torch.full((3,), float("nan"), dtype=torch.float64, device=dev)
    lib = L.lib()
    nbytes = int(lib.bbb_scaling_workspace_bytes(bank.capacity, S, C, k))
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    steps = scaling_schedule(lr, iters)
    for t in range(iters + 1):
        flags = (L.SCALING_FIRST if t == 0 else 0) | (L.SCALING_LAST if t == iters else 0) | \
            (L.SCALING_UPDATE if t < iters else 0)
        lr_t = steps[t] if t < iters else 0.0
        L.check(lib.bbb_scaling_nll_grad(
            Fn._ptr(bank._logits), Fn._ptr(bank._labels), Fn._ptr(bank._cursor), bank.capacity, S, C, k,
            flags, Fn._ptr(theta), Fn._ptr(state), Fn._ptr(best), Fn._ptr(fit), None, Fn._ptr(out.params), l2_offdiag,
            l2_bias, lr_t, 1.0 - 0.9 ** (t + 1), 1.0 - 0.999 ** (t + 1), Fn._ptr(ws), nbytes, Fn._stream(dev)),
            "bbb_scaling_nll_grad")
    return ScalingFit(bank, out, fit, iters)


def calibrate_scaling(net, cal_loader, num_ens: int, kind: str = "vector", *, init: Optional[str] = None,
                      iters: int = 300, lr: float = 0.1, l2_offdiag: float = 0.0, l2_bias: float = 0.0,
                      out: Optional[LogitScaling] = None, **evaluate_kwargs) -> dict:
    """Vector or matrix scaling over a whole calibration set, as calibrate_temperature: ``evaluate`` over
    ``cal_loader`` into the LogitBank kept on the net (the one calibrate_temperature keeps), then fit_scaling on it.
    ``init="temperature"`` fits T first (fit_temperature's defaults) and starts from a = 1 / T or W = I / T.  Returns ``scaling`` (the LogitScaling;
    ``out`` when given), ``fit`` (ScalingFit.read()), ``evaluate`` (evaluate's figures on the calibration set) and,
    with ``init="temperature"``, ``temperature_fit`` (TemperatureFit.read()).  The intended use:

        cal = mc.calibrate_scaling(net, cal_loader, num_ens, init="temperature")
        test = mc.evaluate(net, test_loader, num_ens, train_size, scaling=cal["scaling"])"""
    _check_kind(kind, "calibrate_scaling", net.num_classes if net is not None else None)
    if init not in (None, "temperature"):
        raise ValueError(f"calibrate_scaling: init must be None or 'temperature' (got {init!r})")
    dev = next(net.parameters()).device
    kw = dict(evaluate_kwargs)
    train_size = kw.pop("train_size", 1.0)
    S, Cc = int(num_ens), int(net.num_classes)
    group = kw.get("group")
    bank = _kept_log(net, net.__dict__.setdefault("_temperature_banks", {}), "calibration", cal_loader,
                     lambda n: LogitBank(dev, n, S, Cc, group=group),
                     lambda b: (b.num_ens, b.num_classes) == (S, Cc) and b.group is group)
    m = evaluate(net, cal_loader, num_ens, train_size, logit_bank=bank, **kw)
    res = {"evaluate": m}
    T = None
    if init == "temperature":
        tf = fit_temperature(bank)
        res["temperature_fit"] = tf.read()
        T = tf.temperature
    fit = fit_scaling(bank, kind, iters=iters, lr=lr, l2_offdiag=l2_offdiag, l2_bias=l2_bias, init_temperature=T,
                      out=out)
    res.update(scaling=fit.scaling, fit=fit.read())
    return res

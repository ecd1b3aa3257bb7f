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

import ctypes as C
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
    import math
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


class MCForward:
    """``out = MCForward(net, example_x, num_ens, ...)(x, labels=None)`` -- the sharded MC step on the engine.

    Returns a dict of device tensors (the same objects every call; identical on all ranks):
      log_outputs [B,C], kl (= sum_j kl_j / num_ens), and with ``want_uncertainty`` pred / epistemic / aleatoric [B,C]
      and entropy [B]; with ``with_labels`` head = [loss, nll, accuracy, beta*kl] (metrics.py:12-14, 23-24); with
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
                 batch_shards: int = 1, metrics: Optional[torch.Tensor] = None):
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
        take); None = as many as ``fold_budget`` bytes of activations allow (layer_fold_groups)."""
        if want_information and not want_uncertainty:
            raise L.EngineError("MCForward: want_information needs want_uncertainty")
        Fn._require_cuda(example_x, "MCForward")
        lib = L.lib()
        if metrics is not None:
            if not with_labels:
                raise L.EngineError("MCForward: metrics needs with_labels")
            n = int(lib.bbb_mc_metrics_bytes()) // 8
            if not (metrics.device == example_x.device and metrics.dtype == torch.float64 and metrics.is_contiguous()
                    and metrics.numel() >= n):
                raise L.EngineError(f"MCForward: metrics must be a contiguous float64 tensor of >= {n} elements on "
                                    f"{example_x.device} (mc.new_metrics)")
        self.metrics = self._metrics = metrics      # _metrics: the accumulator the exchange adds to
        self.net, self.group = net, group
        self.dist, self.world, self.rank = _dist_info(group)
        if self.world > 16:
            raise L.EngineError("MCForward: at most 16 ranks (one node)")
        dev = self.dev = example_x.device
        self.num_ens = int(num_ens)
        self.sample_shards, self.group_index, self.block = shard_layout(self.world, self.rank, batch_shards)
        self.batch_shards = int(batch_shards)
        self.ids = local_samples(self.num_ens, self.sample_shards, self.group_index)
        self.B = int(example_x.shape[0])
        if self.batch_shards > self.B:
            raise L.EngineError(f"MCForward: batch_shards={self.batch_shards} > batch {self.B} (a row block would be empty)")
        self.rows = row_block(self.B, self.batch_shards, self.block)     # this rank's images [b0, b1)
        self.nb = self.rows[1] - self.rows[0]
        self.C = int(num_classes if num_classes is not None else net.num_classes)
        self.flags = (L.MC_MOMENTS if want_uncertainty else 0) | (L.MC_NORMALIZED if normalized else 0) | \
            (L.MC_INFO if want_information else 0)
        self.want_uncertainty, self.with_labels = want_uncertainty, with_labels
        self.train_size, self.beta = float(train_size), float(beta)
        # every rank must draw sample j from the same (seed, stream): share rank 0's seed unless one is given
        if seed is None:
            box = [Fn.current_seed()]
            if self.world > 1:
                self.dist.broadcast_object_list(box, src=self.dist.get_global_rank(group, 0) if group is not None else 0, group=group)
            seed = box[0]
        self.seed = int(seed)
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
        self._imported, self._own = [], None
        if self.world == 1:
            self._buf = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
            ptrs = [self._buf.data_ptr()]
        else:
            ptrs = self._open_peers(nbytes)
        self.peers = (C.c_void_p * self.world)(*ptrs)
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
        # layer_fold = (G, number of groups) when it does.
        self.layer_fold, self._groups = None, None
        if self.fold_steps is None and fold and len(self.ids) > 1:
            self._groups = self._plan_layer_fold(net, kids, example_x, fold_group, fold_budget)
        if self._groups is not None:
            G = max(n for _, n in self._groups)
            self.layer_fold = (G, len(self._groups))
            # the first layer's input: x repeated G times, one buffer per concurrently running step
            self.xrep_all = [torch.empty((G * self.nb,) + tuple(example_x.shape[1:]), dtype=example_x.dtype, device=dev)
                             for _ in range(nbuf)]
        self.graph, self.graphs = None, []
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
        lib = L.lib()
        for n in sorted({n for _, n in groups}):
            for m, xs in layers:
                cfg = m._cfg(True)
                d = Fn.make_desc((n * xs[0],) + tuple(xs[1:]), tuple(m.W_mu.shape), cfg["conv"], cfg["variant"], True,
                                 m.bias_mu is not None, cfg["prior_mu"], cfg["prior_sigma"], cfg["math"],
                                 cfg["kl_convention"], cfg["act"], fold=(self.nb, self.sample_shards << 40),
                                 first_image=self.rows[0])
                if lib.bbb_forward_supported(C.byref(d)) != 0:
                    return None
        return groups

    # -- peer-mapped receive buffers (CUDA IPC; handles travel over torch.distributed) -----------------------
    def _open_peers(self, nbytes):
        lib = L.lib()
        torch.cuda.synchronize(self.dev)
        own = C.c_void_p()
        with torch.cuda.device(self.dev):
            L.check(lib.bbb_comm_alloc(C.c_size_t(nbytes), C.byref(own)), "bbb_comm_alloc")
            self._own = own.value
            handle = (C.c_ubyte * 64)()
            L.check(lib.bbb_comm_export(C.c_void_p(self._own), handle), "bbb_comm_export")
            handles = [None] * self.world
            self.dist.all_gather_object(handles, bytes(handle), group=self.group)
            ptrs = []
            for q, h in enumerate(handles):
                if q == self.rank:
                    ptrs.append(self._own)
                    continue
                peer = C.c_void_p()
                L.check(lib.bbb_comm_import((C.c_ubyte * 64).from_buffer_copy(h), C.byref(peer)), f"bbb_comm_import (rank {q})")
                self._imported.append(peer.value)
                ptrs.append(peer.value)
        self.dist.barrier(group=self.group)
        return ptrs

    def timeouts(self) -> int:
        """Exchange waits that gave up because a peer never delivered (results of those steps are invalid)."""
        return int(self.state[8:12].view(torch.int32).item())

    def close(self):
        """Unmap the peers' buffers and free the local one (after every rank is done with them)."""
        lib = L.lib()
        if self.world > 1 and self._own is not None:
            torch.cuda.synchronize(self.dev)
            self.dist.barrier(group=self.group)
            for p in self._imported:
                lib.bbb_comm_unimport(C.c_void_p(p))
            lib.bbb_comm_free(C.c_void_p(self._own))
            self._imported, self._own = [], None

    # -- one step ----------------------------------------------------------------------------------------------
    def _step(self, x, base=None, advance=False):
        """This rank's samples through the engine, then the exchange kernel."""
        kl_ptr, n_kl = self._chain(x, base, advance)
        self._exchange(kl_ptr, n_kl)
        return self.out

    def _chain(self, x, base=None, advance=False, par=0):
        """This rank's samples through the engine into the sample buffer ``par``.  A fused chain writes its logits
        straight into it and hands over its per-layer KL scalars un-summed (fused.direct_output).  Returns the (pointer,
        count) of the floats whose sum is one sample's KL."""
        from . import fused
        from .graph import _STRIDE
        logits_buf = self.logits_all[par]
        kl_buf = self.kl_terms_all[par] if self.overlap else None
        inc = _STRIDE * self.inflight
        b0, nb = self.rows[0], self.nb
        x = x[b0:b0 + nb]                                 # this rank's row block (a view: NCHW rows are contiguous)
        with torch.no_grad(), Fn.workspace_slot(par if self.inflight > 1 else Fn.current_workspace_slot()), \
                Fn.first_image(b0):
            # The Philox base moves at the HEAD of a captured step, BEFORE the prep streams fork: with this one-thread
            # kernel as the single root of the graph every GEMM kernel of the chain is launched programmatically behind
            # its predecessor; with the fork in front of it (prep kernels as further root nodes) or with no plain kernel
            # at the head, the programmatic edges of the whole chain are lost and every GEMM waits for its predecessor.
            if advance:
                Fn.noise_advance(base, inc)
            kl_ptr, n_kl = None, 0
            if self.fold_steps is not None:
                with Fn.stream_base(base), Fn.mc_sample(self.ids[0], self.seed):
                    _, kls = fused._run(self.fold_steps, x, True, logits_buf.view(len(self.ids) * nb, self.C), True, None,
                                        fold=self.fold, kls_out=kl_buf)
                self._kl_terms = kls
                kl_ptr, n_kl = Fn._ptr(kls), kls.numel()
            if self._groups is not None:
                # group (s0, n): local samples s0 .. s0+n-1 in one pass over n x nb rows; row block k is global sample
                # ids[s0] + k * Rs (stream stride Rs << 40, as in the fused fold) and lands in logits_buf[s0 + k]
                xr = self.xrep_all[par]
                G = self.layer_fold[0]
                xr.view((G,) + tuple(x.shape)).copy_(x.unsqueeze(0).expand((G,) + tuple(x.shape)))
                for gi, (s0, n) in enumerate(self._groups):
                    with Fn.stream_base(base), Fn.mc_sample(self.ids[s0], self.seed), \
                            Fn.layer_fold(nb, self.sample_shards << 40):
                        logits, kl = self.net(xr[:n * nb])
                    logits_buf[s0:s0 + n].view(n * nb, self.C).copy_(logits.reshape(n * nb, self.C))
                    if gi == 0:                               # every sample has the same KL, computed once per pass
                        one = self.kl_one_all[par:par + 1]
                        one.copy_(torch.as_tensor(kl, dtype=torch.float32, device=self.dev).reshape(1))
                        kl_ptr, n_kl = Fn._ptr(one), 1
            for k, j in enumerate(self.ids if self.fold_steps is None and self._groups is None else ()):
                with Fn.stream_base(base), Fn.mc_sample(j, self.seed), \
                        fused.direct_output(logits_buf[k], kl_buf if k == 0 else None) as hook:
                    logits, kl = self.net(x)
                if not hook.used:
                    logits_buf[k].copy_(logits.reshape(nb, self.C))
                if k == 0:
                    if hook.used:
                        self._kl_terms = kl                       # per-layer scalars of sample 0 (every sample has the same KL)
                        kl_ptr, n_kl = Fn._ptr(kl), kl.numel()
                    else:
                        one = self.kl_one_all[par:par + 1]
                        one.copy_(torch.as_tensor(kl, dtype=torch.float32, device=self.dev).reshape(1))
                        kl_ptr, n_kl = Fn._ptr(one), 1
            if not self.ids and self.group_index == 0:
                raise L.EngineError("MCForward: sample group 0 must own a sample")
        return kl_ptr, n_kl

    def _exchange(self, kl_ptr, n_kl, advance_base=None, par=0):
        """The one kernel behind the samples: combine + exchange + heads (bbb_mc_exchange_info)."""
        from .graph import _STRIDE
        o = self.out
        lib = L.lib()
        args = (
            Fn._ptr(self.logits_all[par]), len(self.ids), self.num_ens, self.B, self.C, kl_ptr, n_kl, self.flags,
            Fn._ptr(self.labels_all[par] if self.labels_all is not None else None), C.c_float(self.train_size), C.c_float(self.beta), self.rank, self.world, self.peers,
            Fn._ptr(self.state), Fn._ptr(o["log_outputs"]), Fn._ptr(o["kl"]), Fn._ptr(o.get("pred")),
            Fn._ptr(o.get("epistemic")), Fn._ptr(o.get("aleatoric")), Fn._ptr(o.get("entropy")), Fn._ptr(o.get("head")),
            Fn._ptr(advance_base), C.c_uint64(_STRIDE if advance_base is not None else 0),
            Fn._ptr(o.get("expected_entropy")), Fn._ptr(o.get("mutual_info")))
        if self._metrics is not None:
            L.check(lib.bbb_mc_exchange_metrics(*args, self.batch_shards, Fn._ptr(self._metrics), Fn._stream(self.dev)),
                    "bbb_mc_exchange_metrics")
        elif self.batch_shards == 1:
            L.check(lib.bbb_mc_exchange_info(*args, Fn._stream(self.dev)), "bbb_mc_exchange_info")
        else:
            L.check(lib.bbb_mc_exchange_sharded(*args, self.batch_shards, Fn._stream(self.dev)), "bbb_mc_exchange_sharded")

    def _capture(self, warmup: int = 2):
        from .graph import _STRIDE
        dev = self.dev
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
        live = self._metrics
        if live is not None:
            self._metrics = torch.zeros_like(live)      # the warm-up steps do not count
        with torch.cuda.stream(side):
            for _ in range(warmup):                 # eager: creates plans / workspaces; every rank runs the same exchanges
                self._step(self.x, self.base)
            for p_ in range(1, self.inflight):      # the other in-flight steps' own layer workspaces
                self._exchange(*self._chain(self.x, self.base, par=p_), par=p_)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        self._metrics = live
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
                with torch.cuda.graph(g, stream=cap):
                    self._exchange(kl_ptr, n_kl, par=par)
                self.exch_graphs.append(g)
            self.kernels_per_step = n_chain + 1
            self.graphs = self.chain_graphs[0]
            # the exchange kernel is tiny and latency-critical (peers wait for it): highest priority the device offers
            lo = getattr(torch.cuda.Stream, "priority_range", lambda: (-1, 0))()
            self.result_stream = torch.cuda.Stream(device=dev, priority=min(lo))
            self._chain_done = [torch.cuda.Event() for _ in range(nb)]
            self._exch_done = [None] * nb
            self._in_ready = [torch.cuda.Event() for _ in range(nb)]
            self.chain_streams = [torch.cuda.Stream(device=dev, priority=-1) for _ in range(nb)] if self.inflight > 1 else None
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
        if self.overlap:
            cur = torch.cuda.current_stream(self.dev)
            par = self.replays % self.nbuf
            run = cur
            if self.inflight > 1:                        # even / odd steps on their own streams, behind the caller's work so far
                run = self.chain_streams[par]
                self._in_ready[par].record(cur)
                run.wait_event(self._in_ready[par])
            if self._exch_done[par] is not None:          # buffers `par` were last read by the exchange of two steps ago
                run.wait_event(self._exch_done[par])
            with torch.cuda.stream(run):
                if labels is not None:
                    self.labels_all[par].copy_(labels, non_blocking=True)
                if x is not None:
                    self.inputs[slot].copy_(x, non_blocking=True)
                self.chain_graphs[par][slot].replay()
                self._chain_done[par].record(run)
            rs = self.result_stream
            rs.wait_event(self._chain_done[par])
            with torch.cuda.stream(rs):
                self.exch_graphs[par].replay()
                ev = self._exch_done[par] = self._exch_done[par] or torch.cuda.Event()
                ev.record(rs)
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
        if self.overlap and self.replays and self._exch_done[self._last] is not None:
            # exchanges run in step order on one stream and each follows its chain: the last one covers everything before
            torch.cuda.current_stream(self.dev).wait_event(self._exch_done[self._last])
        return self.out

    def input_consumed(self):
        """Event after which the input of the LAST step may be rewritten (its layer chain has read it); None = stream order
        of the current stream already says so."""
        return self._chain_done[self._last] if (self.overlap and self.replays) else None


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
            if parts is None:
                parts = [lsm.clone(), torch.ones_like(lsm), p.clone(), p * p, logits.clone(), klv.clone()]
                if information:
                    parts.append(h)
            else:
                m = torch.maximum(parts[0], lsm)
                parts[1] = parts[1] * (parts[0] - m).exp() + (lsm - m).exp()
                parts[0] = m
                parts[2] += p; parts[3] += p * p; parts[4] += logits; parts[5] += klv
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
    p_bar = (sum(plane(2)) / S).view(full)
    p2 = (sum(plane(3)) / S).view(full)
    pred = (sum(plane(4)) / S).view(full)
    epistemic = p2 - p_bar * p_bar                    # diag((p-pbar)^T (p-pbar))/T  (uncertainty_estimation.py:89-91)
    aleatoric = p_bar - p2                            # diag(diag(pbar) - p^T p / T)  (:94-95)
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
        cache = net.__dict__.setdefault("_mc_engines", {})
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


def evaluate(net, loader, num_ens: int, train_size: float, beta_type=0.1, epoch=None, num_epochs=None, group=None,
             seed: Optional[int] = None, inflight: int = 4, batch_shards: int = 1) -> dict:
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
    requires)."""
    dev = next(net.parameters()).device
    key = (int(num_ens), float(train_size), seed, id(group), int(inflight), int(batch_shards))
    ev = net.__dict__.setdefault("_mc_eval", {}).get(key)
    if ev is None:
        ev = net.__dict__["_mc_eval"][key] = {"acc": new_metrics(dev), "engines": {}, "seed": seed}
    acc, engines, nslots = ev["acc"], ev["engines"], max(2, int(inflight))
    cur = torch.cuda.current_stream(dev)
    acc.zero_()
    last, n = None, 0
    for x, y in loader:
        shape = (tuple(x.shape), x.dtype)
        e = engines.get(shape)
        if e is None:
            slots = [torch.zeros(x.shape, dtype=x.dtype, device=dev) for _ in range(nslots)]
            # the k-th engine built draws noise blocks k * 2^16, k * 2^16 + 1, ...: engines do not share noise
            eng = MCForward(net, slots[0], num_ens, group, with_labels=True, train_size=train_size, seed=ev["seed"],
                            static_inputs=slots, first_replay=len(engines) << 16, overlap=True, inflight=inflight,
                            batch_shards=batch_shards, metrics=acc)
            ev["seed"] = eng.seed               # every engine draws from the same seed
            e = engines[shape] = {"eng": eng, "slots": slots, "consumed": [None] * nslots, "steps": 0,
                                  "labels": [torch.zeros(x.shape[0], dtype=torch.int64, device=dev) for _ in range(nslots)],
                                  "pinned": [None] * nslots}
        eng = e["eng"]
        if last is not None and last is not eng:
            last.wait()                         # the accumulator takes the steps one after another
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
        eng(labels=e["labels"][s], slot=s)
        e["consumed"][s] = eng.input_consumed()
        e["steps"] += 1
        last, n = eng, n + 1
    if last is None:
        raise ValueError("evaluate: the loader yielded no batch")
    last.wait()
    m = read_metrics(acc)
    beta_sum = sum(get_beta(i - 1, n, beta_type, epoch, num_epochs) for i in range(n))
    m["valid_loss"] = (float(train_size) * m["sum_nll_step"] + beta_sum * m["klsum"]) / n
    m["valid_acc"] = m["sum_acc_step"] / n
    return m


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


def engine_forward_fn(net) -> Callable:
    """forward_fn for a net built on the engine: draws Monte-Carlo sample j (and leaves the training stream untouched)."""
    def fn(x, j):
        with Fn.mc_sample(j), torch.no_grad():
            return net(x)
    return fn


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
    reference's default) and Rb = world this is a data-parallel step."""

    def __init__(self, net, example_x, num_ens, train_size, group=None, seed=None, batch_shards: int = 1):
        super().__init__(net, example_x, num_ens, group=group, with_labels=True, train_size=train_size, seed=seed,
                         graph=False, fold=False, batch_shards=batch_shards)
        self.params = [p for p in net.parameters() if p.requires_grad]
        self.steps = 0

    def __call__(self, x, labels, beta: float = 0.0):
        from .graph import _STRIDE
        self.beta = float(beta)
        self.labels.copy_(labels, non_blocking=True)
        for p in self.params:
            p.grad = None
        logits, kls = [], []
        b0, b1 = self.rows
        xb = x[b0:b1]                                                  # this rank's row block
        for k, j in enumerate(self.ids):
            with Fn.mc_sample(j, self.seed, offset=self.steps * _STRIDE), Fn.first_image(b0):
                lg, kl = self.net(xb)                                  # autograd on: per-layer kernels (no fused chain)
            logits.append(lg)
            kls.append(kl)
            self.logits[k].copy_(lg.detach().reshape(self.nb, self.C))
        kl_ptr, n_kl = None, 0
        if self.ids:
            self.kl_one.copy_(kls[0].detach())
            kl_ptr, n_kl = Fn._ptr(self.kl_one), 1
        self._exchange(kl_ptr, n_kl)
        o = self.out
        if self.ids:
            S = float(self.num_ens)
            idx = self.labels[b0:b1].view(-1, 1)
            p_bar_y = o["log_outputs"][b0:b1].gather(1, idx).exp()          # p_bar[b, y_b] of the block's rows
            grads = []
            for lg in logits:
                sm = torch.softmax(lg.detach().float(), dim=1)
                w = sm.gather(1, idx) / (S * p_bar_y)
                onehot = torch.zeros_like(sm).scatter_(1, idx, 1.0)
                grads.append((-(self.train_size / self.B)) * w * (onehot - sm))
            # the KL does not depend on the rows: one block per sample group adds its gradient
            kl_t = [k_ for k_ in kls if torch.is_tensor(k_) and k_.requires_grad] if self.block == 0 else []
            kl_g = [torch.full_like(k_, self.beta / S) for k_ in kl_t]
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

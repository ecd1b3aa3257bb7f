"""CUDA-graph capture of a whole forward(+KL): the six layer kernels and the
interleaved aten activation/pool kernels become one graph launch, which is what
the problem size needs (SURVEY.md H1: the whole BBBAlexNet forward is ~18-29 us of
roofline time on an H100, i.e. the cost of its own kernel launches).

Noise under replay: kernel arguments are frozen at capture, so the Philox stream
is taken relative to a device scalar that a captured bbb_noise_advance kernel
moves forward at the head of every replay.
"""
from __future__ import annotations

import torch

from . import _lib
from . import functional as Fn

_STRIDE = 1 << 20      # stream ids one replay may consume (>= Bayesian layer calls per forward)


class GraphedForward:
    """logits, kl = GraphedForward(net, example_x)(x).  Replay r draws Philox streams
    first_stream + r*2^20 + (0, 1, 2, ...) -- reproducible from (seed, first_stream).

    ``static_inputs``: a list of device tensors the caller fills in place (e.g. the targets of its
    host->device copies).  One graph is captured per tensor, reading it directly, so ``self(slot=k)``
    runs the forward on ``static_inputs[k]`` without the staging copy that ``self(x)`` makes."""

    def __init__(self, net, example_x: torch.Tensor, first_stream: int = 0, warmup: int = 2, post=None,
                 static_inputs=None, ws_slot: int = 0):
        """post(logits, kl) -> outputs is captured behind the forward (e.g. the multi-GPU combine with
        its NCCL all-reduce), so a whole step is one graph launch.  ``ws_slot``: graphs that will be replayed
        concurrently on different streams need different slots (functional.workspace_slot) and keep warmup > 0,
        so that their private layer workspaces are created before the capture."""
        assert example_x.is_cuda
        self.net = net
        dev = example_x.device
        self.inputs = list(static_inputs) if static_inputs else [example_x.clone()]
        assert all(t.is_cuda and t.shape == example_x.shape and t.is_contiguous() for t in self.inputs)
        self.x = self.inputs[0]
        self.base = torch.zeros(1, dtype=torch.int64, device=dev)
        self.first_stream = int(first_stream)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.no_grad(), Fn.workspace_slot(ws_slot):
            for _ in range(warmup):
                with Fn.stream_base(self.base):
                    out = net(self.x)
                if post is not None:
                    post(*out)
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        from .modules import PriorGuard
        self.prior_guard = PriorGuard(net)        # the layers' prior buffers as the graphs read them
        self.graphs, self.outputs = [], []
        cap = torch.cuda.Stream(device=dev, priority=-1)     # GEMM chain above the parameter preps on the (default-priority) side streams
        for xin in self.inputs:
            graph = torch.cuda.CUDAGraph()
            n0 = _lib.launch_count()
            with torch.cuda.graph(graph, stream=cap), torch.no_grad(), Fn.workspace_slot(ws_slot):
                Fn.noise_advance(self.base, _STRIDE)
                with Fn.stream_base(self.base):
                    out = net(xin)
                if post is not None:
                    out = post(*out)
            self.kernels_per_replay = _lib.launch_count() - n0     # engine kernels captured in one graph
            self.graphs.append(graph)
            self.outputs.append(tuple(out))
        self.graph = self.graphs[0]
        self.logits, self.kl = self.outputs[0]
        self.replays = 0
        self.reset(self.first_stream)

    def reset(self, first_stream: int = 0):
        """Next replay uses streams first_stream + (0, 1, ...)."""
        self.base.fill_(int(first_stream) - _STRIDE)

    def __call__(self, x: torch.Tensor | None = None, non_blocking: bool = True, slot: int = 0):
        self.prior_guard.check("GraphedForward")
        if x is not None:
            self.inputs[slot].copy_(x, non_blocking=non_blocking)
        self.graphs[slot].replay()
        self.replays += 1
        return self.outputs[slot]

"""Cost of the information outputs (BBB_MC_INFO: expected entropy and mutual information) of the Monte-Carlo step on
one GPU, the default kernel and the INFO instantiation alternating window by window in one job:

* the exchange kernel alone, one rank: a captured graph of --launches back-to-back launches over fixed random logits,
  CUDA events, median per launch over --windows windows.  Shapes: C3-like (B=512, C=10, 10 samples), C4-like
  (B=1024, C=100, the 4 samples rank 0 of C4 holds) and C5 (B=2048, C=10, 100 samples);
* the whole C5 MCForward step (BBB3Conv3FC-10, 1x32x32, B=2048, 100 samples, LRT, uncertainty), one step at a time,
  with and without want_information.

Prints one JSON line per measurement with the GPU's name and power limit.

    python tools/mc_info_bench.py [--windows 7] [--launches 50] [--steps 5] [--no-step]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from tools.mc_fold_bench import gpu_info

SHAPES = {"C3-like": (512, 10, 10), "C4-like": (1024, 100, 4), "C5": (2048, 10, 100)}


def _events_ms(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def exchange_graph(dev, B, Cc, S, info, launches):
    """A captured graph of `launches` solo exchange launches (with uncertainty outputs) and the tensors it uses."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    lib = L.lib()
    flags = L.MC_MOMENTS | (L.MC_INFO if info else 0)
    logits = torch.randn(S, B, Cc, device=dev, generator=torch.Generator(device=dev).manual_seed(1)) * 4
    keep = {"logits": logits,
            "buf": torch.zeros(int(lib.bbb_mc_buffer_bytes(B, Cc, flags, 1)), dtype=torch.uint8, device=dev),
            "state": torch.zeros(int(lib.bbb_mc_state_bytes()), dtype=torch.uint8, device=dev),
            "lo": torch.empty(B, Cc, device=dev), "kl": torch.empty((), device=dev),
            "pred": torch.empty(B, Cc, device=dev), "epi": torch.empty(B, Cc, device=dev),
            "ale": torch.empty(B, Cc, device=dev), "ent": torch.empty(B, device=dev),
            "ee": torch.empty(B, device=dev) if info else None, "mi": torch.empty(B, device=dev) if info else None}
    peers = (C.c_void_p * 1)(keep["buf"].data_ptr())
    keep["peers"] = peers

    def launch():
        rc = lib.bbb_mc_exchange_info(
            Fn._ptr(logits), S, S, B, Cc, None, 0, flags, None, C.c_float(1.0), C.c_float(0.0), 0, 1, peers,
            Fn._ptr(keep["state"]), Fn._ptr(keep["lo"]), Fn._ptr(keep["kl"]), Fn._ptr(keep["pred"]),
            Fn._ptr(keep["epi"]), Fn._ptr(keep["ale"]), Fn._ptr(keep["ent"]), None, None, 0,
            Fn._ptr(keep["ee"]), Fn._ptr(keep["mi"]), Fn._stream(dev))
        L.check(rc, "bbb_mc_exchange_info")
    side = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(side):
        launch()                                       # eager once: module load
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        for _ in range(launches):
            launch()
    keep["graph"] = g
    return keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--launches", type=int, default=50, help="exchange launches per captured graph (one window)")
    ap.add_argument("--steps", type=int, default=5, help="C5 steps per window")
    ap.add_argument("--no-step", action="store_true", help="skip the whole C5 step")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    dev = torch.device("cuda:0")
    name, power = gpu_info()
    for sname, (B, Cc, S) in SHAPES.items():
        graphs = {info: exchange_graph(dev, B, Cc, S, info, args.launches) for info in (False, True)}
        times = {False: [], True: []}
        for info in (False, True):
            graphs[info]["graph"].replay()             # warm-up
        for _ in range(args.windows):
            for info in (False, True):
                times[info].append(1000.0 * _events_ms(graphs[info]["graph"].replay, args.launches))
        for info in (False, True):
            print(json.dumps({"what": "exchange kernel", "shape": sname, "batch": B, "classes": Cc, "local_samples": S,
                              "info": info, "us_per_launch_median": round(statistics.median(times[info]), 2),
                              "us_per_launch_min": round(min(times[info]), 2), "windows": args.windows,
                              "launches_per_window": args.launches, "gpu": name, "power_limit": power}), flush=True)
        del graphs
    if args.no_step:
        return
    from bench import build_net
    from pytorch_bayesiancnn_b200 import mc
    net = build_net("lrt", 10, dev, "auto", "3conv3fc", 1)
    x = torch.randn(2048, 1, 32, 32, device=dev)
    engines = {info: mc.MCForward(net, x, 100, want_uncertainty=True, want_information=info, seed=2024)
               for info in (False, True)}
    times = {False: [], True: []}

    def steps(eng):
        def run():
            for _ in range(args.steps):
                eng()
        return run
    for info in (False, True):
        steps(engines[info])()                         # warm-up
    for _ in range(args.windows):
        for info in (False, True):
            times[info].append(_events_ms(steps(engines[info]), args.steps))
    for info in (False, True):
        e = engines[info]
        print(json.dumps({"what": "MCForward step", "config": "C5", "batch": 2048, "mc_samples": 100, "info": info,
                          "layer_fold": e.layer_fold, "kernels_per_step": e.kernels_per_step,
                          "ms_per_step_median": round(statistics.median(times[info]), 3),
                          "ms_per_step_min": round(min(times[info]), 3), "windows": args.windows,
                          "steps_per_window": args.steps, "gpu": name, "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()

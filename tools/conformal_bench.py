"""Cost of the conformal log (bbb_mc_conformal_log) and of a split-conformal run on one GPU, variants alternating window
by window in one job, medians over --windows windows.

* kernel: the conformal-log kernel alone (randomised APS with a threshold set), a captured graph of --launches
  launches, at (B=512, C=10), (B=1024, C=100) and (B=2048, C=1000);
* inflight: the MCForward step with four in flight (overlap=True, inflight=4, resident batches, labels), without and
  with a conformal log: headline-like (BBBAlexNet-10, B=512, 1 sample), C3-like (BBBAlexNet-10, B=512, 10 samples)
  and C5 (BBB3Conv3FC-10, B=2048, 100 samples);
* conformal: calibrate on --batches host batches and predict on --batches more (randomised APS, alpha = 0.1): the
  reference-style loop (one serial step per batch, ``.cpu()`` of log_outputs, scores, quantile and sets in numpy)
  against mc.conformal.  Both draw the same noise and the same u, and must pick the same sets (classes within 1e-12
  of q_hat excepted).  Both build their engines in a first, untimed run.

Prints one JSON line per measurement with the GPU's name and power limit.

    python tools/conformal_bench.py [--windows 7] [--launches 50] [--inflight-steps 100] [--batches 10]
                                    [--only kernel,inflight,conformal] [--workloads headline,C3]
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from tools.mc_fold_bench import gpu_info
from tools.mc_info_bench import _events_ms
from tests import conformal_ref as R

WORKLOADS = {"headline": ("alexnet", 3, 512, 1), "C3": ("alexnet", 3, 512, 10), "C5": ("3conv3fc", 1, 2048, 100)}
KERNEL_SHAPES = ((512, 10), (1024, 100), (2048, 1000))
ALPHA, SEED = 0.1, 2024


def kernel_bench(args, dev, gpu, power):
    from pytorch_bayesiancnn_b200 import mc
    for B, Cc in KERNEL_SHAPES:
        g = torch.Generator(device=dev).manual_seed(1)
        lo = torch.log_softmax(torch.randn(B, Cc, device=dev, generator=g) * 3, 1)
        y = torch.randint(0, Cc, (B,), device=dev, generator=g)
        log = mc.ConformalLog(dev, args.launches * B, Cc, method="aps", seed=1)
        log.set_threshold(0.9)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            log.append(lo, y)
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=side):
            log.reset()                                  # every replay writes all its entries
            for _ in range(args.launches):
                log.append(lo, y)
        gr.replay()
        times = [1000.0 * _events_ms(gr.replay, args.launches) for _ in range(args.windows)]
        torch.cuda.synchronize()
        assert len(log) == args.launches * B and log.dropped == 0
        print(json.dumps({"what": "conformal-log kernel", "batch": B, "classes": Cc,
                          "us_per_launch_median": round(statistics.median(times), 2),
                          "us_per_launch_min": round(min(times), 2), "windows": args.windows,
                          "launches_per_window": args.launches, "gpu": gpu, "power_limit": power}), flush=True)


def inflight_bench(args, dev, gpu, power):
    from bench import build_net
    from pytorch_bayesiancnn_b200 import mc
    for name, (key, inputs, B, S) in WORKLOADS.items():
        net = build_net("lrt", 10, dev, "auto", key, inputs)
        xs = [torch.randn(B, inputs, 32, 32, device=dev) for _ in range(4)]
        y = torch.randint(0, 10, (B,), device=dev)
        steps = args.inflight_steps if name != "C5" else max(2, args.inflight_steps // 10)
        logs = {False: None, True: mc.ConformalLog(dev, steps * B, 10, method="aps", seed=1)}
        logs[True].set_threshold(0.9)
        engines = {m: mc.MCForward(net, xs[0], S, with_labels=True, seed=SEED, static_inputs=xs, overlap=True,
                                   inflight=4, conformal=logs[m]) for m in (False, True)}

        def run(m):
            def go():
                if logs[m] is not None:
                    logs[m].reset()
                for i in range(steps):
                    engines[m](labels=y, slot=i % len(xs))
                engines[m].wait()
            return go
        for m in (False, True):
            run(m)()
        times = {False: [], True: []}
        for _ in range(args.windows):
            for m in (False, True):
                times[m].append(_events_ms(run(m), steps))
        assert len(logs[True]) == steps * B and logs[True].dropped == 0
        same = all(torch.equal(engines[False].out[k], engines[True].out[k]) for k in engines[False].out)
        for m in (False, True):
            print(json.dumps({"what": "MCForward step in flight", "workload": name, "batch": B, "mc_samples": S,
                              "inflight": 4, "conformal_log": m, "kernels_per_step": engines[m].kernels_per_step,
                              "ms_per_step_median": round(statistics.median(times[m]), 4),
                              "ms_per_step_min": round(min(times[m]), 4), "steps_per_window": steps,
                              "outputs_bitwise_equal": same, "windows": args.windows, "gpu": gpu,
                              "power_limit": power}), flush=True)
        del engines, net


def reference_conformal(net, S, cal, test, dev, cache):
    """The loop a user writes without the log: per batch one serial step and a host copy of log_outputs; randomised
    APS scores, the quantile and the sets in numpy.  The engines (one per set, as mc.conformal's evaluate keeps one
    per log) and u (stream 0 for calibration, 1 for test) are mc.conformal's."""
    from pytorch_bayesiancnn_b200 import functional as Fn, mc
    seed = SEED & ((1 << 64) - 1)
    out = {}
    for stream, (role, batches) in enumerate((("calibration", cal), ("test", test))):
        eng = cache.get(role)
        if eng is None:
            eng = cache[role] = mc.MCForward(net, batches[0][0].to(dev), S, with_labels=True, seed=SEED)
        los, ys = [], []
        for x, y in batches:
            los.append(eng(x.to(dev), y.to(dev))["log_outputs"].cpu().numpy())
            ys.append(y.numpy())
        lo, y = np.concatenate(los), np.concatenate(ys)
        E = R.scores(lo, R.APS, True, u=R.u_of(seed, stream, np.arange(lo.shape[0])))
        out[role] = (E, y)
    E, y = out["calibration"]
    q = R.quantile(E[np.arange(y.size), y], ALPHA)
    E, y = out["test"]
    sets = E <= q
    return {"qhat": q, "sets": sets, "E": E, "coverage": float(sets[np.arange(y.size), y].mean())}


def conformal_bench(args, dev, gpu, power):
    from bench import build_net
    from pytorch_bayesiancnn_b200 import mc
    for name in args.workloads.split(","):
        key, inputs, B, S = WORKLOADS[name]
        g = torch.Generator().manual_seed(0)
        cal, test = [[(torch.rand(B, inputs, 32, 32, generator=g), torch.randint(0, 10, (B,), generator=g))
                      for _ in range(args.batches)] for _ in range(2)]
        net = build_net("lrt", 10, dev, "auto", key, inputs)
        cache = {}

        def ref():
            return reference_conformal(net, S, cal, test, dev, cache)

        def dev_cf():
            r = mc.conformal(net, cal, test, S, alpha=ALPHA, method="aps", seed=SEED)
            return {"qhat": float(r["qhat"]), "sets": r["logs"]["test"]["sets"].cpu().numpy(),
                    "coverage": r["test"]["coverage"]}
        res = {"reference": ref(), "conformal": dev_cf()}
        a, b = res["reference"], res["conformal"]
        near = np.abs(a["E"] - a["qhat"]) <= 1e-12
        same_sets = bool(np.array_equal(a["sets"] | near, b["sets"] | near))
        times = {"reference": [], "conformal": []}
        for _ in range(args.windows):
            for k, fn in (("reference", ref), ("conformal", dev_cf)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res[k] = fn()
                torch.cuda.synchronize()
                times[k].append(1000.0 * (time.perf_counter() - t0))
        for k in times:
            print(json.dumps({"what": "split conformal: calibrate and predict", "workload": name, "version": k,
                              "batch": B, "mc_samples": S, "batches_per_set": args.batches,
                              "ms_median": round(statistics.median(times[k]), 3), "ms_min": round(min(times[k]), 3),
                              "windows": args.windows, "qhat": res[k]["qhat"], "coverage": res[k]["coverage"],
                              "same_sets": same_sets, "gpu": gpu, "power_limit": power}), flush=True)
        del net, cache


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--launches", type=int, default=50, help="conformal-log launches per captured graph (one window)")
    ap.add_argument("--inflight-steps", type=int, default=100, help="steps per window of the in-flight arm (C5: / 10)")
    ap.add_argument("--batches", type=int, default=10, help="batches per set of the conformal run")
    ap.add_argument("--only", default="kernel,inflight,conformal")
    ap.add_argument("--workloads", default="headline,C3")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    dev = torch.device("cuda:0")
    gpu, power = gpu_info()
    only = args.only.split(",")
    if "kernel" in only:
        kernel_bench(args, dev, gpu, power)
    if "inflight" in only:
        inflight_bench(args, dev, gpu, power)
    if "conformal" in only:
        conformal_bench(args, dev, gpu, power)


if __name__ == "__main__":
    main()

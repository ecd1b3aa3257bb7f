"""Cost of the per-image score log (bbb_mc_score_log) and of an out-of-distribution evaluation on one GPU, variants
alternating window by window in one job, medians over --windows windows.

* kernel: the score-log kernel alone, a captured graph of --launches launches, at the headline-like (B=512, C=10),
  C4-like (B=1024, C=100) and C5 (B=2048, C=10) shapes;
* inflight: the MCForward step with four in flight (overlap=True, inflight=4, resident batches, labels, uncertainty
  and information outputs), without and with a score log: headline-like (BBBAlexNet-10, B=512, 1 sample), C3-like
  (BBBAlexNet-10, B=512, 10 samples) and C5 (BBB3Conv3FC-10, B=2048, 100 samples);
* ood: a whole OOD evaluation of two synthetic sets of --batches host batches each (in-distribution noise against
  shifted noise), every score of mc.OOD_SCORES: the reference-style loop (uncertainty_estimation.py run over the sets:
  one serial step per batch, ``.cpu()`` of its outputs, scores and metrics in numpy) against mc.detect_ood.  Both
  build their engines in a first, untimed run.

Prints one JSON line per measurement with the GPU's name and power limit.

    python tools/ood_bench.py [--windows 7] [--launches 50] [--inflight-steps 100] [--batches 10]
                              [--only kernel,inflight,ood] [--ood-workloads headline,C3]
"""
import argparse
import ctypes as C
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

WORKLOADS = {"headline": ("alexnet", 3, 512, 1), "C3": ("alexnet", 3, 512, 10), "C5": ("3conv3fc", 1, 2048, 100)}
KERNEL_SHAPES = {"headline-like": (512, 10), "C4-like": (1024, 100), "C5": (2048, 10)}


def kernel_bench(args, dev, gpu, power):
    from pytorch_bayesiancnn_b200 import mc
    for name, (B, Cc) in KERNEL_SHAPES.items():
        g = torch.Generator(device=dev).manual_seed(1)
        lo = torch.log_softmax(torch.randn(B, Cc, device=dev, generator=g), 1)
        vec = [torch.rand(B, device=dev, generator=g) for _ in range(3)]
        epi = torch.rand(B, Cc, device=dev, generator=g)
        y = torch.randint(0, Cc, (B,), device=dev, generator=g)
        log = mc.ScoreLog(dev, args.launches * B)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            log.append(lo, *vec, epi, y)
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=side):
            log.reset()                                  # every replay writes all its entries
            for _ in range(args.launches):
                log.append(lo, *vec, epi, y)
        gr.replay()
        times = [1000.0 * _events_ms(gr.replay, args.launches) for _ in range(args.windows)]
        torch.cuda.synchronize()
        assert len(log) == args.launches * B and log.dropped == 0
        print(json.dumps({"what": "score-log kernel", "shape": name, "batch": B, "classes": Cc,
                          "us_per_launch_median": round(statistics.median(times), 2), "us_per_launch_min": round(min(times), 2),
                          "windows": args.windows, "launches_per_window": args.launches, "gpu": gpu, "power_limit": power}),
              flush=True)


def inflight_bench(args, dev, gpu, power):
    from bench import build_net
    from pytorch_bayesiancnn_b200 import mc
    for name, (key, inputs, B, S) in WORKLOADS.items():
        net = build_net("lrt", 10, dev, "auto", key, inputs)
        xs = [torch.randn(B, inputs, 32, 32, device=dev) for _ in range(4)]
        y = torch.randint(0, 10, (B,), device=dev)
        steps = args.inflight_steps if name != "C5" else max(2, args.inflight_steps // 10)
        logs = {False: None, True: mc.ScoreLog(dev, steps * B)}
        engines = {m: mc.MCForward(net, xs[0], S, with_labels=True, want_uncertainty=True, want_information=True,
                                   seed=2024, static_inputs=xs, overlap=True, inflight=4, score_log=logs[m])
                   for m in (False, True)}

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
                              "inflight": 4, "score_log": m, "kernels_per_step": engines[m].kernels_per_step,
                              "ms_per_step_median": round(statistics.median(times[m]), 4),
                              "ms_per_step_min": round(min(times[m]), 4), "steps_per_window": steps,
                              "outputs_bitwise_equal": same, "windows": args.windows, "gpu": gpu,
                              "power_limit": power}), flush=True)
        del engines, net


def _np_auroc(neg, pos):
    from scipy.stats import rankdata
    r = rankdata(np.concatenate([neg, pos]))
    return (r[neg.size:].sum() - pos.size * (pos.size + 1) / 2) / (pos.size * neg.size)


def _np_ap(s, pos):
    order = np.argsort(-s, kind="stable")
    v, p = s[order], pos[order].astype(np.float64)
    ends = np.r_[np.nonzero(np.diff(v))[0], v.size - 1]
    tp, fp = np.cumsum(p)[ends], np.cumsum(1 - p)[ends]
    rec = tp / tp[-1]
    return float((np.diff(np.r_[0.0, rec]) * tp / (tp + fp)).sum())


def _np_ood(si, so):
    s = np.concatenate([si, so])
    out = np.r_[np.zeros(si.size, bool), np.ones(so.size, bool)]
    order = np.argsort(-s, kind="stable")
    v, p = s[order], out[order].astype(np.float64)
    ends = np.r_[np.nonzero(np.diff(v))[0], v.size - 1]
    tpr, fpr = np.cumsum(p)[ends] / so.size, np.cumsum(1 - p)[ends] / si.size
    return {"auroc": _np_auroc(si, so), "aupr_out": _np_ap(s, out), "aupr_in": _np_ap(-s, ~out),
            "fpr_at_95_tpr": float(fpr[tpr >= 0.95].min())}


def reference_ood(engines, in_b, out_b, dev):
    """uncertainty_estimation.py's comparison over whole sets: per batch one serial step and a host copy of its
    outputs; scores and OOD metrics in numpy on the host."""
    from pytorch_bayesiancnn_b200 import mc
    scores = {}
    for role, batches in (("in", in_b), ("out", out_b)):
        parts = {nm: [] for nm in mc.OOD_SCORES}
        for x, y in batches:
            o = engines[tuple(x.shape)](x.to(dev), y.to(dev))
            lo = o["log_outputs"].cpu().numpy()
            parts["confidence"].append(-np.exp(lo.max(1)))
            for nm in ("entropy", "mutual_info", "expected_entropy"):
                parts[nm].append(o[nm].cpu().numpy())
            parts["epistemic"].append(o["epistemic"].cpu().numpy().astype(np.float64).sum(1))
        scores[role] = {nm: np.concatenate(v).astype(np.float64) for nm, v in parts.items()}
    return {nm: _np_ood(scores["in"][nm], scores["out"][nm]) for nm in mc.OOD_SCORES}


def ood_bench(args, dev, gpu, power):
    from bench import build_net
    from pytorch_bayesiancnn_b200 import mc
    for name in args.ood_workloads.split(","):
        key, inputs, B, S = WORKLOADS[name]
        g = torch.Generator().manual_seed(0)
        sets = [[(torch.rand(B, inputs, 32, 32, generator=g) + shift, torch.randint(0, 10, (B,), generator=g))
                 for _ in range(args.batches)] for shift in (0.0, 2.0)]
        net = build_net("lrt", 10, dev, "auto", key, inputs)
        engines = {(B, inputs, 32, 32): mc.MCForward(net, sets[0][0][0].to(dev), S, with_labels=True,
                                                     want_uncertainty=True, want_information=True, seed=2024)}

        def ref():
            return reference_ood(engines, sets[0], sets[1], dev)

        def dev_ood():
            return mc.detect_ood(net, sets[0], sets[1], S, score=None, seed=2024)["ood"]
        res = {"reference": ref(), "detect_ood": dev_ood()}
        times = {"reference": [], "detect_ood": []}
        for _ in range(args.windows):
            for k, fn in (("reference", ref), ("detect_ood", dev_ood)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res[k] = fn()
                torch.cuda.synchronize()
                times[k].append(1000.0 * (time.perf_counter() - t0))
        for k in times:
            print(json.dumps({"what": "OOD evaluation of two sets", "workload": name, "version": k, "batch": B,
                              "mc_samples": S, "batches_per_set": args.batches,
                              "ms_median": round(statistics.median(times[k]), 3), "ms_min": round(min(times[k]), 3),
                              "windows": args.windows,
                              "auroc": {nm: round(float(v["auroc"]), 6) for nm, v in res[k].items()},
                              "gpu": gpu, "power_limit": power}), flush=True)
        del engines, net


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--launches", type=int, default=50, help="score-log launches per captured graph (one window)")
    ap.add_argument("--inflight-steps", type=int, default=100, help="steps per window of the in-flight arm (C5: / 10)")
    ap.add_argument("--batches", type=int, default=10, help="batches per set of the OOD evaluation")
    ap.add_argument("--only", default="kernel,inflight,ood")
    ap.add_argument("--ood-workloads", default="headline,C3")
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
    if "ood" in only:
        ood_bench(args, dev, gpu, power)


if __name__ == "__main__":
    main()

"""Nets without a weight mask, with an all-ones mask and 95 % pruned (prune_by_snr), on one GPU: ms per step of
  - the headline BBBAlexNet LRT B=512 Monte-Carlo step (mc.MCForward, captured), one step at a time and four in flight,
  - the C3-like folded step (BBBAlexNet LRT, B=512, 10 samples in one pass of the fused chain),
  - the C5 step (BBB3Conv3FC LRT, B=2048, 100 samples, uncertainty),
  - the BBBLeNet LRT training step with the samples folded (MCTrainStep(fold=True) + Adam, B=256, 10 samples),
and the device time of the weight-prep kernels per headline step (torch.profiler, a run of its own after the timings).
The masked nets are copies of the unmasked one (same parameters).  The three modes alternate window by window within one
job; the median of the windows is reported with the GPU's name and power limit.  One JSON line per (config, mode).
Pruning does not make a step faster: the kernels still multiply the zeros.  What this measures is the cost of reading
the mask (one byte per parameter, beside the eight of mu and rho) in the weight preps.

    python tools/mask_bench.py [--steps 20] [--windows 7] [--configs headline,headline_inflight4,C3,C5,LeNet_train]
"""
import argparse
import copy
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from tools.mc_fold_bench import gpu_info

CONFIGS = {
    "headline": dict(net="alexnet", inputs=3, batch=512, samples=1, uncertainty=False, inflight=1, train=False),
    "headline_inflight4": dict(net="alexnet", inputs=3, batch=512, samples=1, uncertainty=False, inflight=4, train=False),
    "C3": dict(net="alexnet", inputs=3, batch=512, samples=10, uncertainty=False, inflight=1, train=False),
    "C5": dict(net="3conv3fc", inputs=1, batch=2048, samples=100, uncertainty=True, inflight=1, train=False, steps=2),
    "LeNet_train": dict(net="lenet", inputs=3, batch=256, samples=10, uncertainty=False, inflight=1, train=True),
}
MODES = ("none", "ones", "pruned95")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--math", default="auto")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from bench import build_net
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import mc
    dev = torch.device("cuda:0")
    name, power = gpu_info()
    for cname in args.configs.split(","):
        cfg = CONFIGS[cname]
        B, S = cfg["batch"], cfg["samples"]
        steps = cfg.get("steps", args.steps)
        x = torch.randn(B, cfg["inputs"], 32, 32, device=dev)
        y = torch.randint(0, 10, (B,), device=dev)
        base = build_net("lrt", 10, dev, args.math, cfg["net"], cfg["inputs"])
        runs = {}
        for m in MODES:
            net = copy.deepcopy(base)
            if m == "ones":
                for layer in net.modules():
                    if hasattr(layer, "W_mu"):
                        layer.set_weight_mask(torch.ones_like(layer.W_mu, dtype=torch.bool))
            elif m == "pruned95":
                bbb.prune_by_snr(net, 0.95)
            if cfg["train"]:
                eng = mc.MCTrainStep(net, x, S, train_size=50000.0, seed=2024, fold=True)
                opt = torch.optim.Adam(eng.params, lr=1e-3)
                fn = lambda eng=eng, opt=opt: (eng(x, y, beta=0.1), opt.step())
            else:
                eng = mc.MCForward(net, x, S, want_uncertainty=cfg["uncertainty"], seed=2024, static_inputs=[x],
                                   overlap=cfg["inflight"] > 1, inflight=cfg["inflight"])
                fn = lambda eng=eng: eng(slot=0)
            runs[m] = (eng, fn)
        times = {m: [] for m in MODES}

        def window(m, n):
            eng, fn = runs[m]
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                fn()
            if getattr(eng, "overlap", False):
                eng.wait()
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / n

        for m in MODES:
            window(m, 3)                                  # warm-up: graphs, workspaces, allocator
        for _ in range(args.windows):
            for m in MODES:
                times[m].append(window(m, steps))
        for m in MODES:
            print(json.dumps({"config": cname, "net": cfg["net"], "variant": "lrt", "math": args.math, "batch": B,
                              "mc_samples": S, "inflight": cfg["inflight"], "train": cfg["train"], "mask": m,
                              "ms_per_step_median": round(statistics.median(times[m]), 4),
                              "ms_per_step_min": round(min(times[m]), 4), "windows": args.windows,
                              "steps_per_window": steps, "gpu": name, "power_limit": power}), flush=True)
        if cname == "headline":
            # device time of the weight-prep kernels per step (profiled after the timings, so they are not disturbed)
            for m in MODES:
                fn = runs[m][1]
                n = 10
                torch.cuda.synchronize()
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for _ in range(n):
                        fn()
                    torch.cuda.synchronize()
                per = {}
                for ev in prof.key_averages():
                    if "prep_kernel" in ev.key:
                        k = ev.key.split("<")[0].replace("void bbb::", "")
                        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
                        per[k] = per.get(k, 0.0) + t / 1000.0 / n
                print(json.dumps({"config": cname, "mask": m, "prep_ms_per_step": {k: round(v, 4) for k, v in per.items()},
                                  "prep_ms_per_step_total": round(sum(per.values()), 4), "gpu": name,
                                  "power_limit": power}), flush=True)
        del runs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

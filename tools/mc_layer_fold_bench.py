"""ms per Monte-Carlo step of a net the fused chain does not take (BBB3Conv3FC, BBBLeNet) with its samples folded into
grouped passes of the per-layer tensor-core kernel vs run one by one: BASELINE config C5 (BBB3Conv3FC-10, 1x32x32,
B=2048, 100 samples, uncertainty outputs) with lrt and with bbb layers, and BBBLeNet-10 (1x32x32, B=256, 10 samples)
with both variants, on one GPU.  The engines alternate window by window; the median of the windows is reported with
kernels per step and the GPU's name and power limit, one step at a time and with four steps in flight.  Prints one JSON
line per (config, engine).

    python tools/mc_layer_fold_bench.py [--steps 10] [--windows 7] [--configs C5,C5bbb,LeNet,LeNetbbb]
                                        [--groups auto,off] [--flight 1,4]

--groups: the folded engines to compare, `off` = fold=False (sample by sample), `auto` = the default group size
(mc.LAYER_FOLD_BUDGET), an integer = MCForward(fold_group=...).
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from tools.mc_fold_bench import gpu_info

CONFIGS = {
    "C5": dict(net="3conv3fc", variant="lrt", batch=2048, samples=100),
    "C5bbb": dict(net="3conv3fc", variant="bbb", batch=2048, samples=100),
    "LeNet": dict(net="lenet", variant="lrt", batch=256, samples=10),
    "LeNetbbb": dict(net="lenet", variant="bbb", batch=256, samples=10),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--configs", default="C5,C5bbb,LeNet,LeNetbbb")
    ap.add_argument("--groups", default="auto,off")
    ap.add_argument("--flight", default="1,4", help="steps in flight: 1 = one at a time, k > 1 = overlap with k")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from bench import build_net
    from pytorch_bayesiancnn_b200 import mc
    dev = torch.device("cuda:0")
    name, power = gpu_info()
    modes = args.groups.split(",")
    for cname in args.configs.split(","):
        cfg = CONFIGS[cname]
        B, S = cfg["batch"], cfg["samples"]
        net = build_net(cfg["variant"], 10, dev, "auto", cfg["net"], 1)
        xs = [torch.randn(B, 1, 32, 32, device=dev) for _ in range(4)]
        for inflight in [int(v) for v in args.flight.split(",")]:
            overlap = inflight > 1
            engines = {}
            for m in modes:
                kw = dict(fold=m != "off", fold_group=int(m) if m not in ("off", "auto") else None)
                engines[m] = mc.MCForward(net, xs[0], S, want_uncertainty=True, seed=2024, static_inputs=xs,
                                          overlap=overlap, inflight=inflight, **kw)
                assert (engines[m].layer_fold is None) == (m == "off"), (cname, m)
            times = {m: [] for m in modes}

            def window(eng, n):
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for k in range(n):
                    eng(slot=k % len(xs))
                eng.wait()
                e1.record()
                torch.cuda.synchronize()
                return e0.elapsed_time(e1) / n

            for m in modes:
                window(engines[m], 3)                     # warm-up
            for _ in range(args.windows):
                for m in modes:
                    times[m].append(window(engines[m], args.steps))
            for m in modes:
                e = engines[m]
                print(json.dumps({"config": cname, "net": cfg["net"], "variant": cfg["variant"], "batch": B,
                                  "mc_samples": S, "fold": m, "layer_fold": e.layer_fold, "inflight": inflight,
                                  "kernels_per_step": e.kernels_per_step,
                                  "ms_per_step_median": round(statistics.median(times[m]), 3),
                                  "ms_per_step_min": round(min(times[m]), 3), "windows": args.windows,
                                  "steps_per_window": args.steps, "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 1),
                                  "gpu": name, "power_limit": power}), flush=True)
            del engines
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

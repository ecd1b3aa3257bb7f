"""ms per Monte-Carlo step of a BBB (weight-space sampling) net with its samples folded into one pass of the fused
chain vs run one by one: BASELINE configs C3 (BBBAlexNet-10, B=512, 10 samples) and C4 (BBBAlexNet-100, B=1024,
25 samples) on one GPU, with the variant set to bbb.  The two engines alternate window by window; the median window
is reported with the GPU's name and power limit.  Prints one JSON line per (config, engine mode).

    python tools/mc_fold_bench.py [--steps 20] [--windows 7] [--configs C3,C4]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

CONFIGS = {"C3": dict(classes=10, batch=512, samples=10), "C4": dict(classes=100, batch=1024, samples=25)}


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in q.split(",")]
    except Exception:                                     # the figures still stand; the label says what is missing
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--configs", default="C3,C4")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from bench import build_net
    from pytorch_bayesiancnn_b200 import mc
    dev = torch.device("cuda:0")
    name, power = gpu_info()
    for cname in args.configs.split(","):
        cfg = CONFIGS[cname]
        B, S = cfg["batch"], cfg["samples"]
        net = build_net("bbb", cfg["classes"], dev, "bf16")
        xs = [torch.randn(B, 3, 32, 32, device=dev) for _ in range(4)]
        for overlap, inflight in ((False, 1), (True, 4)):
            engines = {fold: mc.MCForward(net, xs[0], S, seed=2024, static_inputs=xs, fold=fold, overlap=overlap,
                                          inflight=inflight) for fold in (True, False)}
            assert engines[True].fold_steps is not None and engines[False].fold_steps is None
            times = {True: [], False: []}

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

            for fold in (True, False):
                window(engines[fold], 5)                  # warm-up
            for _ in range(args.windows):
                for fold in (True, False):
                    times[fold].append(window(engines[fold], args.steps))
            for fold in (True, False):
                print(json.dumps({"config": cname, "variant": "bbb", "batch": B, "mc_samples": S, "fold": fold,
                                  "overlap": overlap, "inflight": inflight,
                                  "kernels_per_step": engines[fold].kernels_per_step,
                                  "ms_per_step_median": round(statistics.median(times[fold]), 3),
                                  "ms_per_step_min": round(min(times[fold]), 3), "windows": args.windows,
                                  "steps_per_window": args.steps, "gpu": name, "power_limit": power}), flush=True)
            del engines
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

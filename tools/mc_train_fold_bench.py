"""ms per training step (MCTrainStep + Adam) with the Monte-Carlo samples folded into grouped passes, forward and
backward (fold=True), against the sample loop (fold=False), on one GPU: BBBLeNet LRT (3x32x32, B=256, 10 samples),
BBB3Conv3FC LRT (1x32x32, B=256, 10 samples) and BBBAlexNet LRT (3x32x32, B=512, 4 samples).  The two steps alternate
window by window within one job; the median of the windows is reported with the engine kernels per step
(bbb.launch_count()) and the GPU's name and power limit.  Prints one JSON line per (config, mode).

    python tools/mc_train_fold_bench.py [--steps 10] [--windows 7] [--configs LeNet,3Conv3FC,AlexNet] [--math auto]
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
    "LeNet": dict(net="lenet", inputs=3, batch=256, samples=10),
    "3Conv3FC": dict(net="3conv3fc", inputs=1, batch=256, samples=10),
    "AlexNet": dict(net="alexnet", inputs=3, batch=512, samples=4),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--configs", default="LeNet,3Conv3FC,AlexNet")
    ap.add_argument("--math", default="auto")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from bench import build_net
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import mc
    dev = torch.device("cuda:0")
    name, power = gpu_info()
    modes = ("fold", "loop")
    for cname in args.configs.split(","):
        cfg = CONFIGS[cname]
        B, S = cfg["batch"], cfg["samples"]
        x = torch.rand(B, cfg["inputs"], 32, 32, device=dev)
        y = torch.randint(0, 10, (B,), device=dev)
        runs = {}
        for m in modes:
            # one net and optimizer per mode: each trains on its own from the same starting point
            net = build_net("lrt", 10, dev, args.math, cfg["net"], cfg["inputs"])
            step = mc.MCTrainStep(net, x, S, train_size=50000.0, seed=2024, fold=m == "fold")
            assert (step.layer_fold is None) == (m == "loop"), (cname, m)
            runs[m] = (step, torch.optim.Adam(step.params, lr=1e-3), [], [0])
        times = {m: [] for m in modes}

        def window(m, n):
            step, opt, _, kern = runs[m]
            torch.cuda.synchronize()
            k0 = bbb.launch_count()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                step(x, y, beta=0.1)
                opt.step()
            e1.record()
            torch.cuda.synchronize()
            kern[0] = (bbb.launch_count() - k0) // n
            return e0.elapsed_time(e1) / n

        for m in modes:
            window(m, 3)                                  # warm-up: workspaces, allocator, Adam state
        for _ in range(args.windows):
            for m in modes:
                times[m].append(window(m, args.steps))
        for m in modes:
            step = runs[m][0]
            print(json.dumps({"config": cname, "net": cfg["net"], "variant": "lrt", "math": args.math, "batch": B,
                              "mc_samples": S, "mode": m, "layer_fold": step.layer_fold,
                              "kernels_per_step": runs[m][3][0],
                              "ms_per_step_median": round(statistics.median(times[m]), 3),
                              "ms_per_step_min": round(min(times[m]), 3), "windows": args.windows,
                              "steps_per_window": args.steps, "gpu": name, "power_limit": power}), flush=True)
        del runs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

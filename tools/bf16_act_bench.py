"""fp32 against bf16 activations on one GPU: the same workload fed an fp32 input and its bf16 copy (BBB_DTYPE_BF16 on the
tensor-core layer kernel, bf16 aten activations and pools between the layers), engines alternating window by window in
one job; the median of the windows is reported with the GPU's name and power limit.

  layer      one sampled forward of the per-layer path (no grad, one MC sample): BBBLeNet LRT (3x32x32, B=256) and
             BBB3Conv3FC LRT (1x32x32, B=2048)
  C5         the C5-shaped MCForward step (BBB3Conv3FC LRT, 1x32x32, B=2048, 100 samples, uncertainty outputs; captured)
  train      MCTrainStep(fold=True) + Adam: BBBLeNet LRT (3x32x32) and BBB3Conv3FC LRT (1x32x32), B=256, 10 samples,
             with the peak of torch.cuda.max_memory_allocated during a step (above what was allocated before it)

Prints one JSON line per (workload, activation dtype).

    python tools/bf16_act_bench.py [--windows 7] [--only layer,C5,train]
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from tools.mc_fold_bench import gpu_info

DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16}


def _alternate(fns, windows):
    """fns: {mode: callable() -> ms per iteration of one window}; one warm-up window each, then `windows` rounds."""
    for f in fns.values():
        f()
    times = {m: [] for m in fns}
    for _ in range(windows):
        for m, f in fns.items():
            times[m].append(f())
    return times


def _events(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--layer-iters", type=int, default=20)
    ap.add_argument("--c5-steps", type=int, default=5)
    ap.add_argument("--train-steps", type=int, default=10)
    ap.add_argument("--only", default="layer,C5,train")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from bench import build_net
    from pytorch_bayesiancnn_b200 import mc
    if not torch.cuda.is_available():
        raise SystemExit("bf16_act_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    gpu, power = gpu_info()
    only = args.only.split(",")
    common = {"windows": args.windows, "gpu": gpu, "power_limit": power}

    def emit(d, times):
        for m, t in times.items():
            print(json.dumps({**d, "act_dtype": m, "ms_median": round(statistics.median(t), 3),
                              "ms_min": round(min(t), 3), **common}), flush=True)

    if "layer" in only:
        for key, inputs, B in (("lenet", 3, 256), ("3conv3fc", 1, 2048)):
            net = build_net("lrt", 10, dev, "auto", key, inputs)
            x32 = torch.rand(B, inputs, 32, 32, device=dev)
            xs = {m: x32.to(dt) for m, dt in DTYPES.items()}

            def fwd(m):
                def go():
                    with torch.no_grad():
                        net(xs[m])
                return lambda: _events(go, args.layer_iters)
            times = _alternate({m: fwd(m) for m in DTYPES}, args.windows)
            emit({"what": "per-layer forward", "net": key, "variant": "lrt", "batch": B, "iters": args.layer_iters},
                 times)
            del net
            torch.cuda.empty_cache()

    if "C5" in only:
        net = build_net("lrt", 10, dev, "auto", "3conv3fc", 1)
        x32 = torch.rand(2048, 1, 32, 32, device=dev)
        engs = {m: mc.MCForward(net, x32.to(dt), 100, want_uncertainty=True, seed=7) for m, dt in DTYPES.items()}
        times = _alternate({m: (lambda e=e: _events(e, args.c5_steps)) for m, e in engs.items()}, args.windows)
        emit({"what": "MCForward step", "config": "C5", "net": "3conv3fc", "variant": "lrt", "batch": 2048,
              "mc_samples": 100, "layer_fold": engs["fp32"].layer_fold, "steps": args.c5_steps}, times)
        del engs, net
        torch.cuda.empty_cache()

    if "train" in only:
        for key, inputs in (("lenet", 3), ("3conv3fc", 1)):
            B, S = 256, 10
            x32 = torch.rand(B, inputs, 32, 32, device=dev)
            y = torch.randint(0, 10, (B,), device=dev)
            runs, peak = {}, {}
            for m, dt in DTYPES.items():
                # one net and optimizer per dtype: each trains on its own from the same starting point
                net = build_net("lrt", 10, dev, "auto", key, inputs)
                step = mc.MCTrainStep(net, x32.to(dt), S, train_size=50000.0, seed=2024, fold=True)
                runs[m] = (step, torch.optim.Adam(step.params, lr=1e-3), x32.to(dt))
                peak[m] = 0

            def train(m):
                step, opt, x = runs[m]

                def go():
                    step(x, y, beta=0.1)
                    opt.step()

                def window():
                    torch.cuda.synchronize()
                    base = torch.cuda.memory_allocated(dev)
                    torch.cuda.reset_peak_memory_stats(dev)
                    ms = _events(go, args.train_steps)
                    peak[m] = max(peak[m], torch.cuda.max_memory_allocated(dev) - base)
                    return ms
                return window
            times = _alternate({m: train(m) for m in DTYPES}, args.windows)
            for m, t in times.items():
                print(json.dumps({"what": "MCTrainStep(fold=True) + Adam", "net": key, "variant": "lrt", "batch": B,
                                  "mc_samples": S, "layer_fold": runs[m][0].layer_fold, "act_dtype": m,
                                  "steps": args.train_steps, "ms_median": round(statistics.median(t), 3),
                                  "ms_min": round(min(t), 3), "peak_step_mib": round(peak[m] / 2 ** 20, 1), **common}),
                      flush=True)
            del runs
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

"""Scalar Gaussian prior against the scale-mixture prior (set_mixture_prior), on one GPU.

  - the Monte-Carlo KL kernels alone, on one flat parameter vector of BBBAlexNet's 2.18 M and BBB3Conv3FC's 1.78 M
    parameters, 1 and 10 draws: us per call and the achieved bytes/s of the 8 B per parameter the forward must read
    (mu, rho; the backward also reads and writes g_mu, g_rho: 24 B), beside the stand-alone Gaussian KL kernel;
  - ms per step of the headline BBBAlexNet LRT B=512 Monte-Carlo step (mc.MCForward, captured), one step at a time and
    four in flight; the C3-like 10-sample folded step; the BBBLeNet LRT training step with the samples folded
    (MCTrainStep(fold=True) + Adam, B=256, 10 samples).
The mixture net is the scalar one after mixture_prior(net) (same parameters).  The two modes alternate window by window
within one job; the median of the windows is reported with the GPU's name and power limit.  One JSON line per result.

    python tools/kl_mc_bench.py [--steps 200] [--windows 7] [--configs kernel,headline,headline_inflight4,C3,LeNet_train]
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
    "headline": dict(net="alexnet", inputs=3, batch=512, samples=1, inflight=1, train=False),
    "headline_inflight4": dict(net="alexnet", inputs=3, batch=512, samples=1, inflight=4, train=False),
    "C3": dict(net="alexnet", inputs=3, batch=512, samples=10, inflight=1, train=False),
    "LeNet_train": dict(net="lenet", inputs=3, batch=256, samples=10, inflight=1, train=True, steps=5),
}
MODES = ("scalar", "mixture")
KERNEL_SIZES = {"alexnet": 3, "3conv3fc": 1}


def timed(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def kernel_bench(args, dev, name, power):
    import ctypes as C
    from bench import build_net
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn
    lib = L.lib()
    mix = (0.5, 1.0, 0.0024787522)
    for net_name, inputs in KERNEL_SIZES.items():
        n = sum(p.numel() for p in build_net("lrt", 10, dev, "auto", net_name, inputs).parameters()) // 2
        mu = 0.1 * torch.randn(n, device=dev)
        rho = -5.0 + 0.1 * torch.randn(n, device=dev)
        g_mu, g_rho = torch.zeros_like(mu), torch.zeros_like(rho)
        one = torch.ones(16, device=dev)
        kl1 = torch.empty((), device=dev)

        def gauss():
            ws = Fn.workspace(dev)
            L.check(lib.bbb_kl_forward(Fn._ptr(mu), Fn._ptr(rho), n, None, None, 0, 0.0, 0.1, 0, Fn._ptr(kl1), Fn._ptr(ws),
                                       ws.numel(), Fn._stream(dev)), "bbb_kl_forward")
        cases = [("kl_forward (Gaussian)", 1, 8, gauss)]
        for draws in (1, 10):
            kl = torch.empty(draws, device=dev)
            cases.append(("kl_mc_forward", draws, 8,
                          lambda kl=kl: Fn.kl_mc_forward(kl, mu, rho, None, None, mix, 1, 2, None, 1 << 40)))
            cases.append(("kl_mc_backward", draws, 24, lambda draws=draws: L.check(lib.bbb_kl_mc_backward(
                Fn._ptr(mu), Fn._ptr(rho), n, 0, Fn.mixture_arg(mix), 1, 2, None, draws, C.c_uint64(1 << 40), Fn._ptr(one),
                Fn._ptr(g_mu), Fn._ptr(g_rho), Fn._stream(dev)), "bbb_kl_mc_backward")))
        times = {i: [] for i in range(len(cases))}
        for i, c in enumerate(cases):
            timed(c[3], 5)
        for _ in range(args.windows):
            for i, c in enumerate(cases):
                times[i].append(timed(c[3], 200))
        for i, (kname, draws, bytes_per, _) in enumerate(cases):
            ms = statistics.median(times[i])
            print(json.dumps({"config": "kernel", "kernel": kname, "parameters_of": net_name, "parameters": n, "draws": draws,
                              "us_per_call_median": round(ms * 1e3, 2), "us_per_call_min": round(min(times[i]) * 1e3, 2),
                              "bytes_per_parameter": bytes_per, "achieved_GB_per_s": round(bytes_per * n / (ms * 1e-3) / 1e9, 1),
                              "calls_per_window": 200, "windows": args.windows, "gpu": name, "power_limit": power}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--configs", default="kernel," + ",".join(CONFIGS))
    ap.add_argument("--math", default="auto")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    from bench import build_net
    import pytorch_bayesiancnn_b200 as bbb
    from pytorch_bayesiancnn_b200 import mc
    if not torch.cuda.is_available():
        raise SystemExit("kl_mc_bench: needs a CUDA device (nothing is measured without one)")
    dev = torch.device("cuda:0")
    name, power = gpu_info()
    for cname in args.configs.split(","):
        if cname == "kernel":
            kernel_bench(args, dev, name, power)
            continue
        cfg = CONFIGS[cname]
        B, S = cfg["batch"], cfg["samples"]
        steps = cfg.get("steps", args.steps)
        x = torch.randn(B, cfg["inputs"], 32, 32, device=dev)
        y = torch.randint(0, 10, (B,), device=dev)
        base = build_net("lrt", 10, dev, args.math, cfg["net"], cfg["inputs"])
        runs = {}
        for m in MODES:
            net = copy.deepcopy(base)
            if m == "mixture":
                bbb.mixture_prior(net)
            if cfg["train"]:
                eng = mc.MCTrainStep(net, x, S, train_size=50000.0, seed=2024, fold=True)
                opt = torch.optim.Adam(eng.params, lr=1e-3)
                fn = lambda eng=eng, opt=opt: (eng(x, y, beta=0.1), opt.step())
            else:
                eng = mc.MCForward(net, x, S, seed=2024, static_inputs=[x], overlap=cfg["inflight"] > 1,
                                   inflight=cfg["inflight"])
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
            eng = runs[m][0]
            print(json.dumps({"config": cname, "net": cfg["net"], "variant": "lrt", "math": args.math, "batch": B,
                              "mc_samples": S, "inflight": cfg["inflight"], "train": cfg["train"], "prior": m,
                              "ms_per_step_median": round(statistics.median(times[m]), 4),
                              "ms_per_step_min": round(min(times[m]), 4), "kernels_per_step": eng.kernels_per_step,
                              "kl": round(float(eng.out["kl"]), 3), "windows": args.windows,
                              "steps_per_window": steps, "gpu": name, "power_limit": power}), flush=True)
        del runs
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

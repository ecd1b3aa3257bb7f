"""Cost of temperature scaling (bbb_mc_logit_log, bbb_mc_temper, bbb_temperature_nll, mc.calibrate_temperature) on one
GPU, variants alternating window by window in one job, medians over --windows windows.

* kernels: the temper and the logit-log kernels alone, a captured graph of --launches launches each, at (S, B, C) =
  (1, 512, 10), (10, 512, 10), (100, 2048, 10) and (25, 1024, 100); GB/s counts the bytes each must move (temper: read
  and write S B C fp32; logit log: the same plus the labels) against HBM3's 3.35 TB/s.  The temper rewrites one buffer
  in place (L2-resident when it fits); the logit-log launches of a window append to consecutive entries of one bank
  whose cursor is reset once per window, outside the graph;
* fit: mc.fit_temperature with the defaults (32 points, 4 rounds) on n = 10000 images at (S, C) = (100, 10), (25, 100)
  and (1, 10) (the reference's one-sample setting: 1 of 32 lanes works), and on n = 2000 at (10, 1000).  Exponentials: the C-loop's ex2 per (image, sample, class, evaluated point), useful (33 + 3 x 32 points)
  and executed (the kernel sweeps 11 points per row pass).  The SFU bound is 16 ex2 per clock per SM (sm_90) x the SMs
  x the SM clock nvidia-smi reports right after the timed windows;
* inflight: the MCForward step with four in flight (overlap=True, inflight=4, resident batches, labels), without and
  with a temperature: headline-like (BBBAlexNet-10, B=512, 1 sample), C3-like (10 samples) and C5 (BBB3Conv3FC-10,
  B=2048, 100 samples);
* calibrate: --batches batches of an overconfident BBBLeNet-10 (B=256, 10 samples; classifier means x 5), labels
  drawn from its own predictive tempered by T0 = 3 so that the optimum lies inside [0.05, 20], through a reference-style
  loop (a serial captured step per batch, .cpu() of its per-sample logits, scipy.optimize.minimize_scalar of the
  float64 NLL over ln T) against mc.calibrate_temperature.  Both arms' engines are built before the timed windows.  The
  first call of either arm draws the same noise, so both fit the same logits: the difference of their ln T is
  reported beside the search's resolution.

Prints one JSON line per measurement with the GPU's name and power limit.

    python tools/temperature_bench.py [--windows 5] [--launches 100] [--inflight-steps 100] [--batches 10]
                                      [--only kernels,fit,inflight,calibrate]
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from tools.mc_fold_bench import gpu_info
from tools.mc_info_bench import _events_ms

KERNEL_SHAPES = ((1, 512, 10), (10, 512, 10), (100, 2048, 10), (25, 1024, 100))
FIT_SHAPES = ((10000, 100, 10), (10000, 25, 100), (10000, 1, 10), (2000, 10, 1000))
WORKLOADS = {"headline": ("alexnet", 3, 512, 1), "C3": ("alexnet", 3, 512, 10), "C5": ("3conv3fc", 1, 2048, 100)}
HBM = 3.35e12
SEED = 2024


def sm_clock_mhz():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return float(q)
    except Exception:
        return float("nan")


def _graph(fn, dev, launches):
    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        for _ in range(launches):
            fn()
    g.replay()
    torch.cuda.synchronize()
    return g


def kernel_bench(args, dev, gpu, power):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn, mc
    lib = L.lib()
    for S, B, C in KERNEL_SHAPES:
        z = torch.randn(S, B, C, device=dev)
        y = torch.randint(0, C, (B,), device=dev)
        t = torch.ones(1, dtype=torch.float32, device=dev)       # z / 1: the values stay put over many launches
        bank = mc.LogitBank(dev, (args.launches + 1) * B, S, C)     # every launch of a window writes its own entries
        temper = lambda: L.check(lib.bbb_mc_temper(Fn._ptr(z), z.numel(), Fn._ptr(t), Fn._stream(dev)), "temper")
        log = lambda: bank._launch(z, y, B)
        graphs = {"temper": _graph(temper, dev, args.launches), "logit_log": _graph(log, dev, args.launches)}
        nbytes = {"temper": 2 * z.numel() * 4, "logit_log": 2 * z.numel() * 4 + 2 * B * 8}
        times = {k: [] for k in graphs}
        for _ in range(args.windows):
            for k, g in graphs.items():
                bank.reset()                                           # once per window, outside the timed graph
                times[k].append(1000.0 * _events_ms(g.replay, args.launches))
        assert bank.dropped == 0
        for k in graphs:
            us = statistics.median(times[k])
            print(json.dumps({"what": f"{k} kernel", "S": S, "B": B, "C": C, "us_per_launch_median": round(us, 2),
                              "us_per_launch_min": round(min(times[k]), 2), "bytes": nbytes[k],
                              "GBps": round(nbytes[k] / us / 1e3, 1), "share_of_hbm": round(nbytes[k] / us / 1e-6 / HBM, 3),
                              "windows": args.windows, "launches_per_window": args.launches, "gpu": gpu,
                              "power_limit": power}), flush=True)


def fit_bench(args, dev, gpu, power):
    from pytorch_bayesiancnn_b200 import mc
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    for n, S, C in FIT_SHAPES:
        g = torch.Generator(device=dev).manual_seed(1)
        bank = mc.LogitBank(dev, n, S, C)
        for b0 in range(0, n, 1000):
            bank.append(torch.randn(S, 1000, C, device=dev, generator=g) * 3,
                        torch.randint(0, C, (1000,), device=dev, generator=g))
        out = torch.empty(1, dtype=torch.float32, device=dev)
        fit = lambda: mc.fit_temperature(bank, out=out)
        r = fit().read()
        times = [_events_ms(fit, 1) for _ in range(args.windows)]
        mhz = sm_clock_mhz()
        useful = n * S * C * (33 + 3 * 32)
        executed = n * S * C * 11 * (3 + 3 * 3)
        ms = statistics.median(times)
        bound = sms * 16 * mhz * 1e6
        print(json.dumps({"what": "fit_temperature", "n": n, "S": S, "C": C, "ms_per_fit_median": round(ms, 3),
                          "ms_per_fit_min": round(min(times), 3), "temperature": r["temperature"],
                          "ex2_useful_per_s": useful / ms * 1e3, "ex2_executed_per_s": executed / ms * 1e3,
                          "sm_clock_mhz": mhz, "sms": sms, "sfu_bound_ex2_per_s": bound,
                          "share_of_sfu_bound_executed": round(executed / ms * 1e3 / bound, 3),
                          "windows": args.windows, "gpu": gpu, "power_limit": power}), flush=True)


def inflight_bench(args, dev, gpu, power):
    from bench import build_net
    from pytorch_bayesiancnn_b200 import mc
    for name, (key, inputs, B, S) in WORKLOADS.items():
        net = build_net("lrt", 10, dev, "auto", key, inputs)
        xs = [torch.randn(B, inputs, 32, 32, device=dev) for _ in range(4)]
        y = torch.randint(0, 10, (B,), device=dev)
        steps = args.inflight_steps if name != "C5" else max(2, args.inflight_steps // 10)
        temps = {False: None, True: 1.5}
        engines = {m: mc.MCForward(net, xs[0], S, with_labels=True, seed=SEED, static_inputs=xs, overlap=True,
                                   inflight=4, temperature=temps[m]) for m in (False, True)}

        def run(m):
            def go():
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
        for m in (False, True):
            print(json.dumps({"what": "MCForward step in flight", "workload": name, "batch": B, "mc_samples": S,
                              "inflight": 4, "temperature": temps[m], "kernels_per_step": engines[m].kernels_per_step,
                              "ms_per_step_median": round(statistics.median(times[m]), 4),
                              "ms_per_step_min": round(min(times[m]), 4), "steps_per_window": steps,
                              "windows": args.windows, "gpu": gpu, "power_limit": power}), flush=True)
        del engines, net


def calibrate_bench(args, dev, gpu, power):
    from scipy.optimize import minimize_scalar
    from scipy.special import logsumexp
    from bench import build_net
    from pytorch_bayesiancnn_b200 import mc
    B, S, C, T0 = 256, 10, 10, 3.0
    net = build_net("lrt", C, dev, "auto", "lenet", 1)
    last = [m for m in net.children() if hasattr(m, "W_mu")][-1]
    with torch.no_grad():
        last.W_mu.mul_(5.0)                                        # an overconfident net
    g = torch.Generator().manual_seed(3)
    xs_host = [torch.randn(B, 1, 32, 32, generator=g).pin_memory() for _ in range(args.batches)]
    xs = [torch.zeros(B, 1, 32, 32, device=dev) for _ in range(args.batches)]
    # labels drawn from the net's own predictive tempered by T0 (on the logits of replays 0 .. batches-1, the ones the
    # first call of either arm draws): the optimum lies inside [t_min, t_max], near T0
    label_eng = mc.MCForward(net, xs[0], S, seed=SEED, static_inputs=xs)
    ys_host = []
    for i, x in enumerate(xs_host):
        label_eng(x, slot=i)
        z = label_eng.logits_all[0].double() / T0
        p = torch.softmax(z, 2).mean(0)
        ys_host.append(torch.multinomial(p.cpu(), 1, generator=g)[:, 0].pin_memory())
    del label_eng
    batches = list(zip(xs_host, ys_host))
    ref_eng = mc.MCForward(net, xs[0], S, with_labels=True, seed=SEED, static_inputs=xs)   # built once, untimed

    def reference():
        zs, ys = [], []
        for i, (x, y) in enumerate(batches):
            ref_eng(x, y.to(dev, non_blocking=True), slot=i)
            zs.append(ref_eng.logits_all[0].cpu().double().numpy().transpose(1, 0, 2))
            ys.append(y.numpy())
        z, yy = np.concatenate(zs), np.concatenate(ys)

        def nll(tau):
            x = z / math.exp(tau)
            lp = np.take_along_axis(x, yy[:, None, None].repeat(S, 1), 2)[:, :, 0] - logsumexp(x, axis=2)
            return float(-(logsumexp(lp, axis=1) - math.log(S)).mean())
        return minimize_scalar(nll, bounds=(math.log(0.05), math.log(20.0)), method="bounded",
                               options={"xatol": 1e-6}).x

    def ours():
        return mc.calibrate_temperature(net, batches, S, seed=SEED)["fit"]
    first = ours()              # builds evaluate's engines; its first call draws the noise of the reference's first
    times = {"reference_loop": [], "calibrate_temperature": []}
    tau_ref = None
    for _ in range(args.windows):
        for k, fn in (("reference_loop", reference), ("calibrate_temperature", ours)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn()
            torch.cuda.synchronize()
            times[k].append(1000.0 * (time.perf_counter() - t0))
            if k == "reference_loop" and tau_ref is None:
                tau_ref = r
    res = (math.log(20.0) - math.log(0.05)) / 31 * (2 / 31) ** 3
    print(json.dumps({"what": "calibrate", "batches": len(batches), "batch": B, "mc_samples": S, "labels_from_T": T0,
                      "reference_loop_ms_median": round(statistics.median(times["reference_loop"]), 2),
                      "calibrate_temperature_ms_median": round(statistics.median(times["calibrate_temperature"]), 2),
                      "T_reference": math.exp(tau_ref), "T_ours": first["temperature"], "at_bound": first["at_bound"],
                      "abs_dlnT": abs(tau_ref - first["tau"]), "search_resolution_lnT": res, "windows": args.windows,
                      "gpu": gpu, "power_limit": power}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--inflight-steps", type=int, default=100, help="steps per window of the in-flight arm (C5: / 10)")
    ap.add_argument("--batches", type=int, default=10)
    ap.add_argument("--only", default="kernels,fit,inflight,calibrate")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("temperature_bench: needs a CUDA device")
    import __graft_entry__ as g
    g.build()
    dev = torch.device("cuda:0")
    gpu, power = gpu_info()
    only = set(args.only.split(","))
    for name, fn in (("kernels", kernel_bench), ("fit", fit_bench), ("inflight", inflight_bench),
                     ("calibrate", calibrate_bench)):
        if name in only:
            fn(args, dev, gpu, power)


if __name__ == "__main__":
    main()

"""Cost of vector scaling (bbb_mc_logit_scale, bbb_scaling_nll_grad, mc.fit_scaling) on one GPU, variants alternating
window by window in one job, medians over --windows windows.

* kernels: the apply kernel alone (vector and matrix), a captured graph of --launches launches, at (S, B, C) = (1, 512, 10), (10, 512, 10)
  and (25, 1024, 100), beside the temper at the same shapes; GB/s counts the bytes it must move (read and write S B C
  fp32) against HBM3's 3.35 TB/s.  Both rewrite one buffer in place (L2-resident when it fits); the apply runs with the
  identity so the values stay put over many launches;
* fit: mc.fit_scaling with the defaults (300 Adam passes + 1), vector and matrix, on n = 10000 images at (S, C) =
  (25, 100) and (100, 10), against a torch float32 autograd + torch.optim.LBFGS fit of the same bank and map on the
  same GPU (lr 1, 100 iterations, strong-Wolfe line search, from the identity); both results' NLLs are evaluated in
  float64 on the device.  Also the time per pass, and for the matrix pass its useful tf32 FLOP/s (two forwards and one
  gradient contraction, 6 n S C^2) against the 495 TFLOP/s dense TF32 figure of the data sheet;
* inflight: the MCForward step with four in flight (overlap=True, inflight=4, resident batches, labels), without and
  with a scaling: headline-like (BBBAlexNet-10, B=512, 1 sample) and C3-like (10 samples).

Prints one JSON line per measurement with the GPU's name and power limit.

    python tools/scaling_bench.py [--windows 5] [--launches 100] [--inflight-steps 100] [--only kernels,fit,inflight]
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from tools.mc_fold_bench import gpu_info
from tools.mc_info_bench import _events_ms
from tools.temperature_bench import HBM, SEED, _graph

KERNEL_SHAPES = ((1, 512, 10), (10, 512, 10), (25, 1024, 100))
FIT_SHAPES = ((10000, 25, 100), (10000, 100, 10))
WORKLOADS = {"headline": ("alexnet", 3, 512, 1), "C3": ("alexnet", 3, 512, 10)}


def kernel_bench(args, dev, gpu, power):
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn, mc
    lib = L.lib()
    for S, B, C in KERNEL_SHAPES:
        z = torch.randn(S, B, C, device=dev)
        sc = mc.LogitScaling(dev, C)                               # the identity: the values stay put
        sm = mc.LogitScaling(dev, C, "matrix")
        t = torch.ones(1, dtype=torch.float32, device=dev)
        apply = lambda: sc._launch(z, Fn._stream(dev))
        apply_m = lambda: sm._launch(z, Fn._stream(dev))
        temper = lambda: L.check(lib.bbb_mc_temper(Fn._ptr(z), z.numel(), Fn._ptr(t), Fn._stream(dev)), "temper")
        graphs = {"logit_scale vector": _graph(apply, dev, args.launches),
                  "logit_scale matrix": _graph(apply_m, dev, args.launches), "temper": _graph(temper, dev, args.launches)}
        nbytes = 2 * z.numel() * 4
        times = {k: [] for k in graphs}
        for _ in range(args.windows):
            for k, g in graphs.items():
                times[k].append(1000.0 * _events_ms(g.replay, args.launches))
        for k in graphs:
            us = statistics.median(times[k])
            print(json.dumps({"what": f"{k} kernel", "S": S, "B": B, "C": C, "us_per_launch_median": round(us, 2),
                              "us_per_launch_min": round(min(times[k]), 2), "bytes": nbytes,
                              "GBps": round(nbytes / us / 1e3, 1), "share_of_hbm": round(nbytes / us / 1e-6 / HBM, 3),
                              "windows": args.windows, "launches_per_window": args.launches, "gpu": gpu,
                              "power_limit": power}), flush=True)


def _nll64(z, y, a, b):
    """The bank's NLL at (a, b) -- a [C] or W [C, C] -- in float64 on the device."""
    t = (z.double() @ a.double().T if a.dim() == 2 else z.double() * a.double()) + b.double()
    lp = torch.log_softmax(t, 2).gather(2, y[:, None, None].expand(-1, z.shape[1], 1))[:, :, 0]
    return float(-(torch.logsumexp(lp, 1) - torch.log(torch.tensor(float(z.shape[1]), dtype=torch.float64))).mean())


def _torch_lbfgs(z, y, iters, matrix=False):
    """The torch float32 autograd + LBFGS fit of the same objective: (a or W, b)."""
    C = z.shape[2]
    a = (torch.eye(C, device=z.device) if matrix else torch.ones(C, device=z.device)).requires_grad_(True)
    b = torch.zeros(C, device=z.device, requires_grad=True)
    opt = torch.optim.LBFGS([a, b], lr=1.0, max_iter=iters, line_search_fn="strong_wolfe")
    lnS = torch.log(torch.tensor(float(z.shape[1]), device=z.device))

    def closure():
        opt.zero_grad()
        lp = torch.log_softmax((z @ a.T if matrix else z * a) + b, 2).gather(2, y[:, None, None].expand(-1, z.shape[1], 1))[:, :, 0]
        loss = -(torch.logsumexp(lp, 1) - lnS).mean()
        loss.backward()
        return loss
    opt.step(closure)
    return a.detach(), b.detach()


def fit_bench(args, dev, gpu, power):
    from pytorch_bayesiancnn_b200 import mc
    for n, S, C in FIT_SHAPES:
        g = torch.Generator(device=dev).manual_seed(1)
        z = torch.randn(n, S, C, device=dev, generator=g) * 2 + torch.randn(n, 1, C, device=dev, generator=g) * 2
        a0 = torch.rand(C, device=dev, generator=g) * 1.2 + 0.4
        b0 = torch.randn(C, device=dev, generator=g)
        p = torch.softmax(z.double() * a0 + b0, 2).mean(1)
        y = torch.multinomial(p, 1, generator=g)[:, 0]
        bank = mc.LogitBank(dev, n, S, C)
        bank.append(z.permute(1, 0, 2).contiguous(), y)
        for kind in ("vector", "matrix"):
            out = mc.LogitScaling(dev, C, kind)
            ours = lambda: mc.fit_scaling(bank, kind, out=out)
            ref = {}

            def theirs():
                ref["ab"] = _torch_lbfgs(z, y, args.lbfgs_iters, kind == "matrix")
            r = ours().read()
            theirs()
            times = {"fit_scaling": [], "torch_lbfgs": []}
            for _ in range(args.windows):
                for k, fn in (("fit_scaling", ours), ("torch_lbfgs", theirs)):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    times[k].append(1000.0 * (time.perf_counter() - t0))
            ms = statistics.median(times["fit_scaling"])
            us_pass = 1000.0 * ms / (r["iters"] + 1)
            rec = {"what": f"fit_scaling {kind}", "n": n, "S": S, "C": C, "iters": r["iters"],
                   "ms_per_fit_median": round(ms, 3), "ms_per_fit_min": round(min(times["fit_scaling"]), 3),
                   "us_per_pass_median": round(us_pass, 2),
                   "torch_lbfgs_ms_median": round(statistics.median(times["torch_lbfgs"]), 3),
                   "torch_lbfgs_iters": args.lbfgs_iters, "nll_start": r["nll_start"],
                   "nll_fit_scaling": _nll64(z, y, out.W if kind == "matrix" else out.a, out.b),
                   "nll_torch_lbfgs": _nll64(z, y, *ref["ab"]), "nll_planted": _nll64(z, y, a0, b0),
                   "windows": args.windows, "gpu": gpu, "power_limit": power}
            if kind == "matrix":
                # the useful tf32 work of a pass: two forwards Z W^T and one G^T Z, 2 n S C^2 flops each
                flops = 3 * 2.0 * n * S * C * C
                rec.update(tflops_per_s=round(flops / us_pass / 1e6, 3), tf32_bound_tflops=495.0,
                           share_of_tf32_bound=round(flops / us_pass / 1e6 / 495.0, 5))
            print(json.dumps(rec), flush=True)


def inflight_bench(args, dev, gpu, power):
    from bench import build_net
    from pytorch_bayesiancnn_b200 import mc
    for name, (key, inputs, B, S) in WORKLOADS.items():
        net = build_net("lrt", 10, dev, "auto", key, inputs)
        xs = [torch.randn(B, inputs, 32, 32, device=dev) for _ in range(4)]
        y = torch.randint(0, 10, (B,), device=dev)
        steps = args.inflight_steps
        sc = mc.LogitScaling(dev, 10)
        with torch.no_grad():
            sc.a.fill_(0.7)
            sc.b.copy_(torch.linspace(-0.5, 0.5, 10))
        maps = {False: None, True: sc}
        engines = {m: mc.MCForward(net, xs[0], S, with_labels=True, seed=SEED, static_inputs=xs, overlap=True,
                                   inflight=4, scaling=maps[m]) for m in (False, True)}

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
                              "inflight": 4, "scaling": m, "kernels_per_step": engines[m].kernels_per_step,
                              "ms_per_step_median": round(statistics.median(times[m]), 4),
                              "ms_per_step_min": round(min(times[m]), 4), "steps_per_window": steps,
                              "windows": args.windows, "gpu": gpu, "power_limit": power}), flush=True)
        del engines, net


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--inflight-steps", type=int, default=100)
    ap.add_argument("--lbfgs-iters", type=int, default=100)
    ap.add_argument("--only", default="kernels,fit,inflight")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scaling_bench: needs a CUDA device")
    import __graft_entry__ as g
    g.build()
    dev = torch.device("cuda:0")
    gpu, power = gpu_info()
    only = set(args.only.split(","))
    for name, fn in (("kernels", kernel_bench), ("fit", fit_bench), ("inflight", inflight_bench)):
        if name in only:
            fn(args, dev, gpu, power)


if __name__ == "__main__":
    main()

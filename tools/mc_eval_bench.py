"""Cost of a validation epoch on one GPU: the reference-style loop against mc.evaluate(), alternating window by window in
one job, median over --windows windows.

* reference-style (main_bayesian.validate_model): per batch, inputs and labels to the device, one serial MCForward
  step, ``.item()`` of its head and kl, and calibration (nll, Brier, 15-bin ECE) on the host from log_outputs;
* evaluate(): every batch in flight (overlap=True, inflight=4) into one device accumulator, one host read per epoch.

Both build their engines in a first, untimed epoch (evaluate() keeps them on the net): the windows time the steady-state
epoch a training run pays after the first.  The batches are pageable host tensors, as a DataLoader without pin_memory
yields them.

Workloads (a synthetic held-out set of --batches host batches, the last one ragged):
  headline-like: BBBAlexNet-10, B=512, 1 sample;  C3-like: BBBAlexNet-10, B=512, 10 samples;
  C5: BBB3Conv3FC-10, 1x32x32, B=2048, 100 samples (--c5-batches batches).
Also the exchange kernel alone with and without METRICS, as tools/mc_info_bench.py (C3-like and C5 shapes; both arms are
the sample-only instantiations), and the step in flight (overlap=True, inflight=4, resident batches) with and without
the accumulator (headline-like and C5), where the exchange CTA shares the SMs with the next steps' layer kernels.

Prints one JSON line per measurement with the GPU's name and power limit.

    python tools/mc_eval_bench.py [--windows 7] [--batches 10] [--c5-batches 3] [--only kernel,inflight,headline,C3,C5]
"""
import argparse
import ctypes as C
import json
import math
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from tools.mc_fold_bench import gpu_info
from tools.mc_info_bench import _events_ms

WORKLOADS = {"headline": ("alexnet", 3, 512, 1), "C3": ("alexnet", 3, 512, 10), "C5": ("3conv3fc", 1, 2048, 100)}
TRAIN_SIZE = 50000.0


def host_calibration(lo, y, bins=15):
    """nll, correct, brier and per-bin count / conf / correct sums of one batch, in float64 on the host."""
    lo = lo.double()
    p = lo.exp()
    best = lo.argmax(1)
    conf = p.gather(1, best[:, None])[:, 0]
    correct = (best == y).double()
    onehot = torch.zeros_like(p).scatter_(1, y[:, None], 1.0)
    m = (torch.ceil(conf * bins) - 1).clamp(0, bins - 1).long()
    z = torch.zeros(bins, dtype=torch.float64)
    return (float(-lo.gather(1, y[:, None]).sum()), float(correct.sum()), float(((p - onehot) ** 2).sum()),
            z.clone().index_add_(0, m, torch.ones_like(conf)), z.clone().index_add_(0, m, conf),
            z.clone().index_add_(0, m, correct))


def reference_epoch(eng, batches, num_ens, dev):
    """validate_model's loop on a serial engine: one step, one host read, host-side calibration per batch."""
    from pytorch_bayesiancnn_b200 import mc
    n, loss, accs, tot = len(batches), 0.0, [], None
    for i, (x, y) in enumerate(batches):
        out = eng(x.to(dev), y.to(dev))
        nll, kl = out["head"][1].item(), out["kl"].item() * num_ens
        loss += nll * TRAIN_SIZE + mc.get_beta(i - 1, n, 0.1) * kl
        accs.append(out["head"][2].item())
        cal = host_calibration(out["log_outputs"].cpu(), y)
        tot = cal if tot is None else tuple(a + b for a, b in zip(tot, cal))
    images = sum(x.shape[0] for x, _ in batches)
    return {"valid_loss": loss / n, "valid_acc": sum(accs) / n, "nll": tot[0] / images, "accuracy": tot[1] / images,
            "brier": tot[2] / images, "ece": float((tot[5] - tot[4]).abs().sum()) / images}


def epoch_bench(name, args, dev, gpu, power):
    from bench import build_net
    from pytorch_bayesiancnn_b200 import mc
    key, inputs, B, S = WORKLOADS[name]
    nb = args.c5_batches if name == "C5" else args.batches
    g = torch.Generator().manual_seed(0)
    batches = [(torch.randn(B if i < nb - 1 else B // 2 + 8, inputs, 32, 32, generator=g),
                torch.randint(0, 10, (B if i < nb - 1 else B // 2 + 8,), generator=g)) for i in range(nb)]
    net = build_net("lrt", 10, dev, "auto", key, inputs)
    engines = {}

    def ref():
        for x, _ in batches:                            # one serial engine per batch shape, built outside the windows
            if tuple(x.shape) not in engines:
                engines[tuple(x.shape)] = mc.MCForward(net, x.to(dev), S, with_labels=True, train_size=TRAIN_SIZE,
                                                       seed=2024)
        return reference_epoch(_Dispatch(engines), batches, S, dev)

    def ev():
        return mc.evaluate(net, batches, S, TRAIN_SIZE, 0.1, seed=2024, inflight=4)
    res = {"reference": ref(), "evaluate": ev()}       # warm-up: builds and captures every engine
    times = {"reference": [], "evaluate": []}
    for _ in range(args.windows):
        for k, fn in (("reference", ref), ("evaluate", ev)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res[k] = fn()
            torch.cuda.synchronize()
            times[k].append(1000.0 * (time.perf_counter() - t0))
    images = sum(x.shape[0] for x, _ in batches)
    for k in times:
        med = statistics.median(times[k])
        r = res[k]
        print(json.dumps({"what": "validation epoch", "workload": name, "version": k, "batch": B, "mc_samples": S,
                          "batches": nb, "images": images, "ms_per_epoch_median": round(med, 3),
                          "ms_per_epoch_min": round(min(times[k]), 3), "ms_per_batch_median": round(med / nb, 4),
                          "windows": args.windows,
                          **{m: (round(r[m], 6) if math.isfinite(r[m]) else None)
                             for m in ("valid_loss", "valid_acc", "nll", "accuracy", "brier", "ece")},
                          "gpu": gpu, "power_limit": power}), flush=True)


class _Dispatch:
    """The serial engine of the batch's shape (the reference loop's net(inputs) takes any batch size)."""

    def __init__(self, engines):
        self.engines = engines

    def __call__(self, x, y):
        return self.engines[tuple(x.shape)](x, y)


def kernel_bench(args, dev, gpu, power):
    """The exchange kernel alone, one rank, a captured graph of --launches launches: without / with METRICS."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn, mc
    lib = L.lib()
    for sname, (B, Cc, S) in {"C3-like": (512, 10, 10), "C5": (2048, 10, 100)}.items():
        logits = torch.randn(S, B, Cc, device=dev, generator=torch.Generator(device=dev).manual_seed(1)) * 4
        labels = torch.randint(0, Cc, (B,), device=dev, generator=torch.Generator(device=dev).manual_seed(2))
        graphs, keep = {}, []
        for metrics in (False, True):
            buf = torch.zeros(int(lib.bbb_mc_buffer_bytes(B, Cc, 0, 1)), dtype=torch.uint8, device=dev)
            state = torch.zeros(int(lib.bbb_mc_state_bytes()), dtype=torch.uint8, device=dev)
            lo, kl, head = torch.empty(B, Cc, device=dev), torch.empty((), device=dev), torch.empty(4, device=dev)
            acc = mc.new_metrics(dev)
            peers = (C.c_void_p * 1)(buf.data_ptr())
            keep += [buf, state, lo, kl, head, acc, peers]

            def launch(metrics=metrics, state=state, lo=lo, kl=kl, head=head, acc=acc, peers=peers):
                args_ = (Fn._ptr(logits), S, S, B, Cc, None, 0, 0, Fn._ptr(labels), C.c_float(1.0), C.c_float(0.1), 0, 1,
                         peers, Fn._ptr(state), Fn._ptr(lo), Fn._ptr(kl), None, None, None, None, Fn._ptr(head), None, 0,
                         None, None, 1)
                if metrics:
                    L.check(lib.bbb_mc_exchange_metrics(*args_, Fn._ptr(acc), Fn._stream(dev)), "metrics")
                else:
                    L.check(lib.bbb_mc_exchange_sharded(*args_, Fn._stream(dev)), "sharded")
            side = torch.cuda.Stream(device=dev)
            with torch.cuda.stream(side):
                launch()
            torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=side):
                for _ in range(args.launches):
                    launch()
            graphs[metrics] = gr
        times = {False: [], True: []}
        for m in (False, True):
            graphs[m].replay()
        for _ in range(args.windows):
            for m in (False, True):
                times[m].append(1000.0 * _events_ms(graphs[m].replay, args.launches))
        for m in (False, True):
            print(json.dumps({"what": "exchange kernel", "shape": sname, "batch": B, "classes": Cc, "local_samples": S,
                              "metrics": m, "labels": True, "us_per_launch_median": round(statistics.median(times[m]), 2),
                              "us_per_launch_min": round(min(times[m]), 2), "windows": args.windows,
                              "launches_per_window": args.launches, "gpu": gpu, "power_limit": power}), flush=True)


def inflight_bench(args, dev, gpu, power):
    """K steps in flight over resident batches, engines with and without the accumulator alternating window by window."""
    from bench import build_net
    from pytorch_bayesiancnn_b200 import mc
    for name in ("headline", "C5"):
        key, inputs, B, S = WORKLOADS[name]
        net = build_net("lrt", 10, dev, "auto", key, inputs)
        xs = [torch.randn(B, inputs, 32, 32, device=dev) for _ in range(4)]
        y = torch.randint(0, 10, (B,), device=dev)
        engines = {m: mc.MCForward(net, xs[0], S, with_labels=True, train_size=TRAIN_SIZE, seed=2024, static_inputs=xs,
                                   overlap=True, inflight=4, metrics=mc.new_metrics(dev) if m else None)
                   for m in (False, True)}
        steps = args.inflight_steps if name != "C5" else max(2, args.inflight_steps // 10)

        def run(eng):
            def go():
                for i in range(steps):
                    eng(labels=y, slot=i % len(xs))
                eng.wait()
            return go
        times = {False: [], True: []}
        for m in (False, True):
            run(engines[m])()
        for _ in range(args.windows):
            for m in (False, True):
                times[m].append(_events_ms(run(engines[m]), steps))
        for m in (False, True):
            print(json.dumps({"what": "MCForward step in flight", "workload": name, "batch": B, "mc_samples": S,
                              "inflight": 4, "metrics": m, "ms_per_step_median": round(statistics.median(times[m]), 4),
                              "ms_per_step_min": round(min(times[m]), 4), "steps_per_window": steps,
                              "windows": args.windows, "gpu": gpu, "power_limit": power}), flush=True)
        del engines, net


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--batches", type=int, default=10, help="batches per epoch (headline / C3)")
    ap.add_argument("--c5-batches", type=int, default=3, help="batches per epoch (C5)")
    ap.add_argument("--launches", type=int, default=50, help="exchange launches per captured graph (one window)")
    ap.add_argument("--inflight-steps", type=int, default=100, help="steps per window of the in-flight arm (C5: / 10)")
    ap.add_argument("--only", default="kernel,inflight,headline,C3,C5")
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
    for name in WORKLOADS:
        if name in only:
            epoch_bench(name, args, dev, gpu, power)


if __name__ == "__main__":
    main()

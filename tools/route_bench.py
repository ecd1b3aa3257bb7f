"""Cost of routing between task experts (bbb_mc_route, mc.ExpertStep, mc.route) on one GPU, variants alternating
window by window in one job, medians over --windows windows.

* kernel: the routing kernel alone (epistemic score, labels, accumulator, no log), a captured graph of --launches
  launches, at (K, B, C) = (2, 256, 5), (5, 256, 2) and (10, 1024, 10);
* step: one routed batch of K BBBLeNet LRT experts (1x32x32, C = 10 / K, B = 256, T = 10 and 25 samples, K = 2 and 5):
  K lone MCForward steps one after another (captured serial engines) and the routing in torch, against ExpertStep with
  one and with four steps in flight; every variant runs --steps batches from resident input slots per window;
* loop: --batches host batches through the reference-style loop (get_uncertainty_per_batch: T drop-in forwards per
  expert through mc.engine_forward_fn, softmax, a numpy loop over the images for the epistemic and aleatoric
  diagonals; np.sum and the least uncertain expert per image, ties to the last) against mc.route.  Sample j of batch t
  draws the noise of the engine's sample j of step t, so both route the same planes up to the exchange's arithmetic:
  the share of identical decisions is reported, overall and where the two smallest scores differ by more than 1e-4
  relative.  mc.route builds its steps in a first, untimed call.

Prints one JSON line per measurement with the GPU's name and power limit.

    python tools/route_bench.py [--windows 7] [--launches 100] [--steps 50] [--batches 10] [--only kernel,step,loop]
"""
import argparse
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

KERNEL_SHAPES = ((2, 256, 5), (5, 256, 2), (10, 1024, 10))
SEED = 2024


def experts(K, C, dev, T=None):
    """K BBBLeNet LRT experts with different weights (bench.py's initialisation, seeds 123 + k)."""
    from bench import build_net
    nets = []
    for k in range(K):
        net = build_net("lrt", C, dev, "auto", "lenet", 1)
        g = torch.Generator().manual_seed(123 + k)
        with torch.no_grad():
            for name, p in net.named_parameters():
                p.copy_(torch.empty(p.shape).normal_(-5.0 if name.endswith("rho") else 0.0, 0.1, generator=g).to(dev))
        nets.append(net)
    return nets


def kernel_bench(args, dev, gpu, power):
    from pytorch_bayesiancnn_b200 import mc
    for K, B, C in KERNEL_SHAPES:
        g = torch.Generator(device=dev).manual_seed(1)
        outs = [{k: torch.rand(B, C, device=dev, generator=g) for k in ("pred", "epistemic", "aleatoric", "log_outputs")}
                for _ in range(K)]
        y = torch.randint(0, K * C, (B,), device=dev, generator=g)
        acc = mc.new_route_metrics(dev)
        res = mc._route_result(B, K, dev)
        launch = mc._route_launcher(outs, "epistemic", None, acc, None, res)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            launch(y, -1)
        torch.cuda.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=side):
            for _ in range(args.launches):
                launch(y, -1)
        gr.replay()
        times = [1000.0 * _events_ms(gr.replay, args.launches) for _ in range(args.windows)]
        torch.cuda.synchronize()
        print(json.dumps({"what": "route kernel", "experts": K, "batch": B, "classes": C,
                          "us_per_launch_median": round(statistics.median(times), 2),
                          "us_per_launch_min": round(min(times), 2), "windows": args.windows,
                          "launches_per_window": args.launches, "gpu": gpu, "power_limit": power}), flush=True)


def torch_route(outs, C):
    """The routing a user writes by hand on K lone steps: sum_c epistemic, the least uncertain expert (ties to the
    last), its argmax."""
    u = torch.stack([o["epistemic"].double().sum(1) for o in outs], 1)
    K = u.shape[1]
    e = K - 1 - torch.argmin(u.flip(1), dim=1)
    pred = torch.stack([o["pred"] for o in outs], 1)
    local = pred[torch.arange(pred.shape[0], device=pred.device), e].argmax(1)
    return e, e * C + local


def step_bench(args, dev, gpu, power):
    from pytorch_bayesiancnn_b200 import mc
    B = 256
    for K in (2, 5):
        C = 10 // K
        nets = experts(K, C, dev)
        for T in (10, 25):
            xs = [torch.randn(B, 1, 32, 32, device=dev) for _ in range(4)]
            lone = [mc.MCForward(n, xs[0], T, want_uncertainty=True, seed=SEED, static_inputs=xs) for n in nets]
            steps = {f: mc.ExpertStep(nets, xs[0], T, seed=SEED, static_inputs=xs, inflight=f) for f in (1, 4)}

            def run_lone():
                for i in range(args.steps):
                    outs = [e(slot=i % 4) for e in lone]
                    torch_route(outs, C)
                torch.cuda.synchronize()

            def run_step(f):
                def go():
                    for i in range(args.steps):
                        steps[f](slot=i % 4)
                    steps[f].wait()
                    torch.cuda.synchronize()
                return go
            variants = {"lone steps + torch routing": run_lone, "ExpertStep inflight=1": run_step(1),
                        "ExpertStep inflight=4": run_step(4)}
            for fn in variants.values():
                fn()
            times = {k: [] for k in variants}
            for _ in range(args.windows):
                for k, fn in variants.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn()
                    times[k].append(1000.0 * (time.perf_counter() - t0) / args.steps)
            for k in variants:
                print(json.dumps({"what": "routed batch", "variant": k, "experts": K, "classes": C, "batch": B,
                                  "mc_samples": T, "ms_per_batch_median": round(statistics.median(times[k]), 4),
                                  "ms_per_batch_min": round(min(times[k]), 4), "batches_per_window": args.steps,
                                  "windows": args.windows, "gpu": gpu, "power_limit": power}), flush=True)
            del lone, steps
        del nets


def reference_route(nets, batches, T, C, dev):
    """predict_using_uncertainty_separate_models for K experts, as the reference writes it: per batch and expert
    get_uncertainty_per_batch (T forwards, softmax, a numpy loop over the images), np.sum, the least uncertain expert
    (ties to the last, `u2 > u1` for K = 2), np.mean of the batch accuracies."""
    import torch.nn.functional as F
    from pytorch_bayesiancnn_b200 import mc
    accs, chosen, scores = [], [], []
    for t, (x, y) in enumerate(batches):
        x = x.to(dev)
        preds, us = [], []
        for net in nets:
            fn = mc.engine_forward_fn(net, SEED, t << 20)
            net_outs, batch_predictions = [], []
            for j in range(T):
                net_out, _ = fn(x, j)
                net_outs.append(net_out)
                batch_predictions.append(F.softmax(net_out, dim=1))
            pr, epis = [], []
            for sample in range(x.shape[0]):
                pred = torch.cat([a[sample].unsqueeze(0) for a in net_outs], dim=0).mean(dim=0)
                pr.append(pred)
                p_hat = torch.cat([a[sample].unsqueeze(0) for a in batch_predictions], dim=0).detach().cpu().numpy()
                p_bar = np.mean(p_hat, axis=0)
                temp = p_hat - np.expand_dims(p_bar, 0)
                epis.append(np.diag(np.dot(temp.T, temp) / T))
            preds.append(torch.cat([p.unsqueeze(0) for p in pr]).cpu().numpy())
            us.append(np.sum(np.vstack(epis), axis=1))
        u = np.stack(us, axis=1)
        e = len(nets) - 1 - np.argmin(u[:, ::-1], axis=1)
        local = np.stack(preds, 1)[np.arange(u.shape[0]), e].argmax(1)
        accs.append(np.mean(e * C + local == y.numpy()))
        chosen.append(e)
        scores.append(u)
    return float(np.mean(accs)), np.concatenate(chosen), np.concatenate(scores)


def loop_bench(args, dev, gpu, power):
    from pytorch_bayesiancnn_b200 import mc
    B, T = 256, 25
    for K in (2, 5):
        C = 10 // K
        nets = experts(K, C, dev)
        g = torch.Generator().manual_seed(0)
        batches = [(torch.rand(B, 1, 32, 32, generator=g), torch.randint(0, K * C, (B,), generator=g))
                   for _ in range(args.batches)]
        first = mc.route(nets, batches, T, seed=SEED)          # steps built; replays 0 .. batches - 1
        ref_acc, ref_e, ref_u = reference_route(nets, batches, T, C, dev)
        got_e = first["per_image"]["expert"].cpu().numpy()
        srt = np.sort(ref_u, axis=1)
        clear = (srt[:, 1] - srt[:, 0]) > 1e-4 * np.abs(srt[:, 1])
        same_all = float(np.mean(got_e == ref_e))
        same_clear = float(np.mean(got_e[clear] == ref_e[clear]))
        variants = {"reference-style loop": lambda: reference_route(nets, batches, T, C, dev),
                    "mc.route": lambda: mc.route(nets, batches, T, seed=SEED)}
        times = {k: [] for k in variants}
        for _ in range(args.windows):
            for k, fn in variants.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                times[k].append(1000.0 * (time.perf_counter() - t0))
        for k in variants:
            print(json.dumps({"what": "route a data set", "variant": k, "experts": K, "classes": C, "batch": B,
                              "mc_samples": T, "batches": args.batches,
                              "ms_median": round(statistics.median(times[k]), 2), "ms_min": round(min(times[k]), 2),
                              "same_decisions": same_all, "same_decisions_clear": same_clear,
                              "clear_share": float(clear.mean()), "accuracy_reference": ref_acc,
                              "local_accuracy_route": first["local_accuracy"], "windows": args.windows, "gpu": gpu,
                              "power_limit": power}), flush=True)
        del nets


def illustrate(args, dev, gpu, power):
    """Two BBBLeNet experts trained briefly on class-disjoint synthetic data (classes 0-4 and 5-9: a class is a fixed
    random image plus noise), then routed on held-out images of both: an illustration, not a gate."""
    from pytorch_bayesiancnn_b200 import mc
    g = torch.Generator().manual_seed(7)
    protos = torch.rand(10, 1, 32, 32, generator=g)

    def draw(classes, n):
        y = torch.tensor(classes)[torch.randint(0, len(classes), (n,), generator=g)]
        return (protos[y] + 0.3 * torch.randn(n, 1, 32, 32, generator=g)).clamp(0, 1), y
    nets = experts(2, 5, dev)
    for k, net in enumerate(nets):
        step = mc.MCTrainStep(net, torch.zeros(128, 1, 32, 32, device=dev), 2, 5000.0, seed=SEED + k)
        opt = torch.optim.Adam(net.parameters(), lr=1e-3)
        for _ in range(200):
            x, y = draw(list(range(5 * k, 5 * k + 5)), 128)
            opt.zero_grad()
            step(x.to(dev), (y - 5 * k).to(dev), beta=1.0 / 5000.0)
            opt.step()
    test = [draw(list(range(10)), 256) for _ in range(8)]
    for score in ("epistemic", "confidence"):
        r = mc.route(nets, test, 10, score=score, log=False, seed=SEED)
        print(json.dumps({"what": "illustration: synthetic split task", "score": score, "accuracy": r["accuracy"],
                          "routing_accuracy": r["routing_accuracy"], "selected": r["selected"], "gpu": gpu,
                          "power_limit": power}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=7)
    ap.add_argument("--launches", type=int, default=100, help="route-kernel launches per captured graph (one window)")
    ap.add_argument("--steps", type=int, default=50, help="routed batches per window of the step arm")
    ap.add_argument("--batches", type=int, default=10, help="host batches of the data-set arm")
    ap.add_argument("--only", default="kernel,step,loop,illustrate")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    dev = torch.device("cuda:0")
    gpu, power = gpu_info()
    only = args.only.split(",")
    for name, fn in (("kernel", kernel_bench), ("step", step_bench), ("loop", loop_bench), ("illustrate", illustrate)):
        if name in only:
            fn(args, dev, gpu, power)


if __name__ == "__main__":
    main()

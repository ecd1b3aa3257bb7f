"""Sample-only against batch-sharded Monte-Carlo steps (MCForward / MCTrainStep ``batch_shards``), alternating window
by window in one job.  Prints one JSON line per measurement with the GPU's name and power limit.

* Under torchrun on >= 2 GPUs: the C4 forward step (BBBAlexNet CIFAR-100, B=1024, 25 samples, LRT, uncertainty) with
  batch_shards 1 and 2 (and world when it divides), and the reference-default training step (num_ens = 1: main_bayesian
  train_ens) of BBBAlexNet CIFAR-10, B=256, with batch_shards 1 and world.  Times are rank 0's, CUDA events, median
  over --windows windows of --steps steps.
* On one GPU a step cannot be split, so it times one rank's SHARE of C4 on 8 ranks as a proxy: the 4 samples x 1024
  rows the busiest rank runs with batch_shards=1, against the 25 samples x 128 rows of batch_shards=8.  This is one
  rank's compute, not a sharded step: it leaves out the exchange over NVLink and the wait for the slowest rank.

    python tools/mc_shard_bench.py [--windows 5] [--steps 5]
    torchrun --nproc-per-node 8 tools/mc_shard_bench.py
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from tools.mc_fold_bench import gpu_info


def _events_ms(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def _alternate(runs, windows, steps, barrier=None):
    """{label: callable one step} -> {label: [ms per step of each window]}, the labels alternating window by window."""
    times = {k: [] for k in runs}
    for fn in runs.values():
        fn()                                            # warm-up
    for _ in range(windows):
        for k, fn in runs.items():
            if barrier is not None:
                barrier()
            times[k].append(_events_ms(lambda: [fn() for _ in range(steps)], steps))
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    import torch.distributed as dist
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if world > 1:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
        dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    dev = torch.device("cuda", torch.cuda.current_device())
    name, power = gpu_info()
    from bench import build_net
    from pytorch_bayesiancnn_b200 import mc

    def report(what, times, **kw):
        if rank == 0:
            for k, t in times.items():
                print(json.dumps({"what": what, "run": k, "ms_per_step_median": round(statistics.median(t), 3),
                                  "ms_per_step_min": round(min(t), 3), "windows": args.windows, "steps": args.steps,
                                  "world": world, **kw, "gpu": name, "power_limit": power}), flush=True)

    net = build_net("lrt", 100, dev, "auto", "alexnet", 3)
    x = torch.randn(1024, 3, 32, 32, device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    if world == 1:
        runs = {"busiest rank, batch_shards=1: 4 samples x 1024 rows": mc.MCForward(net, x, 4, want_uncertainty=True, seed=7),
                "one rank, batch_shards=8: 25 samples x 128 rows": mc.MCForward(net, x[:128].contiguous(), 25,
                                                                                  want_uncertainty=True, seed=7)}
        report("C4 forward, one rank's share on 8 ranks (proxy: no exchange, no wait for other ranks)",
               _alternate(runs, args.windows, args.steps), config="C4")
        return
    shards = [1, 2] + ([world] if world > 2 else [])
    engines = {f"batch_shards={rb}": mc.MCForward(net, x, 25, want_uncertainty=True, seed=7, batch_shards=rb)
               for rb in shards}
    report("C4 forward step", _alternate(engines, args.windows, args.steps, dist.barrier), config="C4")
    for e in engines.values():
        e.close()
    tnet = build_net("lrt", 10, dev, "auto", "alexnet", 3)
    xt = torch.randn(256, 3, 32, 32, device=dev, generator=torch.Generator(device=dev).manual_seed(2))
    yt = torch.randint(0, 10, (256,), device=dev, generator=torch.Generator(device=dev).manual_seed(3))
    steps = {f"batch_shards={rb}": mc.MCTrainStep(tnet, xt, 1, train_size=50000.0, seed=7, batch_shards=rb)
             for rb in (1, world)}
    calls = {k: (lambda s=s: s(xt, yt, beta=0.1)) for k, s in steps.items()}
    report("training step, num_ens = 1", _alternate(calls, args.windows, args.steps, dist.barrier), batch=256)
    for s in steps.values():
        s.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

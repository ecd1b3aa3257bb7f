"""Cost of the logit gather that fills sample banks from sharded Monte-Carlo steps (bbb_mc_logit_gather), on one GPU.

* gather: the kernel on `world` emulated ranks of one device (a receive buffer, a state and a stream per rank), every
  rank's launch of a window enqueued before the one synchronise that ends it; time per launch = host time of the window
  / launches.  At the C3-like (10, 512, 10), C4-like (25, 1024, 100) and C5 (100, 2048, 10) shapes.  Bytes per launch,
  over all ranks: every rank stores each of its words into every rank's buffer (world x S B C 8-byte words in all),
  every rank reads its S B C words back and writes S B C fp32, and the ranks read their S B C fp32 logits once between
  them.  These are LOCAL-memory figures: the emulated ranks' stores go to HBM / L2 of the one device, not over NVLink;
* step: a one-rank C3-like step (BBBAlexNet-10, B = 512, 10 samples, four in flight) with a ProbBank made without a
  group and with a one-rank group, alternating window by window: the same kernels run (nothing is gathered on one rank).

Prints one JSON line per measurement with the GPU's name and power limit.

    python tools/bank_gather_bench.py [--windows 5] [--launches 50] [--steps 50] [--worlds 2,4,8] [--only gather,step]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from tools.mc_fold_bench import gpu_info

SHAPES = {"C3-like": (10, 512, 10), "C4-like": (25, 1024, 100), "C5": (100, 2048, 10)}


def gather_windows(dev, world, S, B, Cc, launches, windows):
    """Seconds per launch of each window: `launches` gathers of every emulated rank (sample-only split)."""
    from pytorch_bayesiancnn_b200 import _lib as L, functional as Fn, mc
    lib = L.lib()
    nbytes = int(lib.bbb_mc_gather_bytes(S, B, Cc))
    bufs = [torch.zeros(nbytes, dtype=torch.uint8, device=dev) for _ in range(world)]
    peers = (C.c_void_p * world)(*[b.data_ptr() for b in bufs])
    states = [torch.zeros(int(lib.bbb_mc_state_bytes()), dtype=torch.uint8, device=dev) for _ in range(world)]
    streams = [torch.cuda.Stream(device=dev) for _ in range(world)]
    full = torch.randn(S, B, Cc, device=dev)
    mine = [full[mc.local_samples(S, world, r)].contiguous() if r < S else None for r in range(world)]
    outs = [torch.empty(S, B, Cc, device=dev) for _ in range(world)]

    def run(n):
        for _ in range(n):
            for r in range(world):
                lg = mine[r]
                with torch.cuda.stream(streams[r]):
                    L.check(lib.bbb_mc_logit_gather(Fn._ptr(lg), 0 if lg is None else lg.shape[0], S, B, Cc, r, world,
                                                    1, peers, Fn._ptr(states[r]), Fn._ptr(outs[r]),
                                                    Fn._stream(dev)), "bbb_mc_logit_gather")
        torch.cuda.synchronize()
    run(3)
    res = []
    for _ in range(windows):
        t0 = time.perf_counter()
        run(launches)
        res.append((time.perf_counter() - t0) / launches)
    assert all(int(st[8:12].view(torch.int32).item()) == 0 for st in states), "a gather wait timed out"
    assert all(torch.equal(o, full) for o in outs)
    return res


def step_windows(dev, steps, windows):
    """Milliseconds per step of a one-rank C3-like step with a ProbBank of no group and of a one-rank group,
    alternating window by window."""
    import torch.distributed as dist
    from pytorch_bayesiancnn_b200 import mc, models as M
    from oracle import bbb_oracle as O
    from tests.util import CFG_PRIORS, load_params_into
    dist.init_process_group("gloo", init_method="file://" + os.path.join(tempfile.mkdtemp(), "pg"), rank=0,
                            world_size=1)
    params = O.init_params("alexnet", 10, 3, CFG_PRIORS, seed=123)
    net = load_params_into(M.BBBAlexNet(10, 3, CFG_PRIORS, "lrt", "softplus"), params).to(dev).train()
    net.set_flag("math", "auto")
    B, S = 512, 10
    xs = [torch.randn(B, 3, 32, 32, device=dev) for _ in range(4)]
    arms = {}
    for name, group in (("no group", None), ("one-rank group", dist.group.WORLD)):
        bank = mc.ProbBank(dev, steps * B, S, 10, group=group)
        eng = mc.MCForward(net, xs[0], S, seed=3, static_inputs=xs, overlap=True, inflight=4, prob_bank=bank)
        arms[name] = (eng, bank)
    res = {k: [] for k in arms}
    for _ in range(windows):
        for name, (eng, bank) in arms.items():
            bank.reset()
            for i in range(4):
                eng(slot=i % 4)
            eng.wait()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(steps):
                eng(slot=i % 4)
            eng.wait()
            torch.cuda.synchronize()
            res[name].append((time.perf_counter() - t0) / steps * 1e3)
    kps = {name: eng.kernels_per_step for name, (eng, _) in arms.items()}
    dist.destroy_process_group()
    return res, kps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--worlds", default="2,4,8")
    ap.add_argument("--only", default="gather,step")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bank_gather_bench: needs a CUDA device")
    import __graft_entry__ as g
    g.build()
    dev = torch.device("cuda:0")
    name, power = gpu_info()
    only = set(a.only.split(","))
    if "gather" in only:
        for world in (int(w) for w in a.worlds.split(",")):
            for label, (S, B, Cc) in SHAPES.items():
                t = gather_windows(dev, world, S, B, Cc, a.launches, a.windows)
                words = S * B * Cc
                moved = world * words * 8 + world * words * 8 + world * words * 4 + words * 4
                med = statistics.median(t)
                print(json.dumps({"what": "gather, emulated ranks (local memory, not NVLink)", "shape": label,
                                  "S": S, "B": B, "C": Cc, "world": world, "us_per_launch": med * 1e6,
                                  "spread_us": [min(t) * 1e6, max(t) * 1e6], "bytes_per_launch": moved,
                                  "GB_per_s": moved / med / 1e9, "gpu": name, "power_limit": power}), flush=True)
    if "step" in only:
        res, kps = step_windows(dev, a.steps, a.windows)
        for arm, t in res.items():
            print(json.dumps({"what": "one-rank C3-like step with a ProbBank", "bank": arm, "ms_per_step":
                              statistics.median(t), "windows_ms": t, "kernels_per_step": kps[arm], "gpu": name,
                              "power_limit": power}), flush=True)


if __name__ == "__main__":
    main()

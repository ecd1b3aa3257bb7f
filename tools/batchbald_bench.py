"""Cost of active-learning selection on one GPU, in one job, with the GPU's name and power limit on every line.

* kernel: bbb_joint_entropy alone, one greedy round's scoring, at the MNIST-like (N=60000, S=100, C=10, M=10000) and
  CIFAR-100-like (N=10000, S=20, C=100, M=1000) shapes; FLOP/s and logarithms/s (M N C) against the tf32 MMA rate
  (495 TFLOP/s dense) and the SFU rate (16 per clock per SM).  Two FLOP counts: useful (2 M S N C, the product of the
  unpadded operands) and executed (2 M_pad S_pad N_pad C_pad, what the tensor cores multiply: S padded to 8, C to a
  power of two, M to 64, N to whole 128-column tiles); the MMA bound is given for both;
* select: a whole batchbald(k=10) against the same algorithm with a torch scorer -- chunked float32 matmul (tf32 off)
  or float64 matmul of Pt and the bank, then q log q and the weighted sums in float64 -- alternating, on the same
  configurations (same seed, the same update code): time, whether the indices agree, the largest score difference;
* bank: the MCForward step with and without a probability bank, alternating: C5 (BBB3Conv3FC-10, B=2048, 100
  samples, one step at a time) and headline-like (BBBAlexNet-10, B=512, 1 sample, four steps in flight).

    python tools/batchbald_bench.py [--windows 5] [--only kernel,select,bank] [--select-pool 20000]
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

KERNEL_SHAPES = {"MNIST-like": (60000, 100, 10, 10000), "CIFAR-100-like": (10000, 20, 100, 1000)}


def _random_bank(dev, N, S, C, seed=0):
    from pytorch_bayesiancnn_b200 import mc
    bank = mc.ProbBank(dev, N, S, C)
    g = torch.Generator(device=dev).manual_seed(seed)
    for i0 in range(0, N, 4096):
        n = min(4096, N - i0)
        bank.append(torch.randn(S, n, C, device=dev, generator=g) * 3)
    torch.cuda.synchronize()
    return bank


def _sm_clock_ghz():
    import subprocess
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, check=True).stdout.split()[0]
        return float(out) / 1000.0
    except Exception:
        return 1.98


def kernel_bench(args, dev, gpu, power):
    from pytorch_bayesiancnn_b200 import mc
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    ghz = _sm_clock_ghz()
    for name, (N, S, C, M) in KERNEL_SHAPES.items():
        bank = _random_bank(dev, N, S, C)
        g = torch.Generator(device=dev).manual_seed(1)
        w = torch.rand(M, S, device=dev, dtype=torch.float64, generator=g) ** 4
        pt = w / w.sum(1, keepdim=True)
        om = torch.full((M,), 1.0 / M, device=dev, dtype=torch.float64)
        sc = mc._Scorer(bank, N, M)
        sc(pt, om)
        reps = 3
        times = [_events_ms(lambda: [sc(pt, om) for _ in range(reps)], reps) for _ in range(args.windows)]
        # the tf32 / omega copies of _Scorer run in the timed window too: time them alone and take them out
        copy = [_events_ms(lambda: [sc.pt[:M, :S].copy_(mc._tf32(pt)) for _ in range(reps)], reps)
                for _ in range(args.windows)]
        ms = statistics.median(times) - statistics.median(copy)
        flop, logs = 2.0 * M * S * N * C, float(M) * N * C
        cand = 128 // bank.C_pad
        flop_x = 2.0 * (-(-M // 64) * 64) * bank.S_pad * (-(-N // cand) * 128)
        t_mma, t_mma_x, t_sfu = flop / 495e12, flop_x / 495e12, logs / (16 * sms * ghz * 1e9)
        print(json.dumps({"what": "joint-entropy kernel, one round", "shape": name, "N": N, "S": S, "C": C, "M": M,
                          "ms_median": round(ms, 3), "ms_min_with_pt_copy": round(min(times), 3),
                          "useful_tflops": round(flop / ms / 1e9, 1), "executed_tflops": round(flop_x / ms / 1e9, 1),
                          "glogs_per_s": round(logs / ms / 1e6, 1), "mma_bound_useful_ms": round(1e3 * t_mma, 3),
                          "mma_bound_executed_ms": round(1e3 * t_mma_x, 3), "sfu_bound_ms": round(1e3 * t_sfu, 3),
                          "binding_bound": "tf32 MMA" if t_mma_x > t_sfu else "SFU log",
                          "share_of_binding_bound_executed": round(1e3 * max(t_mma_x, t_sfu) / ms, 3), "sms": sms,
                          "sm_clock_ghz": ghz, "windows": args.windows, "gpu": gpu, "power_limit": power}),
              flush=True)
        del bank, sc


class _TorchScorer:
    """The scorer of mc._Scorer in torch: Q = Pt (tf32 values) @ bank chunk as a float32 (tf32 off) or float64 matmul,
    -q log q over the real classes, weighted sum over m in float64."""

    def __init__(self, inner, chunk, dtype):
        self.inner, self.chunk, self.dtype = inner, chunk, dtype
        self.mask, self.bank = inner.mask, inner.bank

    def __call__(self, pt64, omega64):
        from pytorch_bayesiancnn_b200 import mc
        b, n = self.bank, self.inner.n
        S, C = b.num_ens, b.num_classes
        pt = mc._tf32(pt64).to(self.dtype)
        out = torch.empty(n, dtype=torch.float64, device=b.device)
        for i0 in range(0, n, self.chunk):
            i1 = min(n, i0 + self.chunk)
            q = pt @ b._probs[i0:i1, :C, :S].reshape(-1, S).T.to(self.dtype)     # [M, chunk * C]
            h = -torch.special.xlogy(q.clamp_min(0), q.clamp_min(0)).view(q.shape[0], i1 - i0, C).sum(2)
            out[i0:i1] = omega64 @ h.double()
        return out.masked_fill_(self.mask.bool(), float("-inf"))


def select_bench(args, dev, gpu, power):
    from pytorch_bayesiancnn_b200 import mc
    N, S, C = args.select_pool, 100, 10
    bank = _random_bank(dev, N, S, C, seed=3)
    torch.backends.cuda.matmul.allow_tf32 = False
    orig = mc._Scorer

    kinds = {"kernel": None, "torch-float32": torch.float32, "torch-float64": torch.float64}

    def run(kind):
        dt = kinds[kind]
        mc._Scorer = orig if dt is None else (lambda b, n, m: _TorchScorer(orig(b, n, m), args.chunk, dt))
        try:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = mc.batchbald(bank, 10, num_configs=10000, seed=5)
            torch.cuda.synchronize()
            return r, 1000.0 * (time.perf_counter() - t0)
        finally:
            mc._Scorer = orig
    res = {k: run(k)[0] for k in kinds}
    times = {k: [] for k in kinds}
    for _ in range(args.windows):
        for k in times:
            res[k], t = run(k)
            times[k].append(t)
    ref = res["torch-float64"]
    for k in times:
        same = torch.equal(res[k]["indices"], ref["indices"])
        first = next((i for i in range(10) if res[k]["indices"][i] != ref["indices"][i]), 10)
        diff = float((res[k]["scores"][:first] - ref["scores"][:first]).abs().max()) if first else None
        print(json.dumps({"what": "batchbald k=10", "scorer": k, "N": N, "S": S, "C": C, "num_configs": 10000,
                          "ms_median": round(statistics.median(times[k]), 2), "ms_min": round(min(times[k]), 2),
                          "indices_agree_with_float64": same, "rounds_agreeing": first,
                          "max_score_diff_vs_float64": diff, "exact_rounds": res[k]["exact"],
                          "windows": args.windows, "gpu": gpu, "power_limit": power}), flush=True)
    del bank


def bank_bench(args, dev, gpu, power):
    from bench import build_net
    from pytorch_bayesiancnn_b200 import mc
    for name, (key, inputs, B, S, inflight, steps) in {"C5": ("3conv3fc", 1, 2048, 100, 1, 4),
                                                        "headline-like": ("alexnet", 3, 512, 1, 4, 100)}.items():
        net = build_net("lrt", 10, dev, "auto", key, inputs)
        xs = [torch.randn(B, inputs, 32, 32, device=dev) for _ in range(4)]
        banks = {False: None, True: mc.ProbBank(dev, steps * B, S, 10)}
        kw = dict(seed=2024, static_inputs=xs, overlap=inflight > 1, inflight=inflight)
        engines = {m: mc.MCForward(net, xs[0], S, prob_bank=banks[m], **kw) for m in (False, True)}

        def run(m):
            def go():
                if banks[m] is not None:
                    banks[m].reset()
                for i in range(steps):
                    engines[m](slot=i % len(xs))
                engines[m].wait()
            return go
        for m in (False, True):
            run(m)()
        times = {False: [], True: []}
        for _ in range(args.windows):
            for m in (False, True):
                times[m].append(_events_ms(run(m), steps))
        assert len(banks[True]) == steps * B and banks[True].dropped == 0
        same = all(torch.equal(engines[False].out[k], engines[True].out[k]) for k in engines[False].out)
        for m in (False, True):
            print(json.dumps({"what": "MCForward step", "workload": name, "batch": B, "mc_samples": S,
                              "inflight": inflight, "prob_bank": m,
                              "ms_per_step_median": round(statistics.median(times[m]), 4),
                              "ms_per_step_min": round(min(times[m]), 4), "steps_per_window": steps,
                              "outputs_bitwise_equal": same, "windows": args.windows, "gpu": gpu,
                              "power_limit": power}), flush=True)
        del engines, net, banks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--only", default="kernel,select,bank")
    ap.add_argument("--select-pool", type=int, default=20000)
    ap.add_argument("--chunk", type=int, default=2000, help="candidates per matmul of the torch scorer")
    args = ap.parse_args()
    import __graft_entry__ as g
    g.build()
    dev = torch.device("cuda:0")
    gpu, power = gpu_info()
    only = args.only.split(",")
    if "kernel" in only:
        kernel_bench(args, dev, gpu, power)
    if "select" in only:
        select_bench(args, dev, gpu, power)
    if "bank" in only:
        bank_bench(args, dev, gpu, power)


if __name__ == "__main__":
    main()

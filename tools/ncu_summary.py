#!/usr/bin/env python
"""Turn an `ncu --set full` report into two small files:

    python tools/ncu_summary.py prof.ncu-rep ncu_fwd

writes <out>_summary.csv (one row per captured launch, the columns below) and, when the capture holds
exactly the six GEMM kernels of one BBBAlexNet forward (conv1..conv5, classifier, in launch order),
<out>_traffic.json = per-layer DRAM bytes (read + write) per launch, to set against the algorithmic bytes of
bench.py's `per_layer` rows.  Needs the `ncu` CLI (reads the report; no GPU)."""
import csv
import io
import json
import subprocess
import sys

COLS = ["Kernel Name", "Block Size", "Grid Size", "dram__bytes_read.sum", "dram__bytes_write.sum",
        "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed", "gpu__time_duration.sum",
        "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum", "launch__registers_per_thread",
        "launch__shared_mem_per_block_dynamic", "launch__occupancy_limit_shared_mem",
        "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
        "sm__throughput.avg.pct_of_peak_sustained_elapsed", "sm__warps_active.avg.pct_of_peak_sustained_active",
        "smsp__inst_executed.sum", "smsp__pcsamp_warps_issue_stalled_barrier",
        "smsp__pcsamp_warps_issue_stalled_long_scoreboard", "smsp__pcsamp_warps_issue_stalled_no_instructions",
        "smsp__pcsamp_warps_issue_stalled_sleeping", "smsp__pcsamp_warps_issue_stalled_wait"]
LAYERS = ["conv1", "conv2", "conv3", "conv4", "conv5", "classifier"]
UNIT = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}
TIME = {"ns": 1e-3, "us": 1.0, "ms": 1e3, "s": 1e6}


def main(rep, out, variant="lrt", batch=512):
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], check=True, capture_output=True,
                         text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    head, units, body = rows[0], rows[1], rows[2:]
    idx = {c: head.index(c) for c in COLS if c in head}
    with open(out + "_summary.csv", "w", newline="") as f:
        w = csv.writer(f)
        w.writerow(list(idx))
        w.writerow([units[i] for i in idx.values()])
        for r in body:
            w.writerow([r[i] for i in idx.values()])
    print(f"{out}_summary.csv: {len(body)} launches")
    if len(body) != len(LAYERS):
        print("not a six-GEMM capture: no traffic file written")
        return

    def val(r, col, table):
        i = idx[col]
        return float(r[i].replace(",", "")) * table[units[i]]
    layers = {}
    for name, r in zip(LAYERS, body):
        layers[name] = {
            "kernel": r[idx["Kernel Name"]], "grid": r[idx["Grid Size"]],
            "dram_bytes": val(r, "dram__bytes_read.sum", UNIT) + val(r, "dram__bytes_write.sum", UNIT),
            "kernel_us": val(r, "gpu__time_duration.sum", TIME),
            "tensor_pipe_pct": float(r[idx["sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active"]]),
        }
    src = (f"ncu --set full --clock-control none, {out}_summary.csv (GEMM kernel of each layer; BBBAlexNet "
           f"B={batch} {variant.upper()} bf16 fused chain)")
    with open(out + "_traffic.json", "w") as f:
        json.dump({"source": src, "variant": variant, "batch": batch, "layers": layers}, f, indent=1)
    print(f"{out}_traffic.json written")


if __name__ == "__main__":
    main(*sys.argv[1:3])

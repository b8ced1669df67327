#!/usr/bin/env python
"""bench_solver.py -- SGD and Adam solvers side by side on CaffeNet b256, one GPU.

  python bench_solver.py [--runs 3] [--steps 50] [--warmup 10] [--out FILE]

--runs runs of each solver, alternated, each one bench.py's measure_workload (the same device-timed steps, L2 flush
and forward/backward split as bench.py, so the numbers compare with DESIGN.md section 5) on a net whose solver is
SGD (CaffeNet's own hyper-parameters) or Adam (the same base_lr, policy, momentum = beta1, weight decay;
momentum2 0.999, delta 1e-8).  Reports the median and [min, max] of images/s, ms per step, the fused kernel's time
inside the step and back to back, and that kernel's achieved HBM bandwidth on its minimum traffic: 24P bytes for
SGD (read g, w, h; write w, h; zero g) and 32P for Adam (read g, w, m, v; write w, m, v; zero g), against the card's
data-sheet bandwidth.  The card name, power limit and maximum SM clock are read in the same process.

Prints one JSON line; writes nothing in the tree (--out names the file to write, if any).
"""
import argparse
import json
import os
import sys
import tempfile
import types

import bench  # measure_workload, emit; its import sends everything but the JSON line to stderr
from bench_producer_precision import card, stats

WORKLOAD = "caffenet"
SOLVERS = ("SGD", "Adam")
BYTES_PER_PARAM = {"SGD": 24, "Adam": 32}


def nets_for(nets, solver):
    """The nets module with solver_desc() returning `solver` (everything else unchanged)."""
    if solver == "SGD":
        return nets
    shim = types.SimpleNamespace(**vars(nets))
    shim.solver_desc = lambda name, **kw: nets.solver_desc(name, type="Adam", momentum2=0.999, delta=1e-8, **kw)
    return shim


def timing(args):
    import torch
    import torch.distributed as dist
    import caffeonspark_b200 as C
    from caffeonspark_b200 import harness, nets
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.allow_tf32 = True
    keys = ("images_per_s", "ms_per_step", "sync_kernel_in_step_ms", "sync_kernel_back_to_back_ms")
    res = {s: {k: [] for k in keys} for s in SOLVERS}
    clocks = {s: [] for s in SOLVERS}
    bargs = argparse.Namespace(algo=0, kernel=-1, nvls=-1, no_graph=False, steps=args.steps, warmup=args.warmup,
                               dump_outputs="", no_cpu_baseline=True)
    P = nets.solver_desc(WORKLOAD).param_count
    with tempfile.TemporaryDirectory() as tmp:
        for r in range(args.runs):
            for s in SOLVERS:
                bargs.dump_outputs = os.path.join(tmp, f"{s}_{r}")
                out, _ = bench.measure_workload(torch, dist, C, harness, nets_for(nets, s), bargs, WORKLOAD, "fp32",
                                                0, 1, 0, primary=True)
                d = res[s]
                d["images_per_s"].append(out["value"])
                d["ms_per_step"].append(out["ms_per_step"])
                d["sync_kernel_in_step_ms"].append(out["split_ms"]["fused_sync_kernel"])
                d["sync_kernel_back_to_back_ms"].append(out["roofline"]["kernel_ms_back_to_back"])
                clocks[s].append(out.get("clocks"))
                print(f"[solver] {s} run {r}: {out['value']:.0f} images/s, {out['ms_per_step']:.3f} ms/step, "
                      f"sync kernel {out['split_ms']['fused_sync_kernel'] * 1e3:.1f} us in step, "
                      f"{out['roofline']['kernel_ms_back_to_back'] * 1e3:.1f} us back to back", file=sys.stderr,
                      flush=True)
    summary = {}
    for s in SOLVERS:
        summary[s] = {k: stats(v) for k, v in res[s].items()}
        nbytes = BYTES_PER_PARAM[s] * P
        for k in ("sync_kernel_in_step_ms", "sync_kernel_back_to_back_ms"):
            ms = summary[s][k]["median"]
            gbs = nbytes / (ms * 1e-3) / 1e9
            summary[s][k.replace("_ms", "_achieved_gbs")] = gbs
            summary[s][k.replace("_ms", "_frac_of_hbm_peak")] = gbs / bench.HBM_PEAK_GBS
        summary[s]["minimum_bytes"] = nbytes
        summary[s]["clocks"] = clocks[s]
    return {"workload": f"{WORKLOAD} b256, N=1", "P": P, "runs": args.runs, "steps": args.steps,
            "warmup": args.warmup, "hbm_peak_gbs_datasheet": bench.HBM_PEAK_GBS, "solvers": summary}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_solver.py needs a CUDA device (there is no CPU path)")
    res = {"card": card(), **timing(args)}
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    bench.emit(res)


if __name__ == "__main__":
    main()

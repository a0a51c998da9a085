"""Latency of the serial against the time-parallel (segmented) Riccati sweeps at small batch sizes.

In one process, alternating serial and segmented settings on the same handle and inputs, three runs each:
  * rbt_riccati_backward + rbt_riccati_forward, CUDA events over many launches after a warm-up;
  * the whole step-by-step iteration (condense, backward, forward, expand, update).
ANYmal trot N=40 at batch 1 .. 132 and 1024 (control); a sweep over the segment count at batch 1 and 16.  Prints the card
name and power limit beside the numbers.

    python tools/time_parallel_latency.py [--reps 200] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from helpers import trot_schedule  # noqa: E402
from robotoc_b200 import (ANYMAL, DirectMultipleShooting, Layout, RiccatiRecursion, StageDims, StageLayout,  # noqa: E402
                          anymal_constraint_table)
from synth import make_kkt, make_stage_inputs, symmetrize_lin  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, reps, warm):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps * 1e3  # us per call


def sweep_case(ctrl, batch, settings, reps, runs=3):
    dims, L = ANYMAL, Layout(ANYMAL)
    kkt, dx0 = make_kkt(dims, L, ctrl, batch=batch, seed=1)
    rr = RiccatiRecursion(dims, len(ctrl), batch)
    rr.setTimeDiscretization(ctrl)
    rr.backwardRiccatiRecursion(kkt)
    rr.forwardRiccatiRecursion(dx0)
    lib, h = rr._lib, rr._h

    def step():
        lib.rbt_riccati_backward(h, 0, None)
        lib.rbt_riccati_forward(h, None)

    def bwd():
        lib.rbt_riccati_backward(h, 0, None)

    out = {s: {"sweeps_us": [], "bwd_us": []} for s in settings}
    for _ in range(runs):
        for s in settings:
            rr.setTimeSegments(s)
            out[s]["sweeps_us"].append(timed(step, reps, 10))
            out[s]["bwd_us"].append(timed(bwd, reps, 10))
    rr.close()
    return out


def iteration_case(ctrl, batch, settings, reps, runs=3):
    table = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=table.n_contacts, n_box=table.n_box)
    S = StageLayout(sd)
    lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, batch, 2)
    lin = symmetrize_lin(S, lin)
    rr = RiccatiRecursion(ANYMAL, len(ctrl), batch)
    rr.setTimeDiscretization(ctrl)
    dms = DirectMultipleShooting(rr, sd, table)
    dms.condense(lin, con)
    dms.setSolution(sol)
    lib, h = rr._lib, rr._h
    rr.forwardRiccatiRecursion(dx0)

    def it():
        lib.rbt_condense(h, None)
        lib.rbt_riccati_backward(h, 0, None)
        lib.rbt_riccati_forward(h, None)
        lib.rbt_expand_and_step_sizes(h, None)

    out = {s: [] for s in settings}
    for _ in range(runs):
        for s in settings:
            rr.setTimeSegments(s)
            out[s].append(timed(it, reps, 5))
    rr.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--out", default="")
    ap.add_argument("--batches", default="1,2,4,8,16,32,64,132,1024")
    ap.add_argument("--segments", default="4,8,12")
    ap.add_argument("--sweep", default="2,3,4,6,8,12,16,23,46")
    args = ap.parse_args()
    torch.cuda.init()
    print("card:", card(), flush=True)
    ctrl = trot_schedule(40)[2]
    res = {"card": card(), "schedule": "trot N=40 (47 grid points)", "table": {}, "sweep": {}, "iteration": {}}
    cand = [int(x) for x in args.segments.split(",")]
    for batch in [int(x) for x in args.batches.split(",")]:
        reps = args.reps if batch <= 132 else max(10, args.reps // 20)
        r = sweep_case(ctrl, batch, [1] + cand, reps)
        it = iteration_case(ctrl, batch, [1] + cand, max(10, reps // 2))
        res["table"][batch] = {s: r[s] for s in r}
        res["iteration"][batch] = it
        line = " ".join(f"S={s}: {np.median(r[s]['sweeps_us']):8.1f} (bwd {np.median(r[s]['bwd_us']):7.1f}) it {np.median(it[s]):8.1f}"
                        for s in r)
        print(f"batch {batch:5d}  us  {line}", flush=True)
    for batch in (1, 16):
        sw = [int(x) for x in args.sweep.split(",")]
        r = sweep_case(ctrl, batch, [1] + sw, args.reps)
        res["sweep"][batch] = r
        line = " ".join(f"S={s}: {np.median(r[s]['sweeps_us']):.1f}/{np.median(r[s]['bwd_us']):.1f}" for s in r)
        print(f"sweep batch {batch}: sweeps/bwd us  {line}", flush=True)
    print("card:", card(), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1, default=str)


if __name__ == "__main__":
    main()

"""Cost of computing the state-equation rows on the device, ANYmal trot N=40 at batch 1024.

In one process:
  * linearize_state_equation_kernel alone: CUDA events over 200 launches after a warm-up;
  * the H2D bytes rbt_iteration_host_bytes(h, 2, ..) reports with RBT_WIRE_DEVICE_ID | RBT_WIRE_DEVICE_CONTACT, without and with
    RBT_WIRE_DEVICE_STATE;
  * the resident iteration (rbt_iteration_host_resident, pinned host buffers) in both settings, alternating, three runs each:
    host clock around calls that end synchronised;
  * the card name, power limit and maximum SM clock, read in the same call.

    python tools/state_equation_timing.py [--batch 1024] [--reps 20] [--out DIR]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import contact_ref  # noqa: E402
import state_ref  # noqa: E402
import make_model_fixture  # noqa: E402
import rbd_ref  # noqa: E402
from helpers import trot_schedule  # noqa: E402
from robotoc_b200 import ANYMAL, DirectMultipleShooting, RiccatiRecursion, StageDims, StageLayout, anymal_constraint_table  # noqa: E402
from synth import make_stage_inputs, symmetrize_lin  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="", help="directory for state_equation_timing.json")
    args = ap.parse_args()
    torch.cuda.init()
    res = {"card": card(), "schedule": "trot N=40", "batch": args.batch}
    print("card:", res["card"], flush=True)
    ctrl = trot_schedule(40)[2]
    table = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=table.n_contacts, n_box=table.n_box)
    S = StageLayout(sd)
    lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, args.batch, 2)
    lin = symmetrize_lin(S, lin)
    rr = RiccatiRecursion(ANYMAL, len(ctrl), args.batch)
    rr.setTimeDiscretization(ctrl)
    dms = DirectMultipleShooting(rr, sd, table)
    dms.setRobotModel(rbd_ref.to_c(make_model_fixture.load()))
    dms.setContactGains(contact_ref.random_gains(3, table.n_contacts))
    dms.setContactPositions(contact_ref.random_positions(4, args.batch, len(ctrl), table.n_contacts))
    dms.condense(lin, con)
    dms.setSolution(sol)
    dms.setInitialConfiguration(state_ref.random_q0(5, args.batch, S.nq))
    lib, h = rr._lib, rr._h

    # kernel alone
    for _ in range(10):
        lib.rbt_linearize_state_equation(h, None)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 200
    a.record()
    for _ in range(n):
        lib.rbt_linearize_state_equation(h, None)
    b.record()
    b.synchronize()
    res["kernel_ms"] = a.elapsed_time(b) / n
    print(f"linearize_state_equation_kernel: {res['kernel_ms']:.4f} ms per launch", flush=True)

    # resident iteration (device ID and contact rows), host-computed vs device-computed state-equation rows
    res_in = np.ascontiguousarray(con[:, :, S.c_res:S.c_res + S.ncp])
    wires, h2d = {}, {}
    for mode, flag in (("host_state", False), ("device_state", True)):
        dms.setWireCostStructure(False, device_inverse_dynamics=True, device_contact_kinematics=True, device_state_equation=flag)
        wires[mode] = dms.pack_wire(lin)
        h2d[mode] = dms.iteration_host_bytes(resident=True)[0]
    res["h2d_bytes"] = h2d
    print("H2D bytes per iteration:", h2d, f"({100 * (1 - h2d['device_state'] / h2d['host_state']):.1f} % less)", flush=True)

    def pinned(a):
        t = torch.empty(a.shape, dtype=torch.float64, pin_memory=True).numpy()
        t[...] = a
        return t

    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    wires = {k: pinned(w) for k, w in wires.items()}
    lin_p, res_p, dx0_p = pinned(lin), pinned(res_in), pinned(dx0)
    sol_out, sd_out = pinned(np.zeros_like(sol)), pinned(np.zeros((args.batch, len(ctrl), 2 * S.ncp)))
    steps_out = pinned(np.zeros((args.batch, 2)))

    def resident(mode):
        rc = lib.rbt_iteration_host_resident(h, P(wires[mode]), P(lin_p), P(res_p), P(dx0_p), P(sol_out), P(sd_out), P(steps_out),
                                             None)
        assert rc == 0, rr._err()
        lib.rbt_sync(h, None)

    times = {"host_state": [], "device_state": []}
    for _ in range(3):
        for mode in ("host_state", "device_state"):
            dms.setWireCostStructure(False, device_inverse_dynamics=True, device_contact_kinematics=True,
                                     device_state_equation=(mode == "device_state"))
            dms.setSolution(sol)
            dms.setConstraintData(con)
            for _ in range(3):
                resident(mode)
            t0 = time.perf_counter()
            for _ in range(args.reps):
                resident(mode)
            times[mode].append((time.perf_counter() - t0) / args.reps * 1e3)
            print(f"resident iteration {mode}: {times[mode][-1]:.3f} ms", flush=True)
    res["iteration_ms"] = times
    res["card_after"] = card()
    print("card:", res["card_after"], flush=True)
    rr.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "state_equation_timing.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

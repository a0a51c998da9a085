"""Generates tests/golden/golden_ref_ustage.npz: full iterations of the unconstrained (fixed-base, iiwa14) path computed by the
reference's own code (tests/ref_lib.unconstr_iteration: robotoc's UnconstrDynamics, joint-limit constraint components,
SplitSolution and UnconstrRiccatiRecursion compiled unmodified, oracle/Makefile.ref), on the cases of CASES; a fixed, seeded
sample of every section of every record (golden_sample.py), the step sizes whole.  Only runs where a robotoc source tree exists:
    ROBOTOC_REFERENCE=<robotoc source tree> python tests/golden/make_golden_ref_ustage.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)

from synth import bind_unconstr_rows, iiwa14_rows, make_unconstr_stage_inputs, unconstr_table  # noqa: E402
from golden_sample import groups, layout_bounds, put  # noqa: E402

PATH = os.path.join(HERE, "golden_ref_ustage.npz")
NV = 7
FRAC = 0.2  # share of the nonzero entries of every record section that is stored
KEYS = ("kkt", "ex", "con_condensed", "dir", "xd", "steps", "con_expanded", "con", "sol")

# Binding rows of the "bind" case (synth.bind_unconstr_rows), N = 20, batch 3: the primal step of OCP 0 binds on a torque row
# of grid 0, that of OCP 1 on a velocity row of grid 1, that of OCP 2 on grid N - 1; the dual steps bind elsewhere.
BINDS = [(0, 0, 30, "p"), (0, 5, 16, "d"), (1, 1, 20, "p"), (1, 0, 40, "d"), (2, 19, 3, "p"), (2, 1, 22, "d")]
# (b, i, r): a position row on grid 0 whose fraction to boundary would be far below every step if it were counted
GATED = [(0, 0, 2)]

# name -> (acceleration limits, N, batch, dt, seed, binds).  N = 1 and N = 2 end inside the grid points where joint limits
# are partly off (grid 0: torque rows only; grid 1: velocity and torque rows).
CASES = {
    "n20": (False, 20, 2, 0.05, 401, False),
    "n50": (False, 50, 3, 0.02, 402, False),
    "n1": (False, 1, 2, 0.05, 403, False),
    "n2": (False, 2, 2, 0.05, 404, False),
    "n3": (False, 3, 2, 0.05, 405, False),
    "acc": (True, 20, 2, 0.05, 406, False),  # + joint acceleration limits: 56 rows, two 32-lane passes
    "bind": (False, 20, 3, 0.05, 407, True),
}


def gate_would_bind(S, con, gated):
    con = con.copy()
    for b, i, r in gated:
        con[b, i, S.c_slack + r] = 1.0e-6
        con[b, i, S.c_dual + r] = 1.0e-4
        con[b, i, S.c_res + r] = 100.0
    return con


def problem(name, S_getter=None):
    from robotoc_b200.unconstr_dms import UStageLayout
    acc, N, batch, dt, seed, bind = CASES[name]
    tab = unconstr_table(iiwa14_rows(NV, acceleration_limits=acc))
    S = UStageLayout(NV, tab.n_box, getter=S_getter)
    lin, con, sol, dx0 = make_unconstr_stage_inputs(S, N, batch, seed)
    if bind:
        con = gate_would_bind(S, bind_unconstr_rows(S, con, BINDS), GATED)
    return tab, S, N, dt, lin, con, sol, dx0


def record_groups(a, key, S, UL):
    prefix = {"kkt": "k_", "dir": "d_", "ex": "e_", "xd": "x_", "sol": "s_", "con_condensed": "c_", "con_expanded": "c_",
              "con": "c_"}[key]
    return groups(a, layout_bounds(UL if prefix in ("k_", "d_") else S, prefix, a.shape[-1]))


if __name__ == "__main__":
    import oracle_lib
    import ref_lib
    from robotoc_b200.layout import ULayout
    lib = oracle_lib.load()
    UL = ULayout(NV, getter=lib.orc_ulayout_get)
    data = {}
    for n, name in enumerate(CASES):
        tab, S, N, dt, lin, con, sol, dx0 = problem(name, lib.orc_ustage_layout_get)
        out = ref_lib.unconstr_iteration(NV, UL, S, tab, N, dt, lin, con, sol, dx0)
        for m, k in enumerate(KEYS):
            if k == "steps":
                data[f"{name}_{k}"] = out[k]
            else:
                put(data, f"{name}_{k}", out[k], record_groups(out[k], k, S, UL), 4000 + 16 * n + m, frac=FRAC, k_min=3, k_z=1)
    np.savez_compressed(PATH, **data)
    print("wrote", PATH, os.path.getsize(PATH) // 1024, "KiB")

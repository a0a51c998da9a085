"""Generates tests/golden/golden_ref_stage_r2.npz: one FULL hot-path iteration computed by the reference's own code
(tests/ref_lib.reference_iteration: robotoc's src/dynamics, src/constraints, src/core and src/riccati compiled unmodified,
oracle/Makefile.ref) on the small event schedule with switching-time optimisation (Intermediate, Lift, switching-constraint and
Impact stages), batch 1; a fixed, seeded sample of every section of every record (golden_sample.py), the performance
index whole.  Only runs where a robotoc source tree exists:
    ROBOTOC_REFERENCE=<robotoc source tree> python tests/golden/make_golden_ref_stage.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)

from helpers import small_event_schedule  # noqa: E402
from robotoc_b200 import ANYMAL  # noqa: E402
from robotoc_b200.stage import StageDims, anymal_constraint_table  # noqa: E402
from synth import make_stage_inputs  # noqa: E402
from golden_sample import groups, layout_bounds, put  # noqa: E402

PATH = os.path.join(HERE, "golden_ref_stage_r2.npz")
FRAC = 0.3  # share of the nonzero entries of every record section that is stored

SEED, BATCH = 301, 1
KEYS = ("kkt", "cc_cond", "ric", "d", "cc_exp", "xd_exp", "steps", "d_upd", "xd_upd", "cc_upd", "ex_upd", "perf_stage")


def stage_groups(a, key, S, K):
    """Per-section groups of a stage-layer record of reference_iteration (sections of the layout the record follows)."""
    prefix = {"kkt": "k_", "ric": "r_", "d": "d_", "d_upd": "d_", "cc_cond": "c_", "cc_exp": "c_", "cc_upd": "c_",
              "xd_exp": "x_", "xd_upd": "x_", "ex_upd": "e_"}.get(key)
    if prefix is None:
        return groups(a)
    lay = K if prefix in ("k_", "r_", "d_") else S
    return groups(a, layout_bounds(lay, prefix, a.shape[-1]))


def problem(S_getter=None, K_getter=None, impact_cones=False):
    """impact_cones: the same problem with ImpactFrictionCone registered (examples/anymal/run.cpp:173-181): the impact stage
    carries friction-cone rows on the impact forces (golden keys prefixed "ic_")."""
    from robotoc_b200 import Layout, StageLayout
    table = anymal_constraint_table(impact_friction_cone=impact_cones)
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=table.n_contacts, n_box=table.n_box)
    S, K = StageLayout(sd, getter=S_getter), Layout(ANYMAL, getter=K_getter)
    td, ev, ctrl = small_event_schedule(True)
    lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, BATCH, SEED, impact_cones=impact_cones)
    return table, sd, S, K, ctrl, lin, con, sol, dx0


if __name__ == "__main__":
    import oracle_lib
    import ref_lib
    lib = oracle_lib.load()
    table, sd, S, K, ctrl, lin, con, sol, dx0 = problem(lib.orc_stage_layout_get, lib.orc_layout_get)
    data = {}
    for pre, icone in (("", False), ("ic_", True)):
        table, sd, S, K, ctrl, lin, con, sol, dx0 = problem(lib.orc_stage_layout_get, lib.orc_layout_get, impact_cones=icone)
        out = ref_lib.reference_iteration(sd, S, K, table, ctrl, lin, con, dx0)
        for n, k in enumerate(KEYS):
            if k in ("steps", "perf_stage"):
                data[pre + k] = out[k]
            else:
                put(data, pre + k, out[k], stage_groups(out[k], k, S, K), SEED + n, frac=FRAC, k_min=3, k_z=1)
    np.savez_compressed(PATH, **data)
    print("wrote", PATH, os.path.getsize(PATH) // 1024, "KiB")

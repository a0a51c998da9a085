"""Generates tests/golden/golden_ref_live.npz, golden_ref_gaits.npz and golden_ref_horizon.npz: the reference's own outputs
(oracle/_ref/libref_riccati.so, the robotoc sources compiled unmodified by oracle/Makefile.ref) for the cases on which tests/ compare the oracle with the reference code, so that
those comparisons run everywhere without a robotoc checkout.  Only runs where one exists:

    ROBOTOC_REFERENCE=<robotoc source tree> python tests/golden/make_golden_ref_live.py [live] [gaits] [horizon]

golden_ref_gaits.npz holds the cases on the crawl and contact-mask-walk schedules (odd contact counts, single-foot impacts,
every contact mask); golden_ref_horizon.npz the receding-horizon edge schedules (helpers.receding_horizon_schedules: t0 != 0,
events on grid 1 and beside it, at the end of the horizon, tiny steps), sampled on the grid points next to t0, the events and
the terminal; golden_ref_live.npz everything else.  Without arguments all three files are written.

Large records are stored as a fixed, seeded sample of every section of every record (golden_sample.py); small outputs are
stored whole.
"""
import ctypes
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)

from golden_sample import groups, layout_bounds, load, put, restore  # noqa: E402,F401  (load, restore: used by the tests)
from helpers import (RH_SETS, contact_mask_walk_schedule, crawl_schedule, jump_sto_schedule, receding_horizon_schedules,  # noqa: E402
                     small_event_schedule, trot_schedule)

PATH = os.path.join(HERE, "golden_ref_live.npz")
GAITS_PATH = os.path.join(HERE, "golden_ref_gaits.npz")
HORIZON_PATH = os.path.join(HERE, "golden_ref_horizon.npz")
RIC_FIELDS = "r_P r_s r_K r_k r_M r_m r_Psi r_Phi r_T r_W r_psix r_psiu r_phix r_phiu r_mt r_mtn r_sc r_dtsdx r_stosc".split()
STAGE_KEYS = ("kkt", "cc_cond", "ric", "d", "cc_exp", "xd_exp", "steps", "d_upd", "xd_upd", "cc_upd", "ex_upd")


# ---- the cases (inputs are regenerated from these seeds by the tests)
RICCATI_CASES = [("small", 31), ("small_sto", 32), ("trot_n40", 33), ("jump_sto_n80", 34), ("crawl", 35), ("crawl_sto", 36)]
UNCONSTR_CASES = [(20, 0.05, 41), (50, 0.02, 42)]
STAGE_CASES = [("small", 311), ("small_sto", 312), ("trot", 313), ("small_icone", 314), ("small_sto_icone", 315), ("crawl", 317),
               ("crawl_sto", 318), ("crawl_icone", 319), ("mask_walk", 320)]
GAIT_CASES = ("crawl", "crawl_sto", "crawl_icone", "mask_walk")
JOINT_LIMIT_CASES = ["small_sto", "trot"]


JL_SCHEDULES = {"small_sto": lambda: small_event_schedule(True), "trot": lambda: trot_schedule(40)}
SCHEDULES = {"small": lambda: small_event_schedule(False), "small_sto": lambda: small_event_schedule(True),
             "trot": lambda: trot_schedule(40), "trot_n40": lambda: trot_schedule(40), "jump_sto_n80": lambda: jump_sto_schedule(80),
             "crawl": lambda: crawl_schedule(54), "crawl_sto": lambda: crawl_schedule(54, sto=True),
             "mask_walk": contact_mask_walk_schedule}


def schedule(case):
    """(TimeDiscretization, ContactEvents, control table) of a case; `<schedule>_icone` is `<schedule>` with impact cones."""
    return SCHEDULES[case[:-len("_icone")] if case.endswith("_icone") else case]()


def fixture_path(case):
    """The fixture file that holds the reference's outputs of a case."""
    return GAITS_PATH if case in GAIT_CASES else PATH


# receding-horizon edge cases: the edge schedules of the first two events of each gait cycle (a lift and an impact; every
# placement of _edge_offsets), ImpactFrictionCone on every other one
HORIZON_EVENTS = 2


def horizon_cases():
    """[(name, gait, sto, t0, ctrl, impact_cones, seed)] of golden_ref_horizon.npz."""
    out = []
    for g, sto in RH_SETS:
        sched = receding_horizon_schedules(g, sto, "edge")
        per_event = len(sched) // (4 if g == "trot" else 6)
        for k, (t0, td, ev, ctrl) in enumerate(sched[:HORIZON_EVENTS * per_event]):
            out.append((f"{g}{'_sto' if sto else ''}_{k}", g, sto, t0, td, ctrl, k % 2 == 1, 500 + len(out)))
    return out


def horizon_case(case, S_getter=None, K_getter=None):
    """Inputs of one horizon case (batch 1)."""
    from robotoc_b200 import ANYMAL, Layout, StageDims, StageLayout, anymal_constraint_table
    from synth import make_stage_inputs
    name, g, sto, t0, td, ctrl, icone, seed = case
    table = anymal_constraint_table(impact_friction_cone=icone)
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=table.n_contacts, n_box=table.n_box)
    S, K = StageLayout(sd, getter=S_getter), Layout(ANYMAL, getter=K_getter)
    lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, 1, seed, impact_cones=icone)
    return table, sd, S, K, ctrl, lin, con, sol, dx0, icone


def horizon_grids(ctrl):
    """The grid points a horizon case stores: the first three, the last four, and each event's grid with its neighbours."""
    n = len(ctrl)
    keep = {0, 1, 2, n - 4, n - 3, n - 2, n - 1}
    for i, c in enumerate(ctrl):
        if c.type in (1, 2):
            keep |= {i - 2, i - 1, i, i + 1}
    return sorted(i for i in keep if 0 <= i < n)


def joint_limit_problem(sched, batch, seed):
    """Inputs of the joint-limit linearisation: a stage problem and joint limits of the order of ANYmal's URDF."""
    import ctypes as ct
    import oracle_lib
    from robotoc_b200 import ANYMAL, StageDims, StageLayout, anymal_constraint_table
    from synth import make_stage_inputs
    lib = oracle_lib.load()
    table = anymal_constraint_table()
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=table.n_contacts, n_box=table.n_box)
    S = StageLayout(sd, getter=lib.orc_stage_layout_get)
    td, ev, ctrl = sched
    lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, batch, seed)
    rng = np.random.default_rng(seed + 3)
    lim = {0: 1.2, 1: 8.0, 3: 40.0}  # |q|, |v|, |u| limits
    bound = np.array([table.box[r].sign * lim[table.box[r].var] * rng.uniform(0.8, 1.2) for r in range(table.n_box)])
    for k in (2, 4):  # the reference's velocity / torque limits are symmetric (joint_velocity_lower_limit.cpp: vmin = -vmax)
        bound[k * 12:(k + 1) * 12] = -bound[(k + 1) * 12:(k + 2) * 12]
    lib.orc_linearize_joint_limits_batch.argtypes = [ct.c_void_p] * 3 + [ct.c_int, ct.c_int] + [ct.c_void_p] * 4
    return lib, table, sd, S, ctrl, lin, con, sol, bound


def stage_case(which, seed, S_getter, K_getter):
    from robotoc_b200 import ANYMAL, Layout, StageDims, StageLayout, anymal_constraint_table
    from synth import make_stage_inputs
    icone = which.endswith("_icone")
    table = anymal_constraint_table(impact_friction_cone=icone)
    sd = StageDims(ANYMAL, nf_max=12, n_contacts=table.n_contacts, n_box=table.n_box)
    S, K = StageLayout(sd, getter=S_getter), Layout(ANYMAL, getter=K_getter)
    td, ev, ctrl = schedule(which)
    lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, 1, seed, impact_cones=icone)
    return table, sd, S, K, ctrl, lin, con, sol, dx0, icone


def perf_case(sd, S, impact_cones):
    """The trot problem of the PerformanceIndex comparison (switching-constraint residuals made nonzero)."""
    from robotoc_b200 import anymal_constraint_table
    from synth import make_stage_inputs
    table = anymal_constraint_table(impact_friction_cone=impact_cones)
    td, ev, ctrl = trot_schedule(40)
    lin, con, sol, dx0 = make_stage_inputs(sd, S, ctrl, 1, 316, impact_cones=impact_cones)
    rng = np.random.default_rng(5)
    for i, c in enumerate(ctrl):
        if c.ns > 0:
            lin[:, i, S.l_p:S.l_p + c.ns] = rng.uniform(-1, 1, size=(1, c.ns))
    return table, ctrl, lin, con, dx0


def filter_rounds(case_rng):
    """Inputs of one sequence of line searches of the filter comparison."""
    rounds, n_trials = 40, 8
    amax = case_rng.uniform(0.05, 1.0, size=rounds)
    trend = np.linspace(10.0, 1.0, rounds)[:, None]  # costs drift down like a converging solver; violations shrink
    cost = trend + case_rng.normal(0, 0.5, size=(rounds, n_trials))
    viol = np.abs(trend * 0.1 + case_rng.normal(0, 0.05, size=(rounds, n_trials)))
    return amax, cost, viol, cost[:, 0] + 0.1, viol[:, 0] + 0.01


def main(outputs=("live", "gaits", "horizon")):
    import oracle_lib
    import ref_lib
    import make_golden_ref_stage as mgs
    from robotoc_b200 import ANYMAL, Layout, ULayout
    from synth import make_kkt, make_unconstr_kkt
    assert ref_lib.available(), "set ROBOTOC_REFERENCE to a robotoc source tree"
    lib = oracle_lib.load()
    P = oracle_lib.ptr
    files = {PATH: {}, GAITS_PATH: {}}
    out = files[PATH]
    L = Layout(ANYMAL, getter=lib.orc_layout_get)
    for name, seed in RICCATI_CASES:
        td, ev, ctrl = schedule(name)
        kkt, dx0 = make_kkt(ANYMAL, L, ctrl, batch=3, seed=seed)
        kk, ric, d = ref_lib.riccati_batch(ANYMAL, L, ctrl, kkt, dx0)
        out = files[fixture_path(name)]
        put(out, f"ric_{name}_ric", ric, groups(ric, layout_bounds(L, "r_", L.r_stride)), seed, k_min=3, k_z=1)
        put(out, f"ric_{name}_dir", d, groups(d, layout_bounds(L, "d_", L.d_stride)), seed + 1, k_min=3, k_z=1)
        put(out, f"ric_{name}_kkt", kk, groups(kk, layout_bounds(L, "k_", L.k_stride)), seed + 2, k_min=3, k_z=1)
    out = files[PATH]
    UL = ULayout(7, getter=lib.orc_ulayout_get)
    for N, dt, seed in UNCONSTR_CASES:
        kkt, dx0 = make_unconstr_kkt(7, UL, N, 3, seed)
        kk, ric, d = ref_lib.unconstr_batch(7, UL, N, dt, kkt, dx0)
        put(out, f"unconstr_{N}_ric", ric, groups(ric, layout_bounds(UL, "r_", UL.r_stride)), seed, k_min=3, k_z=1)
        put(out, f"unconstr_{N}_dir", d, groups(d, layout_bounds(UL, "d_", UL.d_stride)), seed + 1, k_min=3, k_z=1)
        put(out, f"unconstr_{N}_kkt", kk, groups(kk, layout_bounds(UL, "k_", UL.k_stride)), seed + 2, k_min=3, k_z=1)
    for case, seed in STAGE_CASES:
        table, sd, S, K, ctrl, lin, con, sol, dx0, icone = stage_case(case, seed, lib.orc_stage_layout_get, lib.orc_layout_get)
        ref = ref_lib.reference_iteration(sd, S, K, table, ctrl, lin, con, dx0)
        for k in STAGE_KEYS:
            put(files[fixture_path(case)], f"stage_{case}_{k}", ref[k], mgs.stage_groups(ref[k], k, S, K), seed, k_min=3, k_z=1)
    files[HORIZON_PATH] = {}
    for case in horizon_cases():
        table, sd, S, K, ctrl, lin, con, sol, dx0, icone = horizon_case(case, lib.orc_stage_layout_get, lib.orc_layout_get)
        ref = ref_lib.reference_iteration(sd, S, K, table, ctrl, lin, con, dx0)
        keep = np.zeros(len(ctrl), dtype=bool)
        keep[horizon_grids(ctrl)] = True
        for k in STAGE_KEYS:
            a = ref[k]
            grp = mgs.stage_groups(a, k, S, K)
            n_grp = int(grp.max()) + 1
            if a.ndim == 3:  # records of the kept grid points only: one nonzero entry of every section
                gids, first = np.unique(grp.reshape(-1), return_index=True)
                on = [False] * n_grp
                for gid, pos in zip(gids, first):
                    on[gid] = bool(keep[(pos // a.shape[-1]) % len(ctrl)])
                put(files[HORIZON_PATH], f"h_{case[0]}_{k}", a, grp, case[7], k_min=tuple(1 if o else 0 for o in on),
                    k_z=tuple(0 for o in on))
            else:
                files[HORIZON_PATH][f"h_{case[0]}_{k}"] = a
    for icone in (False, True):
        table, sd, S, K, ctrl, lin, con, sol, dx0 = mgs.problem(lib.orc_stage_layout_get, lib.orc_layout_get, icone)
        table, ctrl, lin, con, dx0 = perf_case(sd, S, icone)
        out[f"perf_icone{int(icone)}"] = ref_lib.reference_iteration(sd, S, K, table, ctrl, lin, con, dx0)["perf_stage"]
    ref = ref_lib.load()
    ref.ref_filter_line_search.argtypes = [ctypes.c_int, ctypes.c_int] + [ctypes.c_double] * 4 + [ctypes.c_void_p] * 7
    rng = np.random.default_rng(3)
    steps, ks = [], []
    for case in range(20):
        amax, cost, viol, cost0, viol0 = filter_rounds(rng)
        step_r, k_r = np.zeros(len(amax)), np.zeros(len(amax), dtype=np.int32)
        ref.ref_filter_line_search(len(amax), cost.shape[1], 0.75, 0.05, 0.005, 0.005, P(amax), P(cost0), P(viol0),
                                   P(np.ascontiguousarray(cost)), P(np.ascontiguousarray(viol)), P(step_r),
                                   k_r.ctypes.data_as(ctypes.c_void_p))
        steps.append(step_r)
        ks.append(k_r)
    out["filter_step"], out["filter_k"] = np.array(steps), np.array(ks)
    ref.ref_linearize_joint_limits.argtypes = [ctypes.c_void_p] * 7
    for which in JOINT_LIMIT_CASES:
        lib_, table, sd, S, ctrl, lin, con, sol, bound = joint_limit_problem(JL_SCHEDULES[which](), 2, 81)
        l_r, c_r = lin.copy(), con.copy()
        csd = sd.c()
        for b in range(lin.shape[0]):
            for i, ct in enumerate(ctrl):
                lr, cr = np.ascontiguousarray(lin[b, i]), np.ascontiguousarray(con[b, i])
                assert ref.ref_linearize_joint_limits(ctypes.byref(csd), ctypes.byref(table), ctypes.byref(ct), P(bound),
                                                      P(np.ascontiguousarray(sol[b, i])), P(lr), P(cr)) == 0
                l_r[b, i], c_r[b, i] = lr, cr
        # every entry the linearisation changes (group 0), plus a sample of the others (group 1)
        put(out, f"jl_{which}_lin", l_r, np.where(l_r != lin, 0, 1), 7, frac=(1.0, 0.0), k_min=(0, 256), k_z=(l_r.size, 32))
        put(out, f"jl_{which}_con", c_r, np.where(c_r != con, 0, 1), 8, frac=(1.0, 0.0), k_min=(0, 256), k_z=(c_r.size, 32))
    for path, data in files.items():
        if {PATH: "live", GAITS_PATH: "gaits", HORIZON_PATH: "horizon"}[path] in outputs:
            np.savez_compressed(path, **data)
            print("wrote", path, os.path.getsize(path) // 1024, "KiB;", ref.ref_version().decode())


if __name__ == "__main__":
    main(sys.argv[1:] or ("live", "gaits", "horizon"))

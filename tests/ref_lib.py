"""ctypes wrapper around oracle/_ref/libref_riccati.so -- the REFERENCE's own Riccati sources (robotoc's src/riccati,
src/core), compiled unmodified against the Eigen / Robot stand-ins of oracle/shim (oracle/Makefile.ref).  TEST
INFRASTRUCTURE: the generators under tests/golden/ use it to store what the reference computes.  The library can only be
built where a robotoc source tree is available: set ROBOTOC_REFERENCE to it."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
LIB = os.path.join(ORACLE_DIR, "_ref", "libref_riccati.so")
REFERENCE = os.environ.get("ROBOTOC_REFERENCE", "")

_lib = None


def available():
    return os.path.exists(LIB) or (bool(REFERENCE) and os.path.isdir(os.path.join(REFERENCE, "src", "riccati")))


def build():
    if REFERENCE and os.path.isdir(os.path.join(REFERENCE, "src", "riccati")):
        subprocess.run(["make", "-s", "-C", ORACLE_DIR, "-f", "Makefile.ref", f"REF={REFERENCE}"], check=True)


def load():
    global _lib
    if _lib is not None:
        return _lib
    build()
    from robotoc_b200._lib import rbt_dims, rbt_stage_ctrl
    L = ctypes.CDLL(LIB)
    c_int, c_dbl, c_vp = ctypes.c_int, ctypes.c_double, ctypes.c_void_p
    L.ref_riccati_batch.argtypes = [ctypes.POINTER(rbt_dims), ctypes.POINTER(rbt_stage_ctrl), c_int, c_dbl, c_int, c_vp, c_vp,
                                    c_vp, c_vp]
    L.ref_unconstr_batch.argtypes = [c_int, c_int, c_dbl, c_int, c_vp, c_vp, c_vp, c_vp]
    L.ref_version.restype = ctypes.c_char_p
    _lib = L
    return L


def _ptr(a):
    assert a.dtype == np.float64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(ctypes.c_void_p)


def riccati_batch(dims, L, ctrl, kkt, dx0, max_dts0=0.1):
    """robotoc::RiccatiRecursion (reference code) over a batch, one OCP after the other.
    Returns (kkt mutated like the reference mutates it, ric, dir)."""
    lib = load()
    batch, n_grid = kkt.shape[0], kkt.shape[1]
    kk = kkt.copy()
    ric = np.zeros((batch, n_grid, L.r_stride))
    d = np.zeros((batch, n_grid, L.d_stride))
    cd = dims.c()
    rc = lib.ref_riccati_batch(ctypes.byref(cd), ctrl, n_grid, max_dts0, batch, _ptr(kk), _ptr(ric), _ptr(dx0), _ptr(d))
    assert rc == 0
    return kk, ric, d


def unconstr_batch(nv, UL, N, dt, kkt, dx0):
    lib = load()
    batch = kkt.shape[0]
    kk = kkt.copy()
    ric = np.zeros((batch, N + 1, UL.r_stride))
    d = np.zeros((batch, N + 1, UL.d_stride))
    rc = lib.ref_unconstr_batch(nv, N, dt, batch, _ptr(kk), _ptr(ric), _ptr(dx0), _ptr(d))
    assert rc == 0
    return kk, ric, d


def stage(sd, table, c, lin, con, d, d_next, alpha_p, alpha_d, phase=3):
    """One OCP stage through the reference's stage-layer code (oracle/ref_wrap/ref_stage_wrap.cpp).  Returns a dict with the
    KKT record, the expansion record, the PDIPM record (cmpl, cond, dslack, ddual, updated slack | dual), the updated direction
    record (costate correction), the expanded direction record and this stage's max step sizes."""
    from robotoc_b200 import ANYMAL, Layout, StageLayout
    import oracle_lib
    lib = load()
    olib = oracle_lib.load()
    S = StageLayout(sd, getter=olib.orc_stage_layout_get)
    K = Layout(ANYMAL, getter=olib.orc_layout_get)
    if not hasattr(lib, "_stage_ready"):
        lib.ref_stage.argtypes = [ctypes.c_void_p] * 11 + [ctypes.c_double, ctypes.c_double, ctypes.c_int]
        lib._stage_ready = True
    kkt, ex, xd = np.zeros(K.k_stride), np.zeros(S.e_stride), np.zeros(S.x_stride)
    cc, dd = con.copy(), d.copy()
    dn = d_next.copy() if d_next is not None else np.zeros(K.d_stride)
    steps = np.ones(2)
    csd = sd.c()
    rc = lib.ref_stage(ctypes.byref(csd), ctypes.byref(table), ctypes.byref(c), _ptr(np.ascontiguousarray(lin)), _ptr(cc), _ptr(kkt),
                       _ptr(ex), _ptr(dd), _ptr(dn), _ptr(xd), _ptr(steps), alpha_p, alpha_d, phase)
    assert rc == 0
    perf = np.zeros(4)  # {cost_barrier, primal_feasibility, dual_feasibility, kkt_error} as the stage's evalKKT summarises them
    lib.ref_last_perf.argtypes = [ctypes.c_void_p]
    lib.ref_last_perf(_ptr(perf))
    return dict(kkt=kkt, ex=ex, con=cc, d=dd, xd=xd, steps=steps, perf=perf)


def reference_iteration(sd, S, K, table, ctrl, lin, con, dx0):
    """One full hot-path iteration computed by the REFERENCE's own code: stage-layer condensing (ref_stage phase 1) ->
    robotoc::RiccatiRecursion backward + forward (ref_riccati_batch) -> primal expansion and step sizes (phase 2) -> horizon
    minimum -> dual expansion, costate correction and slack / dual update (phase 3).  The solution update itself
    (SplitSolution::integrate -> Pinocchio's SE(3) integrate) is not part of it.  Same record dictionary as
    iteration_check.oracle_iteration (minus `sol`)."""
    from robotoc_b200 import ANYMAL
    from robotoc_b200.grid import TERMINAL
    batch, n_grid = lin.shape[0], lin.shape[1]
    kkt = np.zeros((batch, n_grid, K.k_stride))
    ex = np.zeros((batch, n_grid, S.e_stride))
    cc_cond = con.copy()
    perf_stage = np.zeros((batch, n_grid, 4))
    zero_d = np.zeros(K.d_stride)
    for b in range(batch):
        for i, c in enumerate(ctrl):
            o = stage(sd, table, c, lin[b, i], con[b, i], zero_d, zero_d, 1.0, 1.0, phase=1)
            kkt[b, i], ex[b, i], cc_cond[b, i] = o["kkt"], o["ex"], o["con"]
            perf_stage[b, i] = o["perf"]
    kk, ric, d = riccati_batch(ANYMAL, K, ctrl, kkt, dx0)
    steps = np.ones((batch, 2))
    cc_exp, xd_exp = con.copy(), np.zeros((batch, n_grid, S.x_stride))
    for b in range(batch):
        for i, c in enumerate(ctrl):
            if c.type == TERMINAL:
                continue
            o = stage(sd, table, c, lin[b, i], con[b, i], d[b, i], d[b, i + 1], 1.0, 1.0, phase=2)
            steps[b] = np.minimum(steps[b], o["steps"])
            cc_exp[b, i], xd_exp[b, i] = o["con"], o["xd"]
    d_upd, xd_upd, cc_upd, ex_upd = d.copy(), xd_exp.copy(), con.copy(), ex.copy()
    for b in range(batch):
        for i, c in enumerate(ctrl):
            dn = d[b, i + 1] if i + 1 < n_grid else None
            o = stage(sd, table, c, lin[b, i], con[b, i], d[b, i], dn, steps[b, 0], steps[b, 1], phase=3)
            d_upd[b, i], xd_upd[b, i], cc_upd[b, i], ex_upd[b, i] = o["d"], o["xd"], o["con"], o["ex"]
    return dict(kkt=kkt, cc_cond=cc_cond, ric=ric, d=d, cc_exp=cc_exp, xd_exp=xd_exp, steps=steps, d_upd=d_upd, xd_upd=xd_upd,
                cc_upd=cc_upd, ex_upd=ex_upd, perf_stage=perf_stage)


def unconstr_iteration(nv, UL, S, tab, N, dt, lin, con, sol, dx0):
    """One hot-path iteration of the unconstrained (fixed-base) path computed by the REFERENCE's own code: stage-layer
    condensing on every grid point (ref_ustage phase 1, oracle/ref_wrap/ref_ustage_wrap.cpp) -> robotoc::UnconstrRiccatiRecursion
    (ref_unconstr_batch) -> expansion and step sizes (phase 2) -> horizon minimum -> solution, slack and dual update (phase 3).
    Same record dictionary as oracle_lib.unconstr_iteration (minus `ric`, `info`)."""
    lib = load()
    if not hasattr(lib, "_ustage_ready"):
        c_int, c_dbl, c_vp = ctypes.c_int, ctypes.c_double, ctypes.c_void_p
        lib.ref_ustage.argtypes = [c_int, c_vp, c_int, c_int, c_dbl] + [c_vp] * 8 + [c_dbl, c_dbl, c_int]
        lib._ustage_ready = True
    batch = lin.shape[0]
    kkt = np.zeros((batch, N + 1, UL.k_stride))
    ex = np.zeros((batch, N + 1, S.e_stride))
    con_c, con_e, con_u = con.copy(), con.copy(), con.copy()
    xd = np.zeros((batch, N + 1, S.x_stride))
    sol_u = sol.copy()
    steps = np.ones((batch, 2))
    zero_d = np.zeros(UL.d_stride)

    def run(b, i, d, phase, alpha, c_out, kkt_out, ex_out, xd_out, sol_out):
        c = con[b, i].copy()
        k, e, x, s = np.zeros(UL.k_stride), np.zeros(S.e_stride), np.zeros(S.x_stride), sol[b, i].copy()
        st = np.ones(2)
        rc = lib.ref_ustage(nv, ctypes.byref(tab), i, N, dt, _ptr(np.ascontiguousarray(lin[b, i])), _ptr(c), _ptr(k), _ptr(e),
                            _ptr(np.ascontiguousarray(d)), _ptr(x), _ptr(s), _ptr(st), alpha[0], alpha[1], phase)
        assert rc == 0, "the reference cannot express this constraint table"
        c_out[b, i] = c
        for out, v in ((kkt_out, k), (ex_out, e), (xd_out, x), (sol_out, s)):
            if out is not None:
                out[b, i] = v
        return st

    for b in range(batch):
        for i in range(N + 1):
            run(b, i, zero_d, 1, (1.0, 1.0), con_c, kkt, ex, None, None)
    _, _, d = unconstr_batch(nv, UL, N, dt, kkt, dx0)
    for b in range(batch):
        for i in range(N):
            steps[b] = np.minimum(steps[b], run(b, i, d[b, i], 2, (1.0, 1.0), con_e, None, None, xd, None))
    for b in range(batch):
        for i in range(N + 1):
            run(b, i, d[b, i], 3, steps[b], con_u, None, None, None, sol_u)
    return dict(kkt=kkt, ex=ex, con_condensed=con_c, dir=d, xd=xd, steps=steps, con_expanded=con_e, con=con_u, sol=sol_u)


LIB_DISCRETIZE = os.path.join(ORACLE_DIR, "_ref", "libref_discretize.so")
_lib_td = None


def discretize(T, N, ev, t0, phase_based=True):
    """robotoc::TimeDiscretization::discretize(t0) (+ correctTimeSteps(t0) if `phase_based`) of the reference, on the
    ContactSequence that `ev` (schedule_fixture.ContactEvents) describes (oracle/ref_wrap/ref_discretize_wrap.cpp).  Returns
    one dict of GridInfo fields per grid point."""
    global _lib_td
    if _lib_td is None:
        build()
        L = ctypes.CDLL(LIB_DISCRETIZE)
        c_int, c_dbl, c_vp = ctypes.c_int, ctypes.c_double, ctypes.c_void_p
        L.ref_discretize.argtypes = [c_dbl, c_int, c_int, c_vp, c_vp, c_vp, c_dbl, c_int, c_int, c_vp, c_vp]
        _lib_td = L
    events = sorted([(t, s) for t, s in zip(ev.impact_times, ev.sto_impact)] + [(t, s) for t, s in zip(ev.lift_times, ev.sto_lift)])
    masks = np.array(ev.phase_mask, dtype=np.int32)
    times = np.array([t for t, _ in events], dtype=np.float64)
    sto = np.array([int(s) for _, s in events], dtype=np.int32)
    n_max = N + 1 + 3 * len(events) + 1
    ints, dbls = np.zeros((n_max, 10), dtype=np.int32), np.zeros((n_max, 4))
    n = _lib_td.ref_discretize(T, N, len(events), masks.ctypes.data, times.ctypes.data, sto.ctypes.data, t0, int(phase_based),
                               n_max, ints.ctypes.data, dbls.ctypes.data)
    assert n > 0, f"ref_discretize failed ({n})"
    names_i = ("type", "phase", "stage", "impact_index", "lift_index", "stage_in_phase", "num_grids_in_phase", "sto", "sto_next",
               "switching_constraint")
    names_d = ("t0", "t", "dt", "dt_next")
    return [dict(**{k: int(v) for k, v in zip(names_i, ints[i])}, **{k: float(v) for k, v in zip(names_d, dbls[i])})
            for i in range(n)]

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

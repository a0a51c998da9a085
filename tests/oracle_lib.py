"""ctypes wrapper around oracle/liboracle.so -- the CPU restatement of the reference (TEST INFRASTRUCTURE)."""
import ctypes
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
LIB = os.path.join(ORACLE_DIR, "liboracle.so")

_lib = None


def build():
    subprocess.run(["make", "-s", "-C", ORACLE_DIR], check=True)


def load():
    global _lib
    if _lib is not None:
        return _lib
    build()  # make is a no-op when up to date; a stale oracle after a header change would mis-read the control table
    from robotoc_b200._lib import rbt_dims, rbt_stage_ctrl
    L = ctypes.CDLL(LIB)
    c_int, c_dbl, c_vp = ctypes.c_int, ctypes.c_double, ctypes.c_void_p
    pdims, pctrl = ctypes.POINTER(rbt_dims), ctypes.POINTER(rbt_stage_ctrl)
    L.orc_layout_get.argtypes = [pdims, ctypes.c_char_p]
    L.orc_ulayout_get.argtypes = [c_int, ctypes.c_char_p]
    L.orc_riccati_backward.argtypes = [pdims, pctrl, c_int, c_dbl, c_vp, c_vp]
    L.orc_riccati_forward.argtypes = [pdims, pctrl, c_int, c_vp, c_vp, c_vp]
    L.orc_riccati_batch.argtypes = [pdims, pctrl, c_int, c_dbl, c_int, c_vp, c_vp, c_vp, c_vp, c_int]
    L.orc_unconstr_backward.argtypes = [c_int, c_int, c_dbl, c_vp, c_vp]
    L.orc_unconstr_forward.argtypes = [c_int, c_int, c_dbl, c_vp, c_vp, c_vp]
    L.orc_unconstr_batch.argtypes = [c_int, c_int, c_dbl, c_int, c_vp, c_vp, c_vp, c_vp, c_int]
    L.orc_backward_full_step.argtypes = [pdims, c_int, c_int, c_int, c_vp, c_vp, c_vp]
    L.orc_backward_impact_step.argtypes = [pdims, c_int, c_vp, c_vp, c_vp]
    L.orc_backward_impact_step.restype = None
    L.orc_phase_transition_step.argtypes = [pdims, c_dbl, c_vp, c_vp, c_vp, c_int]
    L.orc_phase_transition_step.restype = None
    L.orc_max_threads.restype = c_int
    from robotoc_b200.stage import rbt_stage_dims, rbt_constraint_table
    psd, ptab = ctypes.POINTER(rbt_stage_dims), ctypes.POINTER(rbt_constraint_table)
    L.orc_stage_layout_get.argtypes = [psd, ctypes.c_char_p]
    L.orc_mjtjinv.argtypes = [c_int, c_int, c_vp, c_vp, c_int, c_vp, c_int]
    L.orc_condense_batch.argtypes = [psd, ptab, pctrl, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_int]
    L.orc_expand_batch.argtypes = [psd, ptab, pctrl, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int]
    L.orc_expand_batch.restype = None
    L.orc_update_batch.argtypes = [psd, ptab, pctrl, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_int]
    L.orc_update_batch.restype = None
    L.orc_ustage_layout_get.argtypes = [c_int, c_int, ctypes.c_char_p]
    L.orc_ustage_condense.argtypes = [c_int, ptab, c_int, c_vp, c_vp, c_vp, c_vp]
    L.orc_ustage_condense.restype = None
    L.orc_ustage_expand.argtypes = [c_int, ptab, c_dbl, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.orc_ustage_expand.restype = None
    L.orc_ustage_update.argtypes = [c_int, ptab, c_int, c_vp, c_vp, c_vp, c_vp, c_dbl, c_dbl]
    L.orc_ustage_update.restype = None
    L.orc_ustage_condense_at.argtypes = [c_int, ptab, c_int, c_int, c_vp, c_vp, c_vp, c_vp]
    L.orc_ustage_condense_at.restype = None
    L.orc_ucondense_batch.argtypes = [c_int, ptab, c_int, c_int, c_vp, c_vp, c_vp, c_vp]
    L.orc_ucondense_batch.restype = None
    L.orc_uexpand_batch.argtypes = [c_int, ptab, c_int, c_dbl, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.orc_uexpand_batch.restype = None
    L.orc_uupdate_batch.argtypes = [c_int, ptab, c_int, c_int, c_vp, c_vp, c_vp, c_vp, c_vp]
    L.orc_uupdate_batch.restype = None
    _lib = L
    return L


def ptr(a):
    assert a.dtype == np.float64 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(ctypes.c_void_p)


def riccati_batch(dims, L, ctrl, kkt, dx0, max_dts0=0.1, nthreads=0, forward=True):
    """Runs the oracle over a batch.  Returns (kkt_mutated, ric, dir, info); kkt is copied first."""
    lib = load()
    batch, n_grid = kkt.shape[0], kkt.shape[1]
    kk = kkt.copy()
    ric = np.zeros((batch, n_grid, L.r_stride))
    d = np.zeros((batch, n_grid, L.d_stride)) if forward else None
    cd = dims.c()
    info = lib.orc_riccati_batch(ctypes.byref(cd), ctrl, n_grid, max_dts0, batch, ptr(kk), ptr(ric),
                                 ptr(dx0) if forward else None, ptr(d) if forward else None, nthreads)
    return kk, ric, d, info


def unconstr_batch(nv, UL, N, dt, kkt, dx0, nthreads=0, forward=True):
    lib = load()
    batch = kkt.shape[0]
    kk = kkt.copy()
    ric = np.zeros((batch, N + 1, UL.r_stride))
    d = np.zeros((batch, N + 1, UL.d_stride)) if forward else None
    info = lib.orc_unconstr_batch(nv, N, dt, batch, ptr(kk), ptr(ric), ptr(dx0) if forward else None,
                                  ptr(d) if forward else None, nthreads)
    return kk, ric, d, info


def unconstr_iteration(nv, UL, S, tab, N, dt, lin, con, sol, dx0):
    """One hot-path iteration of the unconstrained solver on the oracle (UnconstrOCPSolver::updateSolution's linear-algebra
    body, unconstr_ocp_solver.cpp:101-118).  Returns a dict of every intermediate record."""
    lib = load()
    batch = lin.shape[0]
    con = con.copy()
    sol = sol.copy()
    kkt = np.zeros((batch, N + 1, UL.k_stride))
    ex = np.zeros((batch, N + 1, S.e_stride))
    lib.orc_ucondense_batch(nv, ctypes.byref(tab), N, batch, ptr(lin), ptr(con), ptr(kkt), ptr(ex))
    kkt_c = kkt.copy()
    con_c = con.copy()
    kk, ric, d, info = unconstr_batch(nv, UL, N, dt, kkt, dx0)
    xd = np.zeros((batch, N + 1, S.x_stride))
    steps = np.zeros((batch, 2))
    lib.orc_uexpand_batch(nv, ctypes.byref(tab), N, dt, batch, ptr(lin), ptr(ex), ptr(d), ptr(con), ptr(xd), ptr(steps))
    con_e = con.copy()
    lib.orc_uupdate_batch(nv, ctypes.byref(tab), N, batch, ptr(d), ptr(xd), ptr(con), ptr(sol), ptr(steps))
    return dict(kkt=kkt_c, ex=ex, con_condensed=con_c, ric=ric, dir=d, xd=xd, steps=steps, con_expanded=con_e, con=con,
                sol=sol, info=info)

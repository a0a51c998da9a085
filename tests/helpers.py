"""Shared test helpers: problems, record views, dense KKT reference solve."""
import numpy as np

from robotoc_b200 import ANYMAL, Layout
from robotoc_b200.grid import IMPACT, LIFT, TERMINAL
from schedule_fixture import (ContactEvents, TimeDiscretization, stage_ctrl_array, anymal_trot_events,
                              anymal_jump_sto_events, anymal_crawl_events, contact_mask_walk_events)
from synth import make_kkt, mat


def small_event_schedule(sto=False):
    """ANYmal, T=0.4, N=8: lift at 0.07, impact (dimf 6) at 0.23 -> Lift, Impact, one switching-constraint stage."""
    ev = ContactEvents(phase_dimf=[12], phase_mask=[0b1111])
    ev.push_back(False, 0.07, 6, sto=sto, post_mask=0b1001)
    ev.push_back(True, 0.23, 12, impact_dimf=6, sto=sto, post_mask=0b1111, impact_mask=0b0110)
    td = TimeDiscretization(0.4, 8).discretize(ev, 0.0, sto=sto)
    return td, ev, stage_ctrl_array(td, ev)


def trot_schedule(N=40):
    ev = anymal_trot_events()
    td = TimeDiscretization(1.12, N).discretize(ev, 0.0)
    return td, ev, stage_ctrl_array(td, ev)


def jump_sto_schedule(N=80):
    ev = anymal_jump_sto_events()
    td = TimeDiscretization(1.7, N).discretize(ev, 0.0, sto=True)
    return td, ev, stage_ctrl_array(td, ev)


def crawl_schedule(N=54, sto=False):
    """ANYmal crawl (anymal_crawl_events), T=2.16: three-foot stances, single-foot impacts (nf 3, ns 3) and two impacts at
    which another foot lifts; with `sto` every event's switching time is optimised."""
    ev = anymal_crawl_events(sto)
    td = TimeDiscretization(2.16, N).discretize(ev, 0.0, sto=sto)
    ctrl = stage_ctrl_array(td, ev)
    types = [c.type for c in ctrl]
    assert types.count(IMPACT) == 4 and types.count(LIFT) == 2 and types[-1] == TERMINAL
    assert {c.nf for c in ctrl[:-1]} == {3, 9, 12} and {c.ns for c in ctrl} == {0, 3}
    assert {c.contact_mask for c in ctrl if c.type == IMPACT} == {0b0001, 0b0010, 0b0100, 0b1000}
    assert sum(1 for i, c in enumerate(ctrl) if c.type == IMPACT and ctrl[i - 1].contact_mask & ~ctrl[i + 1].contact_mask) == 2
    assert all(c.sto for c in ctrl[:-1]) if sto else not any(c.sto or c.sto_next for c in ctrl)
    return td, ev, ctrl


# contact sets of contact_mask_walk_schedule's phases: all 16, impacts of 1 / 2 / 3 / 4 feet, impacts that also lift a foot
MASK_WALK = [0b1111, 0b1110, 0b1100, 0b1000, 0b0000, 0b0101, 0b0001, 0b1011, 0b0011, 0b0010, 0b0110, 0b0100, 0b1101, 0b1001,
             0b1010, 0b0111, 0b1111, 0b0000, 0b1111, 0b1000, 0b1111, 0b1110, 0b1111]


def contact_mask_walk_schedule(dt=0.02):
    """Synthetic schedule through every contact set of ANYmal's four feet (contact_mask_walk_events over MASK_WALK), three
    time steps per phase.  Asserts its own coverage: every mask on at least two Intermediate grid points, every single-foot
    impact, switching constraints of dimension 3, 6, 9 and 12, and impacts that also lift a foot."""
    ev = contact_mask_walk_events(MASK_WALK, dt)
    N = 3 * len(MASK_WALK) + 1
    td = TimeDiscretization(N * dt, N).discretize(ev, 0.0, sto=False)
    ctrl = stage_ctrl_array(td, ev)
    per_mask = np.bincount([c.contact_mask for c in ctrl if c.type == 0], minlength=16)
    assert per_mask.min() >= 2, per_mask
    impacts = [i for i, c in enumerate(ctrl) if c.type == IMPACT]
    assert {0b0001, 0b0010, 0b0100, 0b1000} <= {ctrl[i].contact_mask for i in impacts}
    assert {c.ns for c in ctrl} == {0, 3, 6, 9, 12}
    assert {c.nf for c in ctrl} == {0, 3, 6, 9, 12}
    assert sum(1 for i in impacts if ctrl[i - 1].contact_mask & ~ctrl[i + 1].contact_mask) >= 2  # land one foot, lift another
    return td, ev, ctrl


def _events_in_order(ev):
    """The events of `ev` in time order: (time, is_impact, post_dimf, impact_dimf, post_mask, impact_mask, sto)."""
    out = [(t, True, k, s) for k, (t, s) in enumerate(zip(ev.impact_times, ev.sto_impact))]
    out += [(t, False, k, s) for k, (t, s) in enumerate(zip(ev.lift_times, ev.sto_lift))]
    out.sort()
    return [(t, imp, ev.phase_dimf[p + 1], ev.impact_dimf[k] if imp else 0, ev.phase_mask[p + 1], ev.impact_mask[k] if imp else 0, s)
            for p, (t, imp, k, s) in enumerate(out)]


def _cycles(one, period, n, sto):
    """`n` copies of the one-cycle event list `one` (which ends in the contact set it starts from), copy k shifted by
    k * period; every event's STO flag set to `sto`."""
    ev = ContactEvents(phase_dimf=[one.phase_dimf[0]], phase_mask=[one.phase_mask[0]])
    for k in range(n):
        for t, imp, dimf, idimf, mask, imask, _ in _events_in_order(one):
            ev.push_back(imp, k * period + t, dimf, impact_dimf=idimf, sto=sto, post_mask=mask, impact_mask=imask)
    return ev


# receding-horizon gaits: (one-cycle events, cycle period, T, N); the trot of anymal_trot_events repeats every 1.08 s, the
# crawl of anymal_crawl_events every 2.08 s (the next cycle starts 0.04 s after the last impact, like the first one)
RH_GAITS = {"trot": (anymal_trot_events, 1.08, 1.12, 40), "crawl": (anymal_crawl_events, 2.08, 2.16, 54)}


def trot_cycles(n, sto=False):
    return _cycles(anymal_trot_events(), RH_GAITS["trot"][1], n, sto)


def crawl_cycles(n, sto=False):
    return _cycles(anymal_crawl_events(), RH_GAITS["crawl"][1], n, sto)


def _edge_offsets(dt, T):
    """Where edge_t0s puts an event relative to t0: a hair after t0 (tiny first step), exactly on grid 1, 1e-9 either side
    of it (inside the _EPS test of discretize), 2 * _EPS either side of it (outside that test), just inside and just outside
    the last-interval margin, and exactly at t0 (excluded: grid 0 starts in the event's post-phase)."""
    e = 2.0 * 1.4901161193847656e-08
    return (1e-6 * dt, dt, dt - 1e-9, dt + 1e-9, dt - e, dt + e, T - 0.5 * dt - 1e-9, T - 0.5 * dt + 1e-9, 0.0)


def receding_horizon_schedules(gait, sto, which, per_dt=4):
    """The schedules an MPC loop meets while the horizon slides over gait `gait` ("trot" | "crawl", every event STO-enabled
    iff `sto`), discretized like OCPSolver::discretize at each t0: `which` = "sweep" (t0 over one gait cycle in steps of
    dt / per_dt) or "edge" (t0 placed per event of the second cycle by _edge_offsets).  Returns [(t0, td, ev, ctrl)]."""
    one, period, T, N = RH_GAITS[gait]
    ev = _cycles(one(), period, 4, sto)
    dt = T / N
    if which == "sweep":
        t0s = [k * dt / per_dt for k in range(int(round(period / (dt / per_dt))))]
    else:
        cycle = [e[0] for e in _events_in_order(one())]
        t0s = [period + te - off for te in cycle for off in _edge_offsets(dt, T)]
    out = []
    for t0 in t0s:
        td = TimeDiscretization(T, N).discretize(ev, t0, sto=True)
        out.append((t0, td, ev, stage_ctrl_array(td, ev)))
    return out


RH_SETS = (("trot", False), ("trot", True), ("crawl", False))


def receding_horizon_coverage(schedules):
    """Asserts that `schedules` ([(t0, td, ev, ctrl)], e.g. the sweep and edge sets of RH_SETS together) reach the grid
    positions the kernels branch on: an impact on grid 1 (switching constraint on grid 0) with and without STO, an impact on
    n_grid - 3, a lift on n_grid - 2, a one-grid first phase with STO, a step below 1e-5 T / N and three or more n_grid."""
    seen, n_grids = set(), set()
    for t0, td, ev, ctrl in schedules:
        n = len(ctrl)
        n_grids.add(n)
        if ctrl[1].type == IMPACT:
            seen.add(("impact@1", bool(ctrl[0].sto)))
        if ctrl[0].ns > 0:
            seen.add(("switching constraint@0", bool(ctrl[0].sto)))
        if ctrl[n - 3].type == IMPACT:
            seen.add("impact@n-3")
        if ctrl[n - 2].type == LIFT:
            seen.add("lift@n-2")
        if ctrl[0].ngrids_in_phase == 1 and ctrl[0].sto:
            seen.add("one-grid first phase, sto")
        if min(c.dt for c in ctrl[:-1] if c.type != IMPACT) < 1e-5 * td.T / td.N:
            seen.add("tiny step")
    want = {("impact@1", False), ("impact@1", True), ("switching constraint@0", False), ("switching constraint@0", True), "impact@n-3", "lift@n-2", "one-grid first phase, sto", "tiny step"}
    assert want <= seen, want - seen
    assert len(n_grids) >= 3, n_grids
    return seen, n_grids


def dense_kkt_solve(dims, L, ctrl, kkt1, dx0):
    """Independent reference: assemble the full block KKT system of the equality-constrained LQ subproblem
    (no STO) for ONE OCP and solve it with numpy.  Returns dict of per-stage dx, du, lmd, xi."""
    n_grid = len(ctrl)
    N = n_grid - 1
    nx, nu, nv = dims.nx, dims.nu, dims.nv
    idx = {}
    n = 0

    def alloc(name, i, size):
        nonlocal n
        idx[(name, i)] = slice(n, n + size)
        n += size

    for i in range(n_grid):
        alloc("dx", i, nx)
        alloc("lmd", i, nx)
        if i < N and ctrl[i].type != IMPACT:
            alloc("du", i, nu)
            if ctrl[i].ns > 0:
                alloc("xi", i, ctrl[i].ns)
    Kmat = np.zeros((n, n))
    rhs = np.zeros(n)
    I = np.eye(nx)
    # row blocks are indexed by the variable whose stationarity / constraint they express
    for i in range(n_grid):
        rec = kkt1[i]
        sx, sl = idx[("dx", i)], idx[("lmd", i)]
        Qxx = mat(rec, L.k_Qxx, nx, nx)
        lx = rec[L.k_lx:L.k_lx + nx]
        # stationarity wrt dx_i : Qxx dx + Qxu du + lx + A^T lmd_{i+1} - lmd_i + C^T xi = 0
        Kmat[sx, sx] += Qxx
        Kmat[sx, sl] += -I
        rhs[sx] += -lx
        # constraint paired with lmd_i : (i=0) dx_0 = dx0 ; (i>0) A dx_{i-1} + B du_{i-1} + Fx - dx_i = 0
        if i == 0:
            Kmat[sl, sx] += I
            rhs[sl] += dx0
        if i < N:
            A = mat(rec, L.k_Fxx, nx, nx)
            Fx = rec[L.k_Fx:L.k_Fx + nx]
            sxn, sln = idx[("dx", i + 1)], idx[("lmd", i + 1)]
            Kmat[sx, sln] += A.T
            Kmat[sln, sx] += A
            Kmat[sln, sxn] += -I
            rhs[sln] += -Fx
            if ctrl[i].type != IMPACT:
                su = idx[("du", i)]
                Qxu = mat(rec, L.k_Qxu, nx, nu)
                Quu = mat(rec, L.k_Quu, nu, nu)
                lu = rec[L.k_lu:L.k_lu + nu]
                B = np.zeros((nx, nu))
                B[nv:, :] = mat(rec, L.k_Fvu, nv, nu)
                Kmat[sx, su] += Qxu
                Kmat[su, sx] += Qxu.T
                Kmat[su, su] += Quu
                Kmat[su, sln] += B.T
                Kmat[sln, su] += B
                rhs[su] += -lu
                ns = ctrl[i].ns
                if ns > 0:
                    sxi = idx[("xi", i)]
                    C = mat(rec, L.k_Phix, ns, nx)
                    D = mat(rec, L.k_Phiu, ns, nu)
                    p = rec[L.k_p:L.k_p + ns]
                    Kmat[sx, sxi] += C.T
                    Kmat[su, sxi] += D.T
                    Kmat[sxi, sx] += C
                    Kmat[sxi, su] += D
                    rhs[sxi] += -p
    sol = np.linalg.solve(Kmat, rhs)
    return {k: sol[v] for k, v in idx.items()}


def dense_kkt_solve_sto(dims, L, ctrl, kkt1, dx0):
    """Independent reference for the switching-time-optimisation path: the full KKT system of the LQ sub-problem with
    the switching-time increments ts_k of all events as unknowns (every event STO-enabled), ONE OCP, numpy dense solve.
    A stage of the phase between events p and p+1 sees Delta = ts_{p+1} - ts_p through fx (dynamics), hx / hu / h (cost
    gradient), Phit (switching constraint) and the quadratic 0.5*Qtt*Delta^2 - Qtt_prev*Delta*ts_{p+1}; the last form is
    what the reference's accumulation xi += Qtt, chi += Qtt_prev (backward_riccati_recursion_factorizer.cpp:108-120)
    amounts to in the value function 0.5*xi*Delta^2 - chi*Delta*b + 0.5*rho*b^2 that its phase transition
    (riccati_factorizer.cpp:145-175) minimises.  Returns (solution dict, phase of every grid, number of events)."""
    n_grid = len(ctrl); N = n_grid - 1
    nx, nu, nv = dims.nx, dims.nu, dims.nv
    # phase of every grid; events are numbered 1..E; phase p lies between event p and event p+1
    phase = []; p = 0
    for i in range(n_grid):
        if ctrl[i].type == LIFT: p += 1
        phase.append(p)
        if ctrl[i].type == IMPACT: p += 1
    E = p
    idx = {}; n = 0
    def alloc(name, i, size):
        nonlocal n
        idx[(name, i)] = slice(n, n + size); n += size
    for i in range(n_grid):
        alloc("dx", i, nx); alloc("lmd", i, nx)
        if i < N and ctrl[i].type != IMPACT:
            alloc("du", i, nu)
            if ctrl[i].ns > 0: alloc("xi", i, ctrl[i].ns)
    for k in range(1, E + 1): alloc("ts", k, 1)
    K = np.zeros((n, n)); rhs = np.zeros(n); I = np.eye(nx)
    def ts_terms(p):
        out = []
        if p + 1 <= E: out.append((idx[("ts", p + 1)], +1.0))
        if p >= 1: out.append((idx[("ts", p)], -1.0))
        return out
    for i in range(n_grid):
        rec = kkt1[i]; sx, sl = idx[("dx", i)], idx[("lmd", i)]
        K[sx, sx] += mat(rec, L.k_Qxx, nx, nx); K[sx, sl] += -I; rhs[sx] += -rec[L.k_lx:L.k_lx + nx]
        if i == 0:
            K[sl, sx] += I; rhs[sl] += dx0
        if i < N:
            A = mat(rec, L.k_Fxx, nx, nx); Fx = rec[L.k_Fx:L.k_Fx + nx]
            sxn, sln = idx[("dx", i + 1)], idx[("lmd", i + 1)]
            K[sx, sln] += A.T; K[sln, sx] += A; K[sln, sxn] += -I; rhs[sln] += -Fx
            if ctrl[i].type != IMPACT:
                su = idx[("du", i)]
                Qxu = mat(rec, L.k_Qxu, nx, nu); Quu = mat(rec, L.k_Quu, nu, nu)
                B = np.zeros((nx, nu)); B[nv:, :] = mat(rec, L.k_Fvu, nv, nu)
                K[sx, su] += Qxu; K[su, sx] += Qxu.T; K[su, su] += Quu; K[su, sln] += B.T; K[sln, su] += B
                rhs[su] += -rec[L.k_lu:L.k_lu + nu]
                ns = ctrl[i].ns
                if ns > 0:
                    sxi = idx[("xi", i)]
                    C = mat(rec, L.k_Phix, ns, nx); D = mat(rec, L.k_Phiu, ns, nu)
                    K[sx, sxi] += C.T; K[su, sxi] += D.T; K[sxi, sx] += C; K[sxi, su] += D; rhs[sxi] += -rec[L.k_p:L.k_p + ns]
                if ctrl[i].sto:
                    fx = rec[L.k_fx:L.k_fx + nx]; hx = rec[L.k_hx:L.k_hx + nx]; hu = rec[L.k_hu:L.k_hu + nu]
                    Qtt, h = rec[L.k_sc + 0], rec[L.k_sc + 2]
                    tt = ts_terms(phase[i])
                    for (st, sg) in tt:
                        K[sx, st] += sg * hx[:, None]; K[st, sx] += sg * hx[None, :]
                        K[su, st] += sg * hu[:, None]; K[st, su] += sg * hu[None, :]
                        K[sln, st] += sg * fx[:, None]; K[st, sln] += sg * fx[None, :]
                        rhs[st] += -sg * h
                        if ns > 0:
                            Pt = rec[L.k_Phit:L.k_Phit + ns]
                            K[sxi, st] += sg * Pt[:, None]; K[st, sxi] += sg * Pt[None, :]
                        for (st2, sg2) in tt:
                            K[st, st2] += sg * sg2 * Qtt
                    # recursion-implied cross term: - Qtt_prev * (b - a) * b
                    Qtp = rec[L.k_sc + 1]
                    pp = phase[i]
                    if pp + 1 <= E:
                        sb = idx[("ts", pp + 1)]
                        K[sb, sb] += -2.0 * Qtp
                        if pp >= 1:
                            sa = idx[("ts", pp)]
                            K[sa, sb] += Qtp; K[sb, sa] += Qtp
    sol = np.linalg.solve(K, rhs)
    return {k: sol[v] for k, v in idx.items()}, phase, E


def rel_err(a, b):
    """max |a-b| / max(|b|, tiny) over the array (relative to the block's scale, like Eigen isApprox)."""
    a, b = np.asarray(a), np.asarray(b)
    denom = max(np.max(np.abs(b)), 1e-300)
    return float(np.max(np.abs(a - b)) / denom)

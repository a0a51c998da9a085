"""Host-side mirror of the hot-path part of robotoc::UnconstrDirectMultipleShooting
(robotoc/src/unconstr/unconstr_direct_multiple_shooting.cpp:88-179) for fixed-base robots without contacts:

  evalKKT's condensing tail (unconstr_intermediate_stage.cpp:96-98)           -> condense()
  computeStepSizes :128-146, maxPrimalStepSize / maxDualStepSize :149-156     -> computeStepSizes(), max*StepSize()
  integrateSolution :159-179                                                  -> integrateSolution()

It shares the device buffers of an UnconstrRiccatiRecursion handle.  Records: include/rbt_ustage_layout.h.
"""
import ctypes

import numpy as np

from . import _lib
from .riccati import UnconstrRiccatiRecursion, _check, _vp
from .stage import VAR_Q, VAR_V, VAR_U, rbt_constraint_table

LIN, CON, EXP, SOL, XDIR, STEPS = 6, 7, 8, 9, 10, 11

_UFIELDS = ("nv nx nbox ncp l_dIDdq l_dIDdv l_dIDda l_ID l_Qxx l_Qaa l_Quu l_lx l_la l_lu l_Fx l_stride e_lu e_Quu e_stride "
            "c_slack c_dual c_res c_cmpl c_cond c_dslack c_ddual c_stride s_q s_v s_a s_u s_beta s_lmd s_gmm s_stride "
            "x_du x_dbeta x_stride").split()


def iiwa14_constraint_table(barrier=1.0e-3, fraction_to_boundary=0.995):
    """examples/iiwa14/unconstr_ocp_benchmark.cpp / config_space_ocp.cpp: joint position, velocity and torque
    lower + upper limits on the 7 joints -> 42 inequality rows per stage."""
    t = rbt_constraint_table()
    t.n_contacts = 0
    t.barrier, t.fraction_to_boundary = barrier, fraction_to_boundary
    r = 0
    for var in (VAR_Q, VAR_V, VAR_U):
        for sign in (-1, +1):
            for j in range(7):
                t.box[r].var, t.box[r].idx, t.box[r].sign = var, j, sign
                r += 1
    t.n_box = r
    return t


class UStageLayout:
    def __init__(self, nv: int, n_box: int, getter=None):
        get = getter or _lib.lib().rbt_unconstr_stage_layout_get
        for f in _UFIELDS:
            v = get(nv, n_box, f.encode())
            if v < 0:
                raise RuntimeError(f"unconstrained stage layout field {f} unknown to the library")
            setattr(self, f, v)


class UnconstrDirectMultipleShooting:
    def __init__(self, riccati: UnconstrRiccatiRecursion, table):
        self.rr = riccati
        self._lib = riccati._lib
        self._h = riccati._h
        self.table = table
        self.layout = UStageLayout(riccati.nv, table.n_box)
        _check(self._lib.rbt_unconstr_stage_setup(self._h, ctypes.byref(table)), riccati._err,
               "UnconstrDirectMultipleShooting")

    def _shape(self, stride):
        return (self.rr.batch, self.rr.N + 1, stride)

    def _up(self, which, a, stride, stream):
        if a.shape != self._shape(stride):
            raise ValueError(f"[UnconstrDirectMultipleShooting] invalid argument: expected shape {self._shape(stride)}, got {a.shape}")
        _check(self._lib.rbt_unconstr_upload(self._h, which, _vp(a), stream), self.rr._err, "UnconstrDirectMultipleShooting")

    def _down(self, which, shape, stream=None):
        out = np.empty(shape)
        _check(self._lib.rbt_unconstr_download(self._h, which, _vp(out), stream), self.rr._err, "UnconstrDirectMultipleShooting")
        _check(self._lib.rbt_unconstr_sync(self._h, stream), self.rr._err, "UnconstrDirectMultipleShooting")
        return out

    # -- reference API -----------------------------------------------------------------------------------
    def condense(self, lin=None, con=None, stream=None):
        if lin is not None:
            self._up(LIN, lin, self.layout.l_stride, stream)
        if con is not None:
            self._up(CON, con, self.layout.c_stride, stream)
        _check(self._lib.rbt_unconstr_condense(self._h, stream), self.rr._err, "UnconstrDirectMultipleShooting")

    def setSolution(self, sol, stream=None):
        self._up(SOL, sol, self.layout.s_stride, stream)

    def computeStepSizes(self, stream=None):
        _check(self._lib.rbt_unconstr_expand_and_step_sizes(self._h, stream), self.rr._err, "UnconstrDirectMultipleShooting")

    def _steps(self, stream=None):
        return self._down(STEPS, (self.rr.batch, 2), stream)

    def maxPrimalStepSize(self, stream=None):
        return self._steps(stream)[:, 0].copy()

    def maxDualStepSize(self, stream=None):
        return self._steps(stream)[:, 1].copy()

    def integrateSolution(self, stream=None):
        _check(self._lib.rbt_unconstr_update(self._h, stream), self.rr._err, "UnconstrDirectMultipleShooting")

    def iteration_host(self, lin, con, sol, dx0, stream=None):
        """UnconstrOCPSolver::updateSolution's linear-algebra body with host buffers (unconstr_ocp_solver.cpp:101-118)."""
        sol_out, con_out = np.empty_like(sol), np.empty_like(con)
        steps = np.empty((self.rr.batch, 2))
        _check(self._lib.rbt_unconstr_iteration_host(self._h, _vp(lin), _vp(con), _vp(sol), _vp(dx0), _vp(sol_out),
                                                     _vp(con_out), _vp(steps), stream), self.rr._err,
               "UnconstrDirectMultipleShooting")
        _check(self._lib.rbt_unconstr_sync(self._h, stream), self.rr._err, "UnconstrDirectMultipleShooting")
        return sol_out, con_out, steps

    # -- getters -----------------------------------------------------------------------------------------
    def getKKT(self, stream=None):
        return self._down(0, self._shape(self.rr.layout.k_stride), stream)

    def getExpansionData(self, stream=None):
        return self._down(EXP, self._shape(self.layout.e_stride), stream)

    def getConstraintsData(self, stream=None):
        return self._down(CON, self._shape(self.layout.c_stride), stream)

    def getExpandedDirection(self, stream=None):
        return self._down(XDIR, self._shape(self.layout.x_stride), stream)

    def getSolution(self, stream=None):
        return self._down(SOL, self._shape(self.layout.s_stride), stream)

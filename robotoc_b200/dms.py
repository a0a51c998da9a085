"""Host-side mirror of the part of robotoc::DirectMultipleShooting that is on the hot path
(robotoc/include/robotoc/ocp/direct_multiple_shooting.hpp:86-199, src/ocp/direct_multiple_shooting.cpp):

  evalKKT (its "Forms linear system" tail, :129-159 -> intermediate_stage.cpp:133-148)   -> condense()
  computeStepSizes :174-199, maxPrimalStepSize / maxDualStepSize :202-209                -> computeStepSizes(), max*StepSize()
  integrateSolution :212-241                                                             -> integrateSolution()

It shares the device buffers (KKT records, direction records) of a RiccatiRecursion handle, so a full hot-path
iteration is: condense -> backwardRiccatiRecursion -> forwardRiccatiRecursion -> computeStepSizes -> integrateSolution
without any host round trip.
"""
import ctypes

import numpy as np

from .riccati import RiccatiRecursion, _check, _vp
from .stage import StageDims, StageLayout

LIN, CON, EXP, SOL, XDIR, STEPS, PERF, CONTACT_POS, Q0 = 6, 7, 8, 9, 10, 11, 12, 13, 14
RBT_MAX_BODIES, RBT_MAX_CONTACTS = 32, 8
WIRE_DEVICE_ID = 2  # RBT_WIRE_DEVICE_ID (rbt_stage_layout.h)
WIRE_DEVICE_CONTACT = 4  # RBT_WIRE_DEVICE_CONTACT
WIRE_DEVICE_STATE = 16  # RBT_WIRE_DEVICE_STATE


class rbt_robot_model(ctypes.Structure):
    """include/robotoc_b200.h: floating-base tree of revolute joints in Pinocchio's joint order (body b = Pinocchio joint b+1)."""
    _fields_ = [("nv", ctypes.c_int), ("n_bodies", ctypes.c_int), ("n_contacts", ctypes.c_int), ("pad_", ctypes.c_int),
                ("parent", ctypes.c_int * RBT_MAX_BODIES), ("axis", (ctypes.c_double * 3) * RBT_MAX_BODIES),
                ("placement", (ctypes.c_double * 12) * RBT_MAX_BODIES), ("mass", ctypes.c_double * RBT_MAX_BODIES),
                ("com", (ctypes.c_double * 3) * RBT_MAX_BODIES), ("inertia", (ctypes.c_double * 9) * RBT_MAX_BODIES),
                ("contact_parent", ctypes.c_int * RBT_MAX_CONTACTS),
                ("contact_placement", (ctypes.c_double * 12) * RBT_MAX_CONTACTS), ("gravity", ctypes.c_double * 3)]


class DirectMultipleShooting:
    def __init__(self, riccati: RiccatiRecursion, sdims: StageDims, table):
        self.rr = riccati
        self._lib = riccati._lib
        self._h = riccati._h
        self.sdims = sdims
        self.table = table
        self.layout = StageLayout(sdims)
        csd = sdims.c()
        _check(self._lib.rbt_stage_setup(self._h, ctypes.byref(csd), ctypes.byref(table)), riccati._err,
               "DirectMultipleShooting")

    def _shape(self, stride):
        return (self.rr.batch, self.rr.n_grid, stride)

    def _up(self, which, a, stride, stream):
        if a.shape != self._shape(stride):
            raise ValueError(f"[DirectMultipleShooting] invalid argument: expected shape {self._shape(stride)}, got {a.shape}")
        _check(self._lib.rbt_upload(self._h, which, _vp(a), stream), self.rr._err, "DirectMultipleShooting")

    def _down(self, which, shape, stream=None):
        out = np.empty(shape)
        _check(self._lib.rbt_download(self._h, which, _vp(out), stream), self.rr._err, "DirectMultipleShooting")
        self.rr.synchronize(stream)
        return out

    # -- reference API -----------------------------------------------------------------------------------
    def condense(self, lin=None, con=None, stream=None):
        """The condensing tail of evalKKT for every stage of every OCP."""
        if lin is not None:
            self._up(LIN, lin, self.layout.l_stride, stream)
        if con is not None:
            self._up(CON, con, self.layout.c_stride, stream)
        _check(self._lib.rbt_condense(self._h, stream), self.rr._err, "DirectMultipleShooting")

    def setSolution(self, sol, stream=None):
        """Uploads the solution records (the solver state s_ of OCPSolver)."""
        self._up(SOL, sol, self.layout.s_stride, stream)

    def setConstraintData(self, con, stream=None):
        """Uploads the PDIPM records (slack, dual, residual of every inequality row)."""
        self._up(CON, con, self.layout.c_stride, stream)

    def setJointLimits(self, bound):
        """Limit of each box row of the constraint table (qmin / qmax, -vmax / vmax, -umax / umax), for linearizeJointLimits."""
        bound = np.ascontiguousarray(bound, dtype=np.float64)
        _check(self._lib.rbt_set_joint_limits(self._h, _vp(bound)), self.rr._err, "DirectMultipleShooting")

    def linearizeJointLimits(self, stream=None):
        """The joint-limit half of Constraints::linearizeConstraints on the device (rbt_linearize_joint_limits): PDIPM residuals
        of the box rows from the resident solution, and their dual terms added to the gradients of the linearization records."""
        _check(self._lib.rbt_linearize_joint_limits(self._h, stream), self.rr._err, "DirectMultipleShooting")

    def setRobotModel(self, model: rbt_robot_model):
        """Copies the robot model (rbt_robot_model: what pinocchio::Model holds for the tree) to the device, for
        linearizeInverseDynamics and the device-side inverse dynamics of the wire paths."""
        _check(self._lib.rbt_set_robot_model(self._h, ctypes.byref(model)), self.rr._err, "DirectMultipleShooting")

    def linearizeInverseDynamics(self, stream=None):
        """The inverse-dynamics rows of linearizeContactDynamics / linearizeImpactDynamics on the device
        (rbt_linearize_inverse_dynamics): IDC and dIDCdqv ID rows, M, and the beta terms of lq, lv, la | ldv, from the resident
        solution records."""
        _check(self._lib.rbt_linearize_inverse_dynamics(self._h, stream), self.rr._err, "DirectMultipleShooting")

    def setContactGains(self, gains):
        """Baumgarte gains [n_contacts, 2] = {position gain, velocity gain} of each point contact (ContactModelInfo), for
        linearizeContactKinematics and the device-side contact rows of the wire paths."""
        gains = np.ascontiguousarray(gains, dtype=np.float64)
        if gains.shape != (self.sdims.n_contacts, 2):
            raise ValueError(f"[DirectMultipleShooting] invalid argument: gains must have shape {(self.sdims.n_contacts, 2)}")
        _check(self._lib.rbt_set_contact_gains(self._h, _vp(gains)), self.rr._err, "DirectMultipleShooting")

    def setContactPositions(self, pos, stream=None):
        """Desired contact positions [batch, n_grid, n_contacts, 3] (ContactStatus::contactPosition of each grid point's phase),
        read for the active contacts of Intermediate / Lift grid points.  Resident: upload again when the planner changes them."""
        pos = np.ascontiguousarray(pos, dtype=np.float64)
        shape = (self.rr.batch, self.rr.n_grid, self.sdims.n_contacts, 3)
        if pos.shape != shape:
            raise ValueError(f"[DirectMultipleShooting] invalid argument: contact positions must have shape {shape}")
        _check(self._lib.rbt_upload(self._h, CONTACT_POS, _vp(pos), stream), self.rr._err, "DirectMultipleShooting")
        self.rr.synchronize(stream)

    def linearizeContactKinematics(self, stream=None):
        """The contact rows of linearizeContactDynamics / linearizeImpactDynamics on the device
        (rbt_linearize_contact_kinematics): J, the contact rows of dIDCdqv and IDC, and the multiplier terms of lf, lq, lv,
        la | ldv, from the resident solution records (setRobotModel, setContactGains and setContactPositions first)."""
        _check(self._lib.rbt_linearize_contact_kinematics(self._h, stream), self.rr._err, "DirectMultipleShooting")

    def setInitialConfiguration(self, q0, stream=None):
        """The measured configuration q0 [batch, nq] of OCPSolver::solve(t, q, v): grid point 0's q_prev in linearizeStateEquation
        and the device-side state-equation rows of the wire paths.  Resident: upload again with each new measurement."""
        q0 = np.ascontiguousarray(q0, dtype=np.float64)
        shape = (self.rr.batch, self.layout.nq)
        if q0.shape != shape:
            raise ValueError(f"[DirectMultipleShooting] invalid argument: q0 must have shape {shape}")
        _check(self._lib.rbt_upload(self._h, Q0, _vp(q0), stream), self.rr._err, "DirectMultipleShooting")
        self.rr.synchronize(stream)

    def linearizeStateEquation(self, stream=None):
        """The state-equation rows of linearizeStateEquation / linearizeImpactStateEquation / linearizeTerminalStateEquation on
        the device (rbt_linearize_state_equation): Fx, the three SE(3) blocks, the costate terms of lq, lv, la | ldv and, on
        schedules with a switching-time stage, the STO terms, from the resident solution records (setInitialConfiguration
        first)."""
        _check(self._lib.rbt_linearize_state_equation(self._h, stream), self.rr._err, "DirectMultipleShooting")

    def computeStepSizes(self, stream=None):
        _check(self._lib.rbt_expand_and_step_sizes(self._h, stream), self.rr._err, "DirectMultipleShooting")

    def _steps(self, stream=None):
        return self._down(STEPS, (self.rr.batch, 2), stream)

    def maxPrimalStepSize(self, stream=None):
        return self._steps(stream)[:, 0]

    def maxDualStepSize(self, stream=None):
        return self._steps(stream)[:, 1]

    def integrateSolution(self, sol=None, stream=None):
        if sol is not None:
            self._up(SOL, sol, self.layout.s_stride, stream)
        _check(self._lib.rbt_update(self._h, stream), self.rr._err, "DirectMultipleShooting")

    def evalKKT(self, lin=None, con=None, stream=None):
        """The PerformanceIndex of DirectMultipleShooting::evalKKT (direct_multiple_shooting.cpp:129-158) from the stage
        linearisations: returns [batch, 8] = {cost (0), cost_barrier, primal_feasibility, dual_feasibility, kkt_error,
        KKTError() = sqrt(kkt_error), 0, 0} per OCP."""
        if lin is not None:
            self._up(LIN, lin, self.layout.l_stride, stream)
        if con is not None:
            self._up(CON, con, self.layout.c_stride, stream)
        _check(self._lib.rbt_eval_kkt(self._h, stream), self.rr._err, "DirectMultipleShooting")
        return self._down(PERF, (self.rr.batch, 8), stream)

    def KKTError(self, stream=None):
        """OCPSolver::KKTError() (ocp_solver.cpp:429-431) per OCP, of the records currently on the device."""
        return self.evalKKT(stream=stream)[:, 5]

    def setSlackAndDualPositive(self, con=None, stream=None):
        """pdipm::setSlackAndDualPositive (pdipm.hxx:13-24) on the device-resident PDIPM records."""
        if con is not None:
            self._up(CON, con, self.layout.c_stride, stream)
        _check(self._lib.rbt_set_slack_and_dual_positive(self._h, stream), self.rr._err, "DirectMultipleShooting")

    def computeInitialStateDirection(self, dq0, v0, stream=None):
        """direct_multiple_shooting.cpp:161-165 -> state_equation.cpp:98-109.  dq0 = q0 (-) s[0].q ([batch, nv], from the host's
        robot model), v0 [batch, nv]; leaves d[0].dx in the handle's dx0 buffer (what forwardRiccatiRecursion starts from)."""
        nv = self.sdims.dims.nv
        if dq0.shape != (self.rr.batch, nv) or v0.shape != (self.rr.batch, nv):
            raise ValueError("[DirectMultipleShooting] invalid argument: dq0 and v0 must be [batch, nv]")
        buf = np.ascontiguousarray(np.concatenate([dq0, v0], axis=1))
        _check(self._lib.rbt_initial_state_direction(self._h, _vp(buf), stream), self.rr._err, "DirectMultipleShooting")
        self.rr.synchronize(stream)  # `buf` is a temporary: the copy must have been issued from live memory

    def getInitialStateDirection(self, stream=None):
        return self._down(4, (self.rr.batch, self.rr.dims.nx), stream)

    def iteration_host(self, lin, con, sol, dx0, stream=None):
        """The linear-algebra body of OCPSolver::updateSolution (src/solver/ocp_solver.cpp:118-144) in ONE call with host
        buffers (rbt_iteration_host): returns (updated solution, PDIPM record with slack / dual updated, step sizes).
        Only slack and dual of the PDIPM record come back from the device; its other fields are returned as passed in."""
        for a, st in ((lin, self.layout.l_stride), (con, self.layout.c_stride), (sol, self.layout.s_stride)):
            if a.shape != self._shape(st):
                raise ValueError(f"[DirectMultipleShooting] invalid argument: expected shape {self._shape(st)}, got {a.shape}")
        sol_out, con_out = sol.copy(), con.copy()
        steps = np.empty((self.rr.batch, 2))
        _check(self._lib.rbt_iteration_host(self._h, _vp(lin), _vp(con), _vp(sol), _vp(dx0), _vp(sol_out), _vp(con_out),
                                            _vp(steps), stream), self.rr._err, "DirectMultipleShooting")
        self.rr.synchronize(stream)
        return sol_out, con_out, steps

    def iteration_host_bytes(self, wire=False, resident=False):
        """(H2D, D2H) bytes one call moves: dense records, wire records, or wire records with resident solver state."""
        h2d, d2h = ctypes.c_longlong(), ctypes.c_longlong()
        _check(self._lib.rbt_iteration_host_bytes(self._h, 2 if resident else int(wire), ctypes.byref(h2d), ctypes.byref(d2h)),
               self.rr._err, "DirectMultipleShooting")
        return h2d.value, d2h.value

    def setWireCostStructure(self, robotoc_costs: bool, device_inverse_dynamics: bool = False,
                             device_contact_kinematics: bool = False, device_state_equation: bool = False):
        """Which cost-Hessian structure the host's wire records have: False = general (full packed triangles of Qxx, Quu, Qff),
        True = what robotoc's shipped cost components produce (Qqq dense, Qvv / Quu / Qff diagonal, Qqv = 0).
        device_inverse_dynamics: the wire records leave out M and the ID rows of dIDCdqv and IDC (and their gradients the beta
        terms); iteration_host_wire / iteration_host_resident compute them on the device (setRobotModel first).
        device_contact_kinematics: the wire records leave out J and the contact rows of dIDCdqv and IDC (and their gradients
        the multiplier terms of those rows); the wire paths compute them on the device (setRobotModel, setContactGains and
        setContactPositions first).
        device_state_equation: the wire records leave out Fx and the SE(3) blocks (and their gradients and STO sections the
        costate terms); the wire paths compute them on the device (setInitialConfiguration first)."""
        self._cost_structure = ((1 if robotoc_costs else 0) | (WIRE_DEVICE_ID if device_inverse_dynamics else 0)
                                | (WIRE_DEVICE_CONTACT if device_contact_kinematics else 0)
                                | (WIRE_DEVICE_STATE if device_state_equation else 0))
        _check(self._lib.rbt_set_wire_cost_structure(self._h, self._cost_structure), self.rr._err, "DirectMultipleShooting")

    def pack_wire(self, lin):
        """Linearization records [batch, n_grid, l_stride] -> host wire records [batch, wire doubles per OCP] of the schedule in
        force (include/rbt_stage_layout.h: packed symmetric blocks, contact blocks sized by the active contacts, no Qqf, ...)."""
        cs = getattr(self, "_cost_structure", 0)
        csd = self.sdims.c()
        ctrl, n_grid = self.rr._ctrl, self.rr.n_grid
        if n_grid == 0:
            raise RuntimeError("[DirectMultipleShooting] pack_wire: set the time discretization first")
        w = int(self._lib.rbt_wire_doubles(ctypes.byref(csd), ctrl, n_grid, cs))
        out = np.zeros((lin.shape[0], w))
        _check(self._lib.rbt_pack_wire(ctypes.byref(csd), ctrl, n_grid, cs, _vp(lin), _vp(out), lin.shape[0]), self.rr._err,
               "DirectMultipleShooting")
        return out

    def iteration_host_resident(self, wire, lin_switching, res, dx0, stream=None):
        """One iteration with the solver state (solution, slack, dual) resident on the device, as OCPSolver keeps s_ and the
        constraint data between iterations: only the wire records, the PDIPM residuals `res` [batch, n_grid, ncp] and dx0 go up.
        Initialise the state with setSolution / setConstraintData (or one iteration_host_wire call)."""
        S = self.layout
        if res.shape != (self.rr.batch, self.rr.n_grid, S.ncp):
            raise ValueError(f"[DirectMultipleShooting] invalid argument: res must have shape {(self.rr.batch, self.rr.n_grid, S.ncp)}")
        sol_out = np.zeros(self._shape(S.s_stride))
        sd_out = np.zeros(self._shape(2 * S.ncp))  # [slack (ncp) | dual (ncp)] per grid point
        steps = np.empty((self.rr.batch, 2))
        _check(self._lib.rbt_iteration_host_resident(self._h, _vp(wire), _vp(lin_switching), _vp(res), _vp(dx0), _vp(sol_out),
                                                     _vp(sd_out), _vp(steps), stream), self.rr._err, "DirectMultipleShooting")
        self.rr.synchronize(stream)
        return sol_out, sd_out, steps

    def iteration_host_wire(self, wire, lin_switching, con, sol, dx0, stream=None):
        """iteration_host with the linearisations in the wire format (29 % fewer PCIe bytes)."""
        sol_out, con_out = sol.copy(), con.copy()
        steps = np.empty((self.rr.batch, 2))
        _check(self._lib.rbt_iteration_host_wire(self._h, _vp(wire), _vp(lin_switching), _vp(con), _vp(sol), _vp(dx0),
                                                 _vp(sol_out), _vp(con_out), _vp(steps), stream), self.rr._err,
               "DirectMultipleShooting")
        self.rr.synchronize(stream)
        return sol_out, con_out, steps

    # -- data access ---------------------------------------------------------------------------------------
    def getKKT(self, stream=None):
        return self._down(0, self._shape(self.rr.layout.k_stride), stream)

    def getExpansionData(self, stream=None):
        return self._down(EXP, self._shape(self.layout.e_stride), stream)

    def getConstraintData(self, stream=None):
        return self._down(CON, self._shape(self.layout.c_stride), stream)

    def getSolution(self, stream=None):
        return self._down(SOL, self._shape(self.layout.s_stride), stream)

    def getExpandedDirection(self, stream=None):
        return self._down(XDIR, self._shape(self.layout.x_stride), stream)

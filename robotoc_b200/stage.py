"""Per-stage condense / expand / update layer (SURVEY.md 8a rows a10-a16): layouts and constraint table.

Mirrors, on the host side,
  the tail of IntermediateStage/ImpactStage/TerminalStage::evalKKT ("Forms linear system",
      robotoc/src/ocp/intermediate_stage.cpp:133-148, impact_stage.cpp:115-121, terminal_stage.cpp:102-106),
  DirectMultipleShooting::computeStepSizes / maxPrimalStepSize / maxDualStepSize / integrateSolution
      (robotoc/src/ocp/direct_multiple_shooting.cpp:174-241).
The records are described in include/rbt_stage_layout.h.
"""
import ctypes
from dataclasses import dataclass

import numpy as np

from . import _lib
from .layout import Dims

RBT_MAX_BOX_ROWS = 128
VAR_Q, VAR_V, VAR_A, VAR_U = 0, 1, 2, 3


class rbt_box_row(ctypes.Structure):
    _fields_ = [("var", ctypes.c_int), ("idx", ctypes.c_int), ("sign", ctypes.c_int)]


class rbt_constraint_table(ctypes.Structure):
    _fields_ = [("n_box", ctypes.c_int), ("n_contacts", ctypes.c_int), ("impact_friction_cone", ctypes.c_int),
                ("pad_", ctypes.c_int), ("barrier", ctypes.c_double),
                ("fraction_to_boundary", ctypes.c_double), ("box", rbt_box_row * RBT_MAX_BOX_ROWS)]


class rbt_stage_dims(ctypes.Structure):
    _fields_ = [("nv", ctypes.c_int), ("nu", ctypes.c_int), ("n_passive", ctypes.c_int), ("nf_max", ctypes.c_int),
                ("ns_max", ctypes.c_int), ("n_contacts", ctypes.c_int), ("n_box", ctypes.c_int)]


_SFIELDS = ("nv nu nx np nfm nvf nsm ncon nbox nc ncp nq l_M l_J l_D l_IDC l_Qaa l_Qff l_Qqf l_Qxx l_Quu l_lx l_la l_lf l_lu "
            "l_Fx l_lup l_se3 l_Phix l_Phia l_p l_Phit l_ha l_hf l_hx l_hu l_fx l_sc l_dgdq l_dgdf l_stride e_Z e_R e_r "
            "e_Qafqv e_Qafu e_laf e_Qxup e_Quup e_lup e_Phia e_haf e_Fqqpi e_Qaf e_Quf e_Qaa e_stride c_slack c_dual c_res c_cmpl c_cond "
            "c_dslack c_ddual c_stride s_q s_v s_a s_dv s_u s_f s_lmd s_gmm s_beta s_mu s_nup s_xi s_stride x_daf "
            "x_dbetamu x_dnup x_stride").split()


def anymal_constraint_table(barrier=1.0e-3, fraction_to_boundary=0.995, impact_friction_cone=False):
    """examples/anymal/trot.cpp:131-148: joint position / velocity / torque lower+upper limits on the 12 actuated joints
    (72 box rows) and friction cones on the 4 feet (5 rows each) -> 92 inequalities per stage.  `impact_friction_cone`:
    the same cone rows on the impact forces of Impact stages (ImpactFrictionCone, as examples/anymal/run.cpp:173-181 adds)."""
    t = rbt_constraint_table()
    t.n_contacts = 4
    t.impact_friction_cone = int(bool(impact_friction_cone))
    t.barrier, t.fraction_to_boundary = barrier, fraction_to_boundary
    r = 0
    for var, off in ((VAR_Q, 6), (VAR_V, 6), (VAR_U, 0)):
        for sign in (-1, +1):
            for j in range(12):
                t.box[r].var, t.box[r].idx, t.box[r].sign = var, off + j, sign
                r += 1
    t.n_box = r
    return t


@dataclass(frozen=True)
class StageDims:
    dims: Dims
    nf_max: int
    n_contacts: int
    n_box: int

    def c(self):
        d = self.dims
        return rbt_stage_dims(d.nv, d.nu, d.n_passive, self.nf_max, d.ns_max, self.n_contacts, self.n_box)


class StageLayout:
    def __init__(self, sdims: StageDims, getter=None):
        self.sdims = sdims
        cd = sdims.c()
        get = getter or _lib.lib().rbt_stage_layout_get
        for f in _SFIELDS:
            v = get(ctypes.byref(cd), f.encode())
            if v < 0:
                raise RuntimeError(f"stage layout field {f} unknown to the library")
            setattr(self, f, v)

"""Grid types and the GridInfo mirror (robotoc/include/robotoc/ocp/grid_info.hpp:14-92).

A drop-in host receives GridInfo from robotoc's own TimeDiscretization and fills the rbt_stage_ctrl table from it
(include/robotoc_b200/riccati_recursion.hpp does exactly that in C++); this module only holds the field mirror, the
GridType constants and the event-free control table.  The restatement of TimeDiscretization::discretize that the tests use
to build the BASELINE schedules lives in tests/schedule_fixture.py (test infrastructure).
"""
from dataclasses import dataclass

from . import _lib

INTERMEDIATE, IMPACT, LIFT, TERMINAL = 0, 1, 2, 3  # robotoc::GridType order (grid_info.hpp:14-19)


@dataclass
class GridInfo:
    """Field-for-field mirror of robotoc::GridInfo (grid_info.hpp:25-92)."""
    type: int = INTERMEDIATE
    t0: float = 0.0
    t: float = 0.0
    dt: float = 0.0
    dt_next: float = 0.0
    phase: int = 0
    stage: int = 0
    impact_index: int = -1
    lift_index: int = -1
    stage_in_phase: int = 0
    num_grids_in_phase: int = 0
    sto: bool = False
    sto_next: bool = False
    switching_constraint: bool = False


def plain_schedule(N: int, dt: float, nf: int = 0, contact_mask: int = None):
    """N Intermediate stages + Terminal, no events (e.g. a standing robot).  `contact_mask` (bit per point contact) must be
    given whenever 0 < nf < all contacts: the library does not guess which feet are closed."""
    if contact_mask is None:
        contact_mask = (1 << (nf // 3)) - 1
    if 3 * bin(contact_mask).count("1") != nf:
        raise ValueError("[plain_schedule] invalid argument: 3 * popcount(contact_mask) must equal nf")
    arr = (_lib.rbt_stage_ctrl * (N + 1))()
    for i in range(N + 1):
        arr[i].type = INTERMEDIATE if i < N else TERMINAL
        arr[i].dt = dt if i < N else 0.0
        arr[i].nf = nf
        arr[i].contact_mask = contact_mask
        arr[i].ngrids_in_phase = N if i < N else 0
        arr[i].ineq_gate = max(0, 2 - i) if i < N else 0  # position- / velocity-level limits act from stage 2 / 1 on
    return arr

"""robotoc_b200 -- H100-native (sm_90a) Riccati / KKT inner loop behind robotoc's OCPSolver API.

Host-side Python mirror of the reference interface for the hot path only (SURVEY.md section 8):
  RiccatiRecursion / UnconstrRiccatiRecursion  <-> robotoc/include/robotoc/riccati/*.hpp
  TimeDiscretization (control table producer)  <-> robotoc/src/ocp/time_discretization.cpp
All compute goes through the C ABI of librobotoc_b200.so (include/robotoc_b200.h); there is no CPU path.
"""
from .layout import Dims, Layout, ULayout  # noqa: F401
from .grid import GridInfo, plain_schedule  # noqa: F401
from .riccati import RiccatiRecursion, UnconstrRiccatiRecursion  # noqa: F401
from .stage import StageDims, StageLayout, anymal_constraint_table  # noqa: F401
from .dms import DirectMultipleShooting  # noqa: F401
from .line_search import LineSearch, LineSearchSettings  # noqa: F401

ANYMAL = Dims(nv=18, nu=12, ns_max=12, n_passive=6)
IIWA14_NV = 7
from .unconstr_dms import UnconstrDirectMultipleShooting, iiwa14_constraint_table  # noqa: F401

// oracle/ref_wrap/ref_discretize_wrap.cpp -- TEST INFRASTRUCTURE.  C entry point to the reference's own
// robotoc::TimeDiscretization (src/ocp/time_discretization.cpp) and robotoc::ContactSequence (src/planner/), compiled
// unmodified into _ref/libref_discretize.so (Makefile.ref).  tests/test_schedule_fixture.py compares the discretization
// restatement of tests/schedule_fixture.py with it, field by field.
//
// This translation unit must see the reference's robotoc/ocp/time_discretization.hpp, not the stand-in under shim/: the
// build puts a link to the former first on the include path.
#include <memory>
#include <vector>

#include "robotoc/ocp/time_discretization.hpp"
#include "robotoc/planner/contact_sequence.hpp"
#include "robotoc/robot/robot.hpp"

extern "C" {

// One ContactSequence of ANYmal's four point contacts (the shim's Robot(18, true, 4)): the initial contact set masks[0]
// and n_events events, event k at times[k] switching to masks[k + 1] (bit c = contact c active), STO enabled where
// sto[k] != 0.  discretize(t0), then, when phase_based != 0, correctTimeSteps(t0) as OCPSolver::discretize applies it
// (ocp_solver.cpp:96-100).  Per grid point i of the result: ints[i * 10 + ...] = {type, phase, stage, impact_index,
// lift_index, stage_in_phase, num_grids_in_phase, sto, sto_next, switching_constraint}, dbls[i * 4 + ...] = {t0, t, dt,
// dt_next}.  Returns the number of grid points, -1 if it exceeds max_grid, -2 if the reference throws.
int ref_discretize(double T, int N, int n_events, const int* masks, const double* times, const int* sto, double t0,
                   int phase_based, int max_grid, int* ints, double* dbls) {
  try {
    const robotoc::Robot robot(18, true, 4);
    auto status = [&](int mask) {
      robotoc::ContactStatus cs = robot.createContactStatus();
      for (int c = 0; c < 4; ++c) {
        if (mask & (1 << c)) cs.activateContact(c);
      }
      return cs;
    };
    auto seq = std::make_shared<robotoc::ContactSequence>(robot, n_events);
    seq->init(status(masks[0]));
    for (int k = 0; k < n_events; ++k) seq->push_back(status(masks[k + 1]), times[k], sto[k] != 0);
    robotoc::TimeDiscretization td(T, N, n_events);
    td.discretize(seq, t0);
    if (phase_based) td.correctTimeSteps(seq, t0);
    const int n = td.size();
    if (n > max_grid) return -1;
    for (int i = 0; i < n; ++i) {
      const robotoc::GridInfo& g = td[i];
      int* o = ints + 10 * i;
      o[0] = static_cast<int>(g.type);
      o[1] = g.phase;
      o[2] = g.stage;
      o[3] = g.impact_index;
      o[4] = g.lift_index;
      o[5] = g.stage_in_phase;
      o[6] = g.num_grids_in_phase;
      o[7] = g.sto;
      o[8] = g.sto_next;
      o[9] = g.switching_constraint;
      double* d = dbls + 4 * i;
      d[0] = g.t0;
      d[1] = g.t;
      d[2] = g.dt;
      d[3] = g.dt_next;
    }
    return n;
  } catch (...) {
    return -2;
  }
}

}  // extern "C"

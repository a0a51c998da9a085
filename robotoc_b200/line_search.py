"""Host-side mirror of robotoc::LineSearch's filter method for a BATCH of OCPs
(robotoc/include/robotoc/line_search/line_search.hpp, src/line_search/line_search.cpp:58-86,
line_search_settings.hpp, line_search_filter.cpp) on top of the C ABI (rbt_line_search_*).

The reference evaluates the trial step sizes alpha_max * 0.75^k one after the other; here all trials are generated in one launch
(an extra batch axis) and the acceptance loop runs per OCP on the device.  What the library cannot do is evalOCP at the trial
points (stage costs and dynamics residuals need the robot model): the caller passes an `evaluate(trial, alphas)` callable that
returns cost[k, b] (without the barrier part) and violation[k, b] -- on the reference side that is
DirectMultipleShooting::evalOCP on s_trial.
"""
import ctypes
from dataclasses import dataclass

import numpy as np

from .riccati import _check, _vp


@dataclass
class LineSearchSettings:
    """line_search_settings.hpp:18-44 (Filter method)."""
    step_size_reduction_rate: float = 0.75
    min_step_size: float = 0.05
    filter_cost_reduction_rate: float = 0.005
    filter_constraint_violation_reduction_rate: float = 0.005


class LineSearch:
    def __init__(self, dms, settings: LineSearchSettings = None):
        self.dms = dms
        self.settings = settings or LineSearchSettings()
        s = self.settings
        if s.filter_cost_reduction_rate <= 0:
            raise ValueError("[LineSearchFilter] invalid argument: cost_reduction_rate must be positive!")
        if s.filter_constraint_violation_reduction_rate <= 0:
            raise ValueError("[LineSearchFilter] invalid argument: constraint_violation_reduction_rate must be positive!")
        self._lib, self._h = dms._lib, dms._h
        self.trial_doubles = int(self._lib.rbt_trial_doubles())

    def numTrials(self, max_primal_step_size=1.0):
        """How many step sizes the reference loop can visit: alpha_max * rate^k > min_step_size."""
        s = self.settings
        k = 0
        a = float(np.max(max_primal_step_size))
        while a > s.min_step_size and k < 64:
            a *= s.step_size_reduction_rate
            k += 1
        return max(k, 1)

    def trialSolutions(self, n_trials, want_trials=True, stream=None):
        """integratePrimalSolution for n_trials step sizes at once (call after computeStepSizes, before integrateSolution).
        Returns (alphas [k, b], barrier [k, b], trial [k, b, n_grid, 80] or None)."""
        rr = self.dms.rr
        alphas = np.empty((n_trials, rr.batch))
        barrier = np.empty((n_trials, rr.batch))
        trial = np.empty((n_trials, rr.batch, rr.n_grid, self.trial_doubles)) if want_trials else None
        _check(self._lib.rbt_line_search_trials(self._h, n_trials, self.settings.step_size_reduction_rate, _vp(alphas), _vp(barrier),
                                                _vp(trial), stream), rr._err, "LineSearch")
        rr.synchronize(stream)
        return alphas, barrier, trial

    def computeStepSize(self, cost0, violation0, evaluate, stream=None):
        """LineSearch::computeStepSize (Filter method) for every OCP of the batch.  cost0 / violation0: [batch], cost + barrier and
        primal feasibility of the current iterate (dms.getEval()).  evaluate(trial, alphas) -> (cost [k, b], violation [k, b]).
        Returns (primal step size [batch], accepted trial index [batch], -1 where none was accepted)."""
        rr = self.dms.rr
        n_trials = self.numTrials(self.dms.maxPrimalStepSize(stream))
        alphas, barrier, trial = self.trialSolutions(n_trials, True, stream)
        cost, viol = evaluate(trial, alphas)
        cost, viol = np.ascontiguousarray(cost, dtype=np.float64), np.ascontiguousarray(viol, dtype=np.float64)
        if cost.shape != (n_trials, rr.batch) or viol.shape != (n_trials, rr.batch):
            raise ValueError("[LineSearch] invalid argument: evaluate() must return [n_trials, batch] arrays")
        s = self.settings
        step = np.empty(rr.batch)
        acc = np.empty(rr.batch, dtype=np.int32)
        c0, v0 = np.ascontiguousarray(cost0, dtype=np.float64), np.ascontiguousarray(violation0, dtype=np.float64)
        _check(self._lib.rbt_line_search_filter(self._h, n_trials, s.step_size_reduction_rate, s.min_step_size,
                                                s.filter_cost_reduction_rate, s.filter_constraint_violation_reduction_rate, _vp(c0),
                                                _vp(v0), _vp(cost), _vp(viol), _vp(step), acc.ctypes.data_as(ctypes.c_void_p), stream),
               rr._err, "LineSearch")
        rr.synchronize(stream)
        return step, acc

    def clearHistory(self, stream=None):
        _check(self._lib.rbt_line_search_clear_history(self._h, stream), self.dms.rr._err, "LineSearch")

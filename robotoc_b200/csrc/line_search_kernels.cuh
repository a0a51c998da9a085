// line_search_kernels.cuh -- SURVEY.md 8f-3: the model-free half of robotoc::LineSearch, batched over the trial step sizes.
//   LineSearch::lineSearchFilterMethod   src/line_search/line_search.cpp:58-86   (alpha_k = alpha_max * 0.75^k, one after the other)
//   DirectMultipleShooting::integratePrimalSolution   src/ocp/direct_multiple_shooting.cpp:244-266 (SplitSolution::integrate +
//   Constraints::updateSlack)                          -> trial_solution_kernel: ALL k in one launch (extra batch axis)
//   LineSearchFilter::isAccepted / augment              src/line_search/line_search_filter.cpp:25-56 -> line_search_filter_kernel
// evalOCP at the trial points (costs, dynamics residuals) needs the robot model and stays with the host / a GPU front-end; of
// its PerformanceIndex only the log-barrier of the trial slacks is computed here.
#pragma once
#include "spatial.cuh"        // integrate_free_flyer_dev
#include "stage_kernels.cuh"  // StageParams

namespace rbt {

enum { T_Q = 0, T_V = 20, T_A = 38, T_U = 56, T_F = 68, T_STRIDE = 80 };  // trial record: q | v | a or dv | u | f

struct TrialParams {
  StageParams sp;
  int n_trials;
  double rate;
  double* alphas;         // [n_trials][batch]
  double* trial;          // [n_trials][batch][n_grid][T_STRIDE]
  double* stage_barrier;  // [n_trials][batch][n_grid]
  double* barrier;        // [n_trials][batch]
};

// one warp per (trial, OCP, stage)
__global__ void __launch_bounds__(128) trial_solution_kernel(const TrialParams q) {
  const StageParams& p = q.sp;
  const rbt_stage_layout& S = p.S;
  const rbt_layout& K = p.K;
  const long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const long long per_trial = (long long)p.batch * p.n_grid;
  if (w >= per_trial * q.n_trials) return;
  const int k = int(w / per_trial);
  const long long o = w % per_trial;  // (b, i)
  const int b = int(o / p.n_grid), i = int(o % p.n_grid);
  const rbt_stage_ctrl c = p.ctrl[i];
  double alpha = p.steps[2 * b];
  for (int e = 0; e < k; ++e) alpha *= q.rate;
  const double* sol = p.sol + size_t(o) * S.s_stride;
  const double* d = p.dir + size_t(o) * K.d_stride;
  const double* xd = p.xd + size_t(o) * S.x_stride;
  const double* con = p.con + size_t(o) * S.c_stride;
  double* tr = q.trial + size_t(w) * T_STRIDE;
  const int nv = S.nv, nu = S.nu;
  const bool terminal = c.type == RBT_TERMINAL, impact = c.type == RBT_IMPACT;
  for (int e = lane; e < T_STRIDE; e += 32) tr[e] = 0.0;
  __syncwarp();
  if (S.np == 6) {
    if (lane == 0) {
      double qq[7];
      for (int e = 0; e < 7; ++e) qq[e] = sol[S.s_q + e];
      integrate_free_flyer_dev(qq, d + K.d_dx, alpha);
      for (int e = 0; e < 7; ++e) tr[T_Q + e] = qq[e];
    }
    for (int e = 6 + lane; e < nv; e += 32) tr[T_Q + e + 1] = sol[S.s_q + e + 1] + alpha * d[K.d_dx + e];
  } else {
    for (int e = lane; e < nv; e += 32) tr[T_Q + e] = sol[S.s_q + e] + alpha * d[K.d_dx + e];
  }
  for (int e = lane; e < nv; e += 32) tr[T_V + e] = sol[S.s_v + e] + alpha * d[K.d_dx + nv + e];
  double lb = 0.0;
  if (!terminal) {
    for (int e = lane; e < nv; e += 32) tr[T_A + e] = (impact ? sol[S.s_dv + e] : sol[S.s_a + e]) + alpha * xd[S.x_daf + e];
    if (!impact)
      for (int e = lane; e < nu; e += 32) tr[T_U + e] = sol[S.s_u + e] + alpha * d[K.d_du + e];
    for (int e = lane; e < c.nf; e += 32) tr[T_F + e] = sol[S.s_f + e] + alpha * xd[S.x_daf + nv + e];
    if (!impact || p.tab.impact_friction_cone != 0) {
      for (int r = lane + (impact ? S.nbox : 0); r < S.nc; r += 32) {
        if (r >= S.nbox && !((c.contact_mask >> ((r - S.nbox) / 5)) & 1)) continue;
        if (r < S.nbox && __ldg(p.row_level + r) + c.ineq_gate > 2) continue;
        lb -= p.tab.barrier * log(con[S.c_slack + r] + alpha * con[S.c_dslack + r]);
      }
    }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) lb += __shfl_xor_sync(0xffffffffu, lb, s);
  if (lane == 0) q.stage_barrier[w] = lb;
}

// one thread per (trial, OCP): horizon sum in stage order, and the step size of the trial
__global__ void trial_reduce_kernel(const TrialParams q) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= q.n_trials * q.sp.batch) return;
  const int k = e / q.sp.batch, b = e % q.sp.batch;
  double alpha = q.sp.steps[2 * b];
  for (int s = 0; s < k; ++s) alpha *= q.rate;
  const double* sb = q.stage_barrier + size_t(e) * q.sp.n_grid;
  double acc = 0.0;
  for (int i = 0; i < q.sp.n_grid; ++i) acc += sb[i];
  q.barrier[e] = acc;
  q.alphas[e] = alpha;
}

struct FilterParams {
  int batch, n_trials, cap;
  double rate, min_step, cost_rate, viol_rate;
  const double* steps;                                 // [batch][2]
  const double *cost0, *viol0;                         // [batch]: cost + barrier and primal feasibility of the current iterate
  const double *cost, *barrier, *viol;                 // [n_trials][batch]
  double* filt;                                        // [batch][2 * cap]
  int* nfilt;                                          // [batch]
  double* out_step;                                    // [batch]
  int* out_k;                                          // [batch]
};

__device__ __forceinline__ bool filter_accepted_dev(const double* f, int n, double cr, double vr, double cost, double viol) {
  if (n == 0) return true;
  for (int e = 0; e < n; ++e)
    if (cost < f[2 * e] - cr * f[2 * e + 1] || viol < (1.0 - vr) * f[2 * e + 1]) return true;
  return false;
}
__device__ __forceinline__ void filter_augment_dev(double* f, int& n, int cap, double cr, double vr, double cost, double viol) {
  if (!filter_accepted_dev(f, n, cr, vr, cost, viol)) return;
  int w = 0;
  for (int e = 0; e < n; ++e)
    if (!(f[2 * e] <= cost && f[2 * e + 1] <= viol)) {
      f[2 * w] = f[2 * e];
      f[2 * w + 1] = f[2 * e + 1];
      ++w;
    }
  if (w < cap) {
    f[2 * w] = cost;
    f[2 * w + 1] = viol;
    ++w;
  }
  n = w;
}

// one thread per OCP: the sequential acceptance loop of lineSearchFilterMethod over the pre-evaluated trials
__global__ void line_search_filter_kernel(const FilterParams q) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= q.batch) return;
  double* f = q.filt + size_t(b) * 2 * q.cap;
  int n = q.nfilt[b];
  if (n == 0) filter_augment_dev(f, n, q.cap, q.cost_rate, q.viol_rate, q.cost0[b], q.viol0[b]);
  double alpha = q.steps[2 * b];
  int k = 0, acc = -1;
  while (alpha > q.min_step && k < q.n_trials) {
    const double c = q.cost[size_t(k) * q.batch + b] + q.barrier[size_t(k) * q.batch + b], v = q.viol[size_t(k) * q.batch + b];
    if (filter_accepted_dev(f, n, q.cost_rate, q.viol_rate, c, v)) {
      filter_augment_dev(f, n, q.cap, q.cost_rate, q.viol_rate, c, v);
      acc = k;
      break;
    }
    alpha *= q.rate;
    ++k;
  }
  q.nfilt[b] = n;
  q.out_step[b] = alpha;
  q.out_k[b] = acc;
}

}  // namespace rbt

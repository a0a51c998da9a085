// stage_kernels.cuh -- stage-parallel kernels of the hot path around the Riccati sweeps (SURVEY.md 8a rows a10-a16).
//
//   mjtjinv_kernel      Z = [[M,J^T],[J,0]]^-1 (Robot::computeMJtJinv, robot.hxx:642-683): one warp per stage, DMMA products
//   condense_kernel     PDIPM condensing + contact/impact dynamics condensing + floating-base state-equation correction
//                       (intermediate_stage.cpp:133-148, contact_dynamics.cpp:55-164, impact_dynamics.cpp:38-80,
//                        state_equation.cpp:68-87, joint_*_limit.cpp:68-75, friction_cone.cpp:194-235, pdipm.hxx:27-100)
//   expand_kernel       primal expansion, slack/dual directions, fraction-to-boundary step sizes with the min over the horizon
//                       (contact_dynamics.cpp:167-174, friction_cone.cpp:238-268, pdipm.hxx:121-164,
//                        direct_multiple_shooting.cpp:174-209)
//   update_kernel       dual expansion, costate correction, solution integrate, slack/dual update
//                       (contact_dynamics.cpp:177-202, state_equation.cpp:90-95, split_solution.cpp:58-90)
//   unpack_wire_kernel  host wire records (packed symmetric blocks) -> linearization records, for rbt_iteration_host_wire
//
// Unlike the Riccati sweeps these have NO dependency between stages: the grid is batch x n_grid CTAs (48k for config 3),
// every stage is an independent small dense problem held in shared memory: inputs arrive by cp.async.bulk onto an mbarrier,
// every dense product runs on the fp64 tensor pipe (DMMA m8n8k4), mat-vecs are split over the warps of the CTA.
#pragma once
#include "rbt_device.cuh"
#include "riccati_backward.cuh"  // warp_cholesky, chol_solve_smem
#include "../../include/rbt_stage_layout.h"

namespace rbt {

#define RBT_MAX_TARGETS 96
struct StageParams {
  rbt_layout K;
  rbt_stage_layout S;
  rbt_constraint_table tab;
  const rbt_stage_ctrl* ctrl;
  int n_grid;
  int batch;
  const double* lin;
  double* con;
  double* kkt;
  double* ex;
  double* dir;
  double* xd;
  double* sol;
  double* steps;  // [batch][2]
  int* info;
  const int4* tgt;  // [RBT_MAX_TARGETS] box rows acting on target (var, idx) = var*nv + idx (u: 3*nv + idx), ascending:
                    // (row + 1) * sign of the row, 0 = none
  const int* row_level;  // [n_box] 2 = position-, 1 = velocity-, 0 = acceleration-level row: acts iff level + ctrl.ineq_gate <= 2
};

// C(m x n, ld ldc) = beta*C + alpha * op(A) op(B); all operands in shared (or global) memory; every thread of the CTA calls.
__device__ __forceinline__ void cta_gemm(int ta, int tb, int m, int n, int k, double alpha, const double* A, int lda,
                                         const double* B, int ldb, double beta, double* C, int ldc) {
  for (int e = threadIdx.x; e < m * n; e += blockDim.x) {
    const int i = e % m, j = e / m;
    double acc = 0.0;
    for (int l = 0; l < k; ++l) {
      const double a = ta ? A[l + i * lda] : A[i + l * lda];
      const double b = tb ? B[j + l * ldb] : B[l + j * ldb];
      acc = fma(a, b, acc);
    }
    const double c0 = (beta == 0.0) ? 0.0 : beta * C[i + j * ldc];
    C[i + j * ldc] = fma(alpha, acc, c0);
  }
}

__device__ __forceinline__ void inv3_dev(const double* A, int lda, double* B, int ldb) {
  const double a = A[0], b = A[lda], c = A[2 * lda], d = A[1], e = A[1 + lda], f = A[1 + 2 * lda], g = A[2], h = A[2 + lda],
               i = A[2 + 2 * lda];
  const double det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
  const double r = 1.0 / det;
  B[0] = (e * i - f * h) * r; B[ldb] = (c * h - b * i) * r; B[2 * ldb] = (b * f - c * e) * r;
  B[1] = (f * g - d * i) * r; B[1 + ldb] = (a * i - c * g) * r; B[1 + 2 * ldb] = (c * d - a * f) * r;
  B[2] = (d * h - e * g) * r; B[2 + ldb] = (b * g - a * h) * r; B[2 + 2 * ldb] = (a * e - b * d) * r;
}

// SE3JacobianInverse::compute (se3_jacobian_inverse.hxx:17-32); one thread; Jac may be global, Jinv shared/global (ld 6)
__device__ __noinline__ void se3_jac_inverse_dev(const double* Jac, double* Jinv) {
  double tmp[9];
  for (int q = 0; q < 36; ++q) Jinv[q] = 0.0;
  inv3_dev(Jac, 6, Jinv, 6);
  inv3_dev(Jac + 3 + 18, 6, Jinv + 3 + 18, 6);
  for (int j = 0; j < 3; ++j)
    for (int i = 0; i < 3; ++i) {
      double acc = 0.0;
      for (int l = 0; l < 3; ++l) acc = fma(Jac[i + (3 + l) * 6], Jinv[(3 + l) + (3 + j) * 6], acc);
      tmp[i + 3 * j] = acc;
    }
  for (int j = 0; j < 3; ++j)
    for (int i = 0; i < 3; ++i) {
      double acc = 0.0;
      for (int l = 0; l < 3; ++l) acc = fma(Jinv[i + l * 6], tmp[l + 3 * j], acc);
      Jinv[i + (3 + j) * 6] = -acc;
    }
}

// ------------------------------------------------------------------------------------------------------------------
// K1: Z = [[M, J^T],[J, 0]]^-1  (Robot::computeMJtJinv, include/robotoc/robot/robot.hxx:642-683, dense restatement)
//
// One WARP per stage, no CTA barrier.  With M = L L^T, X = L^-1, W = X J^T, S = W^T W = Ls Ls^T, Y = Ls^-1, V = W Y^T,
// U = X^T V:      Z11 = X^T X - U U^T,   Z12 = U Y,   Z22 = -Y^T Y.
// The two Choleskys and the two triangular inverses are dependency chains on one warp (lane = row / column); the seven
// products run on the fp64 tensor pipe (DMMA m8n8k4, ~200 per stage) fed from 11 KB of shared memory per warp, so ~20
// stages per SM are in flight and hide each other's fp64 latency.  Z goes to the expansion record; K2 reads it from L2.
// Cholesky factor of the leading n x n block of A (lower triangle, column-major, leading dimension LD) by ONE warp: lane r
// holds row r in registers; column j is published through shared memory (it is the storage of L anyway) and read back by
// every lane with 16-byte loads.  Rows / columns >= n are carried as identity (no per-element predicates: entries above the
// diagonal of a lane's row are scratch, and what is stored beyond n is the identity).  Pivots use the MUFU-seeded reciprocal
// square root.  Writes L over A and dinv[j] = 1 / L[j][j].
// (Predicating every update on the runtime n and on lane >= k costs many more instructions; a pure shuffle version is larger
//  too: ptxas wraps every shuffle of this divergence-prone code in WARPSYNC / ENDCOLLECTIVE.)
template <int NMAX, int LD>
__device__ __forceinline__ bool warp_cholesky_ld(double* A, int n, double* dinv) {
  static_assert(NMAX <= 32 && NMAX % 2 == 0 && LD % 2 == 0, "one row per lane; 16-byte column loads of row pairs");
  const int lane = threadIdx.x & 31;
  double a[NMAX];
#pragma unroll
  for (int k = 0; k < NMAX; ++k) a[k] = (lane < n) ? ((k <= lane && k < n) ? A[lane + k * LD] : 0.0) : ((k == lane) ? 1.0 : 0.0);
  bool ok = true;
#pragma unroll
  for (int j = 0; j < NMAX; ++j) {
    const double d = __shfl_sync(0xffffffffu, a[j], j);
    ok = ok && (d > 0.0);
    const double inv = fast_rsqrt(d);
    const double lij = a[j] * inv;  // lane j: sqrt(d); lanes < j: scratch
    if (lane >= j && lane < NMAX) A[lane + j * LD] = lij;
    if (lane == j) dinv[j] = inv;
    __syncwarp();
#pragma unroll
    for (int k0 = (j + 1) & ~1; k0 < NMAX; k0 += 2) {  // column j, two rows per load (k0 even, LD even: 16-byte aligned)
      const double2 l2 = *reinterpret_cast<const double2*>(A + k0 + j * LD);
      if (k0 > j) a[k0] = fma(-lij, l2.x, a[k0]);
      a[k0 + 1] = fma(-lij, l2.y, a[k0 + 1]);
    }
  }
  __syncwarp();
  return ok;
}

// C(M x N) = sum_k fa(i, k) * fb(k, j) on one warp; st(i, j, value) stores one element (overlapped tiles store twice).
template <int M, int N, int K, class FA, class FB, class ST>
__device__ __forceinline__ void warp_gemm(FA fa, FB fb, ST st) {
  constexpr int TM_ = num_tiles(M), TN_ = num_tiles(N);
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int m = 0; m < TM_; ++m) {
    const int i0 = tile_off(m, M);
    double acc[TN_][2];
#pragma unroll
    for (int n = 0; n < TN_; ++n) acc[n][0] = acc[n][1] = 0.0;
    warp_mma_band<K, TN_, N>(acc, i0, fa, fb);
#pragma unroll
    for (int n = 0; n < TN_; ++n) {
      const int j0 = tile_off(n, N);
      st(i0 + g, j0 + 2 * t, acc[n][0]);
      st(i0 + g, j0 + 2 * t + 1, acc[n][1]);
    }
  }
}

template <int NV, int NFM>
struct MjtjCfg {
  static constexpr int WARPS = 2;
  // M | J are adjacent in the linearization record: one bulk copy lands both
  static constexpr int o_L = 0, o_J = o_L + ((NV * NV + 1) & ~1), o_X = o_J + ((NFM * NV + 1) & ~1), o_W = o_X + NV * NV,
                       o_S = o_W + NV * NFM, o_Y = o_S + NFM * NFM, o_d = o_Y + NFM * NFM, o_bar = o_d + 32,
                       PER_WARP = o_bar + 2;
  static constexpr int MJ = o_X;  // doubles copied
};

template <int NV, int NFM>
__global__ void __launch_bounds__(32 * MjtjCfg<NV, NFM>::WARPS, 10) mjtjinv_kernel(const StageParams p) {
  using C = MjtjCfg<NV, NFM>;
  constexpr int NVF = NV + NFM;
  __shared__ __align__(16) double smem[C::WARPS * C::PER_WARP];
  const rbt_stage_layout& S = p.S;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const size_t o = size_t(blockIdx.x) * C::WARPS + wid;
  if (o >= size_t(p.batch) * p.n_grid) return;
  const int i = int(o % p.n_grid), b = int(o / p.n_grid);
  const rbt_stage_ctrl c = p.ctrl[i];
  if (c.type == RBT_TERMINAL) return;
  const int nf = c.nf;
  const double* lin = p.lin + o * S.l_stride;
  double* Z = p.ex + o * S.e_stride + S.e_Z;
  double* sL = smem + wid * C::PER_WARP + C::o_L;
  double* sX = smem + wid * C::PER_WARP + C::o_X;
  double* sJ = smem + wid * C::PER_WARP + C::o_J;  // later V (NV x NFM, ld NV)
  double* sW = smem + wid * C::PER_WARP + C::o_W;  // later U
  double* sS = smem + wid * C::PER_WARP + C::o_S;
  double* sY = smem + wid * C::PER_WARP + C::o_Y;
  double* dinv = smem + wid * C::PER_WARP + C::o_d;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + wid * C::PER_WARP + C::o_bar);
  int bad = 0;
  if (lane == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
    mbar_expect_tx(bar, uint32_t(C::MJ) * 8u);
    tma_load_1d(sL, lin + S.l_M, uint32_t(C::MJ) * 8u, bar);
  }
  for (int e = lane; e < NFM * NFM; e += 32) sY[e] = 0.0;
  __syncwarp();
  mbar_wait(bar, 0);
  for (int e = lane; e < NFM * NV; e += 32)
    if ((e % NFM) >= nf) sJ[e] = 0.0;
  __syncwarp();
  if (!warp_cholesky_ld<NV, NV>(sL, NV, dinv)) bad |= 4;
  __syncwarp();
  if (lane < NV) {  // X = L^-1, one column per lane (forward substitution; rows above the diagonal stay zero)
    double x[NV];
#pragma unroll
    for (int a = 0; a < NV; ++a) x[a] = (a == lane) ? 1.0 : 0.0;
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      x[k] *= dinv[k];
#pragma unroll
      for (int a0 = (k + 1) & ~1; a0 < NV; a0 += 2) {  // column k of L, two rows per (16-byte, broadcast) load
        const double2 l2 = *reinterpret_cast<const double2*>(sL + a0 + k * NV);
        if (a0 > k) x[a0] = fma(-l2.x, x[k], x[a0]);
        if (a0 + 1 < NV) x[a0 + 1] = fma(-l2.y, x[k], x[a0 + 1]);
      }
    }
#pragma unroll
    for (int a = 0; a < NV; ++a) sX[a + lane * NV] = x[a];
  }
  __syncwarp();
  if (nf > 0) {
    // W = X J^T
    warp_gemm<NV, NFM, NV>([&](int ii, int k) { return sX[ii + k * NV]; }, [&](int k, int j) { return sJ[j + k * NFM]; },
                           [&](int ii, int j, double v) { sW[ii + j * NV] = v; });
    __syncwarp();
    // S = W^T W
    warp_gemm<NFM, NFM, NV>([&](int ii, int k) { return sW[k + ii * NV]; }, [&](int k, int j) { return sW[k + j * NV]; },
                            [&](int ii, int j, double v) { sS[ii + j * NFM] = v; });
    __syncwarp();
    if (!warp_cholesky_ld<NFM, NFM>(sS, nf, dinv)) bad |= 8;
    __syncwarp();
    if (lane < nf) {  // Y = Ls^-1
      double x[NFM];
#pragma unroll
      for (int a = 0; a < NFM; ++a) x[a] = (a == lane) ? 1.0 : 0.0;
#pragma unroll
      for (int k = 0; k < NFM; ++k) {
        // (rows / columns >= nf of Ls are the identity -- warp_cholesky_ld -- so the inactive part needs no predicate: it
        //  stays e_lane there, and lanes >= nf do not run this block)
        x[k] *= dinv[k];
#pragma unroll
        for (int a0 = (k + 1) & ~1; a0 < NFM; a0 += 2) {
          const double2 l2 = *reinterpret_cast<const double2*>(sS + a0 + k * NFM);
          if (a0 > k) x[a0] = fma(-l2.x, x[k], x[a0]);
          if (a0 + 1 < NFM) x[a0 + 1] = fma(-l2.y, x[k], x[a0 + 1]);
        }
      }
#pragma unroll
      for (int a = 0; a < NFM; ++a) sY[a + lane * NFM] = x[a];
    }
    __syncwarp();
    // V = W Y^T   (overwrites J)
    warp_gemm<NV, NFM, NFM>([&](int ii, int k) { return sW[ii + k * NV]; }, [&](int k, int j) { return sY[j + k * NFM]; },
                            [&](int ii, int j, double v) { sJ[ii + j * NV] = v; });
    __syncwarp();
    // U = X^T V   (overwrites W)
    warp_gemm<NV, NFM, NV>([&](int ii, int k) { return sX[k + ii * NV]; }, [&](int k, int j) { return sJ[k + j * NV]; },
                           [&](int ii, int j, double v) { sW[ii + j * NV] = v; });
  } else {
    for (int e = lane; e < NV * NFM; e += 32) sW[e] = 0.0;
  }
  __syncwarp();
  {  // Z11 = X^T X - U U^T
    constexpr int TV_ = num_tiles(NV);
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int m = 0; m < TV_; ++m) {
      const int i0 = tile_off(m, NV);
      double acc[TV_][2];
#pragma unroll
      for (int n = 0; n < TV_; ++n) acc[n][0] = acc[n][1] = 0.0;
      warp_mma_band<NV, TV_, NV>(acc, i0, [&](int ii, int k) { return sX[k + ii * NV]; },
                                 [&](int k, int j) { return sX[k + j * NV]; });
      warp_mma_band<NFM, TV_, NV>(acc, i0, [&](int ii, int l) { return -sW[ii + l * NV]; },
                                  [&](int l, int j) { return sW[j + l * NV]; });
#pragma unroll
      for (int n = 0; n < TV_; ++n) {
        const int j0 = tile_off(n, NV);
        Z[(i0 + g) + (j0 + 2 * t) * NVF] = acc[n][0];
        Z[(i0 + g) + (j0 + 2 * t + 1) * NVF] = acc[n][1];
      }
    }
  }
  // Z12 = U Y (and its transpose), Z22 = -Y^T Y
  warp_gemm<NV, NFM, NFM>([&](int ii, int l) { return sW[ii + l * NV]; }, [&](int l, int j) { return sY[l + j * NFM]; },
                          [&](int ii, int j, double v) {
                            Z[ii + (NV + j) * NVF] = v;
                            Z[(NV + j) + ii * NVF] = v;
                          });
  warp_gemm<NFM, NFM, NFM>([&](int ii, int k) { return -sY[k + ii * NFM]; }, [&](int k, int j) { return sY[k + j * NFM]; },
                           [&](int ii, int j, double v) { Z[(NV + ii) + (NV + j) * NVF] = v; });
  bad = __reduce_or_sync(0xffffffffu, bad);
  if (lane == 0 && bad) atomicOr(&p.info[b], bad);
}

// ------------------------------------------------------------------------------------------------------------------
// K2: everything else of "Forms linear system", with all dense products on the fp64 tensor pipe (DMMA m8n8k4).
//
// Shared-memory plan (35.8 KB -> 6 CTAs per SM).  The parts of the linearization record K2 needs are contiguous
// ([l_D, l_Qxx), [l_Quu, l_Phix) and [l_ha, l_dgdq)), so they land IN PLACE with three cp.async.bulk copies and are then
// used (and modified: PDIPM terms) where they lie; Z (from K1) is a fourth copy; the PDIPM inputs (slack|dual|res,
// dg/dq|dg/df) land in the buffer that later holds R.  The cost Hessian Qxx is NOT staged: it is only the accumulator
// seed of the Qxx product, so it is read from global memory (L2: prefetched at kernel start) straight into the DMMA
// accumulator fragments, plus the PDIPM increments that are kept in shared memory (Qqq block + Qvv diagonal).  Only the contact rows of Qafqv / Qafu are materialised (in the dead dIDCdqv
// buffer): their acceleration rows are diag(Qaa) times rows of R / Z and are formed on the fly in the fragment loads.
template <int NV, int NU, int NFM>
struct CondCfg {
  static constexpr int NX = 2 * NV, NVF = NV + NFM;
  static constexpr int TX = num_tiles(NX), TF = num_tiles(NVF), TV = num_tiles(NV), TU = num_tiles(NU), TM = num_tiles(NFM);
  static constexpr int NWARPS = TX;
  static constexpr int NTHREADS = 32 * NWARPS;
  static constexpr int up2(int x) { return (x + 1) & ~1; }
  // mirror of the record from l_D to l_Phix (same relative offsets as rbt_make_stage_layout)
  static constexpr int i_D = 0, i_IDC = i_D + up2(NVF * NX), i_Qaa = i_IDC + up2(NVF), i_Qff = i_Qaa + up2(NV),
                       i_Qqf = i_Qff + up2(NFM * NFM), IN1A = i_Qqf + up2(NV * NFM);   // [l_D, l_Qxx)
  // mirror of the record from l_Quu to l_Phix
  static constexpr int i_Quu = IN1A, i_lx = i_Quu + up2(NU * NU), i_la = i_lx + up2(NX), i_lf = i_la + up2(NV),
                       i_lu = i_lf + up2(NFM), i_Fx = i_lu + up2(NU), i_lup = i_Fx + up2(NX), i_se3 = i_lup + 6,
                       IN1 = i_se3 + 108, IN1B = IN1 - IN1A;
  // mirror of the record from l_ha to l_dgdq
  static constexpr int j_ha = 0, j_hf = j_ha + up2(NV), j_hx = j_hf + up2(NFM), j_hu = j_hx + up2(NX), j_fx = j_hu + up2(NU),
                       j_sc = j_fx + up2(NX), IN2 = j_sc + 4;
  static constexpr int o_in1 = 0;
  static constexpr int o_Z = o_in1 + IN1;          // Z (ld NVF)
  static constexpr int o_R = o_Z + NVF * NVF;      // R (ld NVF); before R exists: PDIPM staging
  static constexpr int o_in2 = o_R + NVF * NX;
  static constexpr int o_vec = o_in2 + IN2;
  static constexpr int v_r = 0, v_laf = NVF, v_haf = 2 * NVF, v_Fi = 3 * NVF, v_FiS = v_Fi + 36, v_dQq = v_FiS + 36,
                       v_dQv = v_dQq + NV * NV, v_end = v_dQv + up2(NV);  // dQq / dQv: PDIPM increments of Qqq, diag(Qvv)
  static constexpr int o_bar = (o_vec + v_end + 1) & ~1;
  static constexpr int SMEM_DOUBLES = o_bar + 2;
  static constexpr size_t SMEM_BYTES = size_t(SMEM_DOUBLES) * 8;
  static constexpr int QAF = 0, QUF = NFM * NX;    // contact rows of Qafqv (NFM x NX) and Qafu (NFM x NV) inside the dead D buffer
  static_assert(TF < NWARPS && TV <= NWARPS && 2 * TM < NWARPS, "one warp per row band, one warp left for the vectors");
  static_assert(NFM * NX + NFM * NV <= NVF * NX, "Qaf | Quf fit in the dIDCdqv buffer");
  static_assert((NFM * NX) % 2 == 0 && (NFM * NV) % 2 == 0, "Qaf | Quf are adjacent in the expansion record (one bulk store)");
};

#ifndef RBT_COND_MIN_CTAS
#define RBT_COND_MIN_CTAS 6
#endif
template <int NV, int NU, int NFM>
__global__ void __launch_bounds__(CondCfg<NV, NU, NFM>::NTHREADS, RBT_COND_MIN_CTAS) condense_kernel(const StageParams p) {
  using C = CondCfg<NV, NU, NFM>;
  constexpr int NX = C::NX, NVF = C::NVF, NTHR = C::NTHREADS, TX = C::TX, TF = C::TF, TV = C::TV, TU = C::TU, TM = C::TM;
  extern __shared__ __align__(16) double smem[];
  const rbt_layout& K = p.K;
  const rbt_stage_layout& S = p.S;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const size_t o = blockIdx.x;  // b * n_grid + i
  if (o >= size_t(p.batch) * p.n_grid) return;
  const int i = int(o % p.n_grid);
  const rbt_stage_ctrl c = p.ctrl[i];
  const double* lin = p.lin + o * S.l_stride;
  double* con = p.con + o * S.c_stride;
  double* kkt = p.kkt + o * K.k_stride;
  double* ex = p.ex + o * S.e_stride;
  constexpr int np = NV - NU;  // dim_passive = dimv - dimu for every robot robotoc builds (checked at rbt_stage_setup)

  if (c.type == RBT_TERMINAL) {  // terminal_stage.cpp:94-106
    for (int e = tid; e < NX * NX; e += NTHR) kkt[K.k_Qxx + e] = lin[S.l_Qxx + e];
    for (int e = tid; e < NX; e += NTHR) kkt[K.k_lx + e] = lin[S.l_lx + e];
    if (np == 6 && tid == 0) se3_jac_inverse_dev(lin + S.l_se3 + 36, ex + S.e_Fqqpi);
    return;
  }
  const bool impact = (c.type == RBT_IMPACT);
  // inequality rows: box limits + friction cones on Intermediate / Lift stages; on Impact stages only the cones, and only if the
  // table registers ImpactFrictionCone (impact_friction_cone.cpp:190-235 -- the same algebra on the impact forces)
  const bool pdipm = !impact || p.tab.impact_friction_cone != 0;
  const int nf = c.nf, nvf = NV + nf, ns = impact ? 0 : c.ns;
  const double dt = c.dt;
  double* in1 = smem + C::o_in1;
  double* sD = in1 + C::i_D;        // dIDCdqv (ld NVF); dead after R = Z D, then:
  double* sQaf = sD + C::QAF;       //   contact rows of Qafqv (ld NFM)
  double* sQuf = sD + C::QUF;       //   contact rows of Qafu  (ld NFM)
  double* vIDC = in1 + C::i_IDC;
  double* vQaa = in1 + C::i_Qaa;
  double* sQff = in1 + C::i_Qff;
  double* sQqf = in1 + C::i_Qqf;
  const double* gQxx = lin + S.l_Qxx;  // cost Hessian: global memory (accumulator seed only)
  double* gQuu = in1 + C::i_Quu;
  double* vlx = in1 + C::i_lx;
  double* vla = in1 + C::i_la;
  double* vlf = in1 + C::i_lf;
  double* vlu = in1 + C::i_lu;
  double* vFx = in1 + C::i_Fx;
  const double* vlup = in1 + C::i_lup;
  const double* sse3 = in1 + C::i_se3;
  double* sZ = smem + C::o_Z;
  double* sR = smem + C::o_R;
  const double* in2 = smem + C::o_in2;
  const double* vha = in2 + C::j_ha;
  const double* vhf = in2 + C::j_hf;
  const double* vhx = in2 + C::j_hx;
  const double* vhu = in2 + C::j_hu;
  const double* vfx = in2 + C::j_fx;
  const double* vsc = in2 + C::j_sc;
  double* vec = smem + C::o_vec;
  double* vr = vec + C::v_r;
  double* vlaf = vec + C::v_laf;
  double* vhaf = vec + C::v_haf;
  double* Fi = vec + C::v_Fi;
  double* FiS = vec + C::v_FiS;
  double* dQq = vec + C::v_dQq;     // PDIPM increment of Qqq (NV x NV)
  double* dQv = vec + C::v_dQv;     // PDIPM increment of diag(Qvv)
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + C::o_bar);
  // PDIPM staging inside the (not yet written) R buffer
  const int ncp = S.ncp, nbox = p.tab.n_box, ncon = p.tab.n_contacts, nc = S.nc;
  double* cSl = sR;                      // slack | dual | res     (bulk copy)
  double* sDq = sR + 3 * ncp;            // dg/dq (5 x nv per contact) | dg/df (5 x 3 per contact)   (bulk copy)
  double* sDf = sDq + (S.l_dgdf - S.l_dgdq);
  const int gsz = (S.l_dgdf - S.l_dgdq) + ((15 * ncon + 1) & ~1);
  double* cW = sDq + ((gsz + 1) & ~1);   // weights dual/slack
  double* cC = cW + ncp;                 // condensing coefficients

  if (tid == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
    uint32_t bytes = uint32_t(C::IN1 + NVF * NVF + C::IN2) * 8u;
    if (pdipm) bytes += uint32_t(3 * ncp + gsz) * 8u;
    mbar_expect_tx(bar, bytes);
    l2_prefetch_bulk(lin + S.l_Qxx, uint32_t(NX * NX) * 8u);
    tma_load_1d(in1, lin + S.l_D, uint32_t(C::IN1A) * 8u, bar);
    tma_load_1d(in1 + C::IN1A, lin + S.l_Quu, uint32_t(C::IN1B) * 8u, bar);
    tma_load_1d(sZ, ex + S.e_Z, uint32_t(NVF * NVF) * 8u, bar);
    tma_load_1d(smem + C::o_in2, lin + S.l_ha, uint32_t(C::IN2) * 8u, bar);
    if (pdipm) {
      tma_load_1d(cSl, con + S.c_slack, uint32_t(3 * ncp) * 8u, bar);
      tma_load_1d(sDq, lin + S.l_dgdq, uint32_t(gsz) * 8u, bar);
    }
  }
  __syncthreads();
  if (np == 6) {  // the SE(3) inverses are long scalar chains: run them under the bulk copies, straight from global memory
    // two lanes of ONE warp (a lone thread still costs its warp every issue slot of the 370-instruction routine)
    if (tid == 32 || tid == 33)  // Fqq_prev_inv (state_equation.cpp:76) | Fqq_inv (:77-78)
      se3_jac_inverse_dev(lin + S.l_se3 + (tid == 32 ? 36 : 72), tid == 32 ? ex + S.e_Fqqpi : Fi);
  }
  mbar_wait(bar, 0);

  // ---- phase 1: mask what lies beyond the active contact dimension, per-row PDIPM quantities
  if (nf < NFM) {  // (loops over the inactive part only: this kernel is bound by issue slots, not by bytes)
    for (int e = tid; e < NFM * NFM; e += NTHR)
      if ((e % NFM) >= nf || (e / NFM) >= nf) sQff[e] = 0.0;
    for (int e = nf * NV + tid; e < NV * NFM; e += NTHR) sQqf[e] = 0.0;
  }
  if (tid < NVF) {
    if (tid >= nvf) vIDC[tid] = 0.0;
    vhaf[tid] = impact ? 0.0 : (tid < NV ? vha[tid] : (tid - NV < nf ? -vhf[tid - NV] : 0.0));
    if (tid >= NV && tid - NV >= nf) vlf[tid - NV] = 0.0;
  }
  for (int e = tid; e < NV * NV + NV; e += NTHR) dQq[e] = 0.0;  // (dQv follows dQq)
  if (pdipm) {
    const double mu = p.tab.barrier;
    for (int r = tid; r < nc; r += NTHR) {  // pdipm.hxx:27-100
      const bool cone = r >= nbox;
      if (!cone && (impact || __ldg(p.row_level + r) + c.ineq_gate > 2)) {
        // box limits do not act on impact stages, position- / velocity-level limits not on the first two grid points
        // (constraints_data.cpp:20-45): no weight, no gradient, record untouched
        cW[r] = 0.0;
        cC[r] = 0.0;
        continue;
      }
      const bool act = !cone || ((c.contact_mask >> ((r - nbox) / 5)) & 1);
      double w = 0.0, cd = 0.0;
      if (act) {
        const double sl = cSl[r], du = cSl[ncp + r];
        const double cm = sl * du - mu;
        // one reciprocal (MUFU seed + 2 Newton steps) and a residual correction per quotient instead of two IEEE divisions:
        // this loop is 92 threads wide and every warp of the CTA waits for it at the next barrier
        const double rs = fast_rcp(sl), num = du * cSl[2 * ncp + r] - cm;
        cd = num * rs;
        cd = fma(fma(-sl, cd, num), rs, cd);
        w = du * rs;
        w = fma(fma(-sl, w, du), rs, w);
        con[S.c_cmpl + r] = cm;
      }
      con[S.c_cond + r] = cd;  // data.cond.setZero() for inactive contacts   friction_cone.cpp:198
      cW[r] = w;
      cC[r] = cd;
    }
    for (int ci = 0; ci < ncon; ++ci)  // cone Jacobians of inactive contacts -> 0 (they are contraction rows of the products below)
      if (!((c.contact_mask >> ci) & 1))
        for (int e = tid; e < 5 * NV + 15; e += NTHR) {
          if (e < 5 * NV) sDq[ci * 5 * NV + e] = 0.0;
          else sDf[ci * 15 + e - 5 * NV] = 0.0;
        }
  }
  __syncthreads();

  // ---- phase 2: PDIPM condensing applied to the working copies       joint_*_limit.cpp:68-75, friction_cone.cpp:194-235
  // A target (variable, index) gathers its box rows in table order (deterministic; a lower and an upper limit share it).
  if (pdipm) {
    auto gather = [&](int tgt, double& w, double& gs) {
      const int4 e4 = __ldg(p.tgt + tgt);
      const int e[4] = {e4.x, e4.y, e4.z, e4.w};
      w = 0.0; gs = 0.0;
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (e[q] != 0) {
          const int r = (e[q] < 0 ? -e[q] : e[q]) - 1;
          w += cW[r];
          gs += (e[q] < 0) ? -cC[r] : cC[r];
        }
    };
    // Qqq += sum_c dg_dq^T diag(w) dg_dq          friction_cone.cpp:217-218  (box diagonal below)
    // One NV x (5 ncon) x NV product on the tensor pipe: the cone rows of all contacts are the contraction index k = 5 ci + r
    // (rows of inactive contacts were zeroed above).  Warp w < TV owns row band w (A fragment and its weight loaded once per
    // k-step, TV column tiles); the other warps do the Qqf / Qff terms meanwhile.  (Generic operand lambdas per tile would spend
    // far more index arithmetic per DMMA.)
    constexpr int KC = 5 * (NFM / 3);
    static_assert(KC % 4 == 0 && TV < NTHR / 32, "cone rows fill whole k-steps; at least one warp left for Qqf / Qff");
    if (warp < TV) {
      const int r0 = tile_off(warp, NV);
      double acc[TV][2];
#pragma unroll
      for (int n = 0; n < TV; ++n) acc[n][0] = acc[n][1] = 0.0;
#pragma unroll
      for (int ks = 0; ks < KC / 4; ++ks) {
        const int k = 4 * ks + t;
        const bool ok = k < 5 * ncon;
        const double* col = sDq + (k / 5) * 5 * NV + (k % 5);   // element (k, x) of the stacked cone Jacobian at col[5 x]
        const double a = ok ? col[(r0 + g) * 5] * cW[nbox + k] : 0.0;
#pragma unroll
        for (int n = 0; n < TV; ++n) {
          const double bv = ok ? col[(tile_off(n, NV) + g) * 5] : 0.0;
          dmma884(acc[n][0], acc[n][1], a, bv);
        }
      }
#pragma unroll
      for (int n = 0; n < TV; ++n) {
        const int j0 = tile_off(n, NV);
        dQq[(r0 + g) + (j0 + 2 * t) * NV] = acc[n][0];
        dQq[(r0 + g) + (j0 + 2 * t + 1) * NV] = acc[n][1];
      }
      // the cone parts of the gradients ride along here (the band products are short): lq += dg_dq^T cond, lf += dg_df^T cond
      if (warp == 0 && lane < NV) {                                                                          // :207
        double a = 0.0;
        for (int ci = 0; ci < ncon; ++ci)
#pragma unroll
          for (int r = 0; r < 5; ++r) a = fma(sDq[ci * 5 * NV + r + lane * 5], cC[nbox + 5 * ci + r], a);
        vlx[lane] += a;
      } else if (warp == 1 && lane < 3 * ncon) {                                                             // :208-209
        const int ci = lane / 3, j = lane % 3;
        if ((c.contact_mask >> ci) & 1) {
          const int fstack = 3 * __popc(c.contact_mask & ((1 << ci) - 1));
          double a = 0.0;
#pragma unroll
          for (int r = 0; r < 5; ++r) a = fma(sDf[ci * 15 + r + j * 5], cC[nbox + 5 * ci + r], a);
          vlf[fstack + j] += a;
        }
      }
    } else {
      // Qqf[:, stack(c)] += dg_dq^T diag(w) dg_df ;  Qff[stack(c), stack(c)] += dg_df^T diag(w) dg_df     :219-222
      // thread u: one element (ii, j) of the NV x 3 block (u < 3 NV) or of the 3 x 3 block, looped over the active contacts
      constexpr int NE = 3 * NV + 9;
      for (int u = tid - 32 * TV; u < NE; u += NTHR - 32 * TV) {
        const bool isqf = u < 3 * NV;
        const int uu = isqf ? u : u - 3 * NV;
        const int ii = isqf ? uu % NV : uu % 3, j = isqf ? uu / NV : uu / 3;
        for (int ci = 0; ci < ncon; ++ci) {
          if (!((c.contact_mask >> ci) & 1)) continue;
          const int fstack = 3 * __popc(c.contact_mask & ((1 << ci) - 1));
          const double* lhs = isqf ? sDq + ci * 5 * NV + ii * 5 : sDf + ci * 15 + ii * 5;
          const double* df = sDf + ci * 15 + j * 5;
          const double* w5 = cW + nbox + 5 * ci;
          double acc = 0.0;
#pragma unroll
          for (int r = 0; r < 5; ++r) acc = fma(lhs[r] * w5[r], df[r], acc);
          if (isqf) sQqf[ii + (fstack + j) * NV] += acc;
          else sQff[(fstack + ii) + (fstack + j) * NFM] += acc;
        }
      }
    }
    __syncthreads();  // the Qqq diagonal below touches elements the loop above also updates
    // (folding the diagonal weight into the tile epilogue would drop this barrier at the price of a divergent gather in
    //  every tile)
    // gradients and diagonals, one target per thread spread over the warps
    if (warp == 0 && lane < NV) {
      double w, gs;
      gather(lane, w, gs);
      vlx[lane] += gs;
      dQq[lane * (NV + 1)] += w;
    } else if (warp == 1 && lane < NV) {
      double w, gs;
      gather(NV + lane, w, gs);
      vlx[NV + lane] += gs;
      dQv[lane] = w;
    } else if (warp == 2 && lane < NV) {
      double w, gs;
      gather(2 * NV + lane, w, gs);
      vQaa[lane] += w;
      vla[lane] += gs;
    } else if (warp == 3 && lane < NU) {
      double w, gs;
      gather(3 * NV + lane, w, gs);
      gQuu[lane * (NU + 1)] += w;
      vlu[lane] += gs;
    }
    __syncthreads();  // staging (in the R buffer) is dead from here on
  }
  // ---- phase 3: R = Z D (tensor pipe) ; r = Z IDC ; Fqq_inv * dSub/dqf         contact_dynamics.cpp:65-66
  if (warp < TF) {
    const int i0 = tile_off(warp, NVF);
    double acc[TX][2];
#pragma unroll
    for (int n = 0; n < TX; ++n) acc[n][0] = acc[n][1] = 0.0;
    warp_mma_band<NVF, TX, NX>(
        acc, i0, [&](int ii, int k) { return sZ[ii + k * NVF]; }, [&](int k, int j) { return sD[k + j * NVF]; });
#pragma unroll
    for (int n = 0; n < TX; ++n) {
      const int j0 = tile_off(n, NX);
      sR[(i0 + g) + (j0 + 2 * t) * NVF] = acc[n][0];
      sR[(i0 + g) + (j0 + 2 * t + 1) * NVF] = acc[n][1];
    }
  } else {
    matvec_N4(sZ, NVF, NVF, NVF, vIDC, lane, 32, [&](int r, double a) { vr[r] = a; });
    if (np == 6)
      for (int e = lane; e < 36; e += 32) {  // FiS = Fqq_inv * (dSub/dqf top-left)        state_equation.cpp:80
        const int ii = e % 6, j = e / 6;
        double acc = 0.0;
        for (int l = 0; l < 6; ++l) acc = fma(Fi[ii + l * 6], sse3[l + j * 6], acc);
        FiS[e] = acc;
      }
  }
  __syncthreads();  // D is dead from here on

  // ---- phase 4: contact rows of Qafqv and Qafu, laf                       contact_dynamics.cpp:68-86
  if (warp < TM) {  // Qaf = -Qff R_f - [Qqf^T | 0]
    const int a0 = tile_off(warp, NFM);
    double acc[TX][2];
#pragma unroll
    for (int n = 0; n < TX; ++n) {
      const int j0 = tile_off(n, NX);
      acc[n][0] = (j0 + 2 * t < NV) ? -sQqf[(j0 + 2 * t) + (a0 + g) * NV] : 0.0;
      acc[n][1] = (j0 + 2 * t + 1 < NV) ? -sQqf[(j0 + 2 * t + 1) + (a0 + g) * NV] : 0.0;
    }
    warp_mma_band<NFM, TX, NX>(
        acc, a0, [&](int a, int l) { return -sQff[a + l * NFM]; }, [&](int l, int j) { return sR[(NV + l) + j * NVF]; });
#pragma unroll
    for (int n = 0; n < TX; ++n) {
      const int j0 = tile_off(n, NX);
      sQaf[(a0 + g) + (j0 + 2 * t) * NFM] = acc[n][0];
      sQaf[(a0 + g) + (j0 + 2 * t + 1) * NFM] = acc[n][1];
    }
  } else if (!impact && warp < 2 * TM) {  // Quf = Qff Z_fa
    const int a0 = tile_off(warp - TM, NFM);
    double acc[TV][2];
#pragma unroll
    for (int n = 0; n < TV; ++n) acc[n][0] = acc[n][1] = 0.0;
    warp_mma_band<NFM, TV, NV>(
        acc, a0, [&](int a, int l) { return sQff[a + l * NFM]; }, [&](int l, int j) { return sZ[(NV + l) + j * NVF]; });
#pragma unroll
    for (int n = 0; n < TV; ++n) {
      const int j0 = tile_off(n, NV);
      sQuf[(a0 + g) + (j0 + 2 * t) * NFM] = acc[n][0];
      sQuf[(a0 + g) + (j0 + 2 * t + 1) * NFM] = acc[n][1];
    }
  } else if (warp == NTHR / 32 - 1) {  // laf
    for (int r = lane; r < NVF; r += 32) {
      double v;
      if (r < NV) {
        v = vla[r] - vQaa[r] * vr[r];
      } else {
        double acc = 0.0;
        for (int l = 0; l < NFM; ++l) acc = fma(sQff[(r - NV) + l * NFM], vr[NV + l], acc);
        v = (r - NV < nf) ? -vlf[r - NV] - acc : 0.0;
      }
      vlaf[r] = v;
      ex[S.e_laf + r] = v;
      ex[S.e_r + r] = vr[r];
      if (!impact) ex[S.e_haf + r] = (c.sto || c.sto_next) ? vhaf[r] : 0.0;
      if (r < NV) ex[S.e_Qaa + r] = vQaa[r];
    }
  }
  __syncthreads();
  // R and the contact rows [Qaf | Quf] are final and only read from here on: they go to the expansion record as two bulk
  // shared -> global copies that run under the Hessian condensing (no element-wise copy-out loop; the acceleration rows of
  // Qafqv / Qafu are not stored at all -- rbt_stage_layout.h)
  if (tid == 0) {
    tma_store_fence();
    tma_store_1d(ex + S.e_R, sR, uint32_t(NVF * NX) * 8u);
    tma_store_1d(ex + S.e_Qaf, sQaf, uint32_t(NFM * NX + NFM * NV) * 8u);
    tma_store_commit();
  }

  // ---- phase 5: Hessian condensing on the tensor pipe           contact_dynamics.cpp:88-121, impact_dynamics.cpp:64-66
  // Qafqv = [-diag(Qaa) R_a ; Qaf], Qafu = [diag(Qaa) Z_aa ; Quf]: the acceleration rows are formed in the fragment loads.
  const int i0 = tile_off(warp, NX);
  {  // Qxx = Qxx' - R^T Qafqv + [Qqf R_f ; 0]
    double acc[TX][2];
#pragma unroll
    for (int n = 0; n < TX; ++n) {
      const int j0 = tile_off(n, NX);
      const int r = i0 + g;
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int cidx = j0 + 2 * t + q;
        double v = __ldg(gQxx + r + cidx * NX);
        if (r < NV && cidx < NV) v += dQq[r + cidx * NV];
        else if (r == cidx) v += dQv[r - NV];
        acc[n][q] = v;
      }
    }
    warp_mma_band<NV, TX, NX>(
        acc, i0, [&](int ii, int l) { return -sR[l + ii * NVF]; }, [&](int l, int j) { return -vQaa[l] * sR[l + j * NVF]; });
    warp_mma_band<NFM, TX, NX>(
        acc, i0, [&](int ii, int l) { return -sR[(NV + l) + ii * NVF]; }, [&](int l, int j) { return sQaf[l + j * NFM]; });
    warp_mma_band<NFM, TX, NX>(
        acc, i0, [&](int ii, int l) { return ii < NV ? sQqf[ii + l * NV] : 0.0; },
        [&](int l, int j) { return sR[(NV + l) + j * NVF]; });
    double* qxx_out = kkt + K.k_Qxx + (i0 + g) + 2 * t * NX;
#pragma unroll
    for (int n = 0; n < TX; ++n) {
      const int j0 = tile_off(n, NX);
      qxx_out[j0 * NX] = acc[n][0];        // (one base pointer, compile-time offsets: the address arithmetic of a fresh
      qxx_out[(j0 + 1) * NX] = acc[n][1];  //  64-bit address per store was two extra instructions per store)
    }
  }
  if (!impact) {
    {  // [Qxu_passive | Qxu] = -R^T Qafu_full - [Qqf Z_fa ; 0]          (NX x NV)
      double acc[TV][2];
#pragma unroll
      for (int n = 0; n < TV; ++n) acc[n][0] = acc[n][1] = 0.0;
      warp_mma_band<NV, TV, NV>(
          acc, i0, [&](int ii, int l) { return -sR[l + ii * NVF]; }, [&](int l, int j) { return vQaa[l] * sZ[l + j * NVF]; });
      warp_mma_band<NFM, TV, NV>(
          acc, i0, [&](int ii, int l) { return -sR[(NV + l) + ii * NVF]; }, [&](int l, int j) { return sQuf[l + j * NFM]; });
      warp_mma_band<NFM, TV, NV>(
          acc, i0, [&](int ii, int l) { return ii < NV ? -sQqf[ii + l * NV] : 0.0; },
          [&](int l, int j) { return sZ[(NV + l) + j * NVF]; });
      double* qxup_out = ex + S.e_Qxup + (i0 + g);
      double* qxu_out = kkt + K.k_Qxu + (i0 + g);
#pragma unroll
      for (int n = 0; n < TV; ++n) {
        const int j0 = tile_off(n, NV);
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int j = j0 + 2 * t + q;
          // passive columns -> expansion record, actuated columns -> KKT record (pre-condense Qxu is zero: no x-u cost term)
          double* dst = (j < np) ? qxup_out + j * NX : qxu_out + (j - np) * NX;
          *dst = acc[n][q];
        }
      }
    }
    if (warp < TV) {  // [Quu_passive_topRight ; Quu' +=] = Z[0:nv, :] Qafu_full[:, np:]     (NV x NU)
      const int r0 = tile_off(warp, NV);
      double acc[TU][2];
#pragma unroll
      for (int n = 0; n < TU; ++n) {
        const int j0 = tile_off(n, NU);
        const int r = r0 + g;
        acc[n][0] = (r >= np) ? gQuu[(r - np) + (j0 + 2 * t) * NU] : 0.0;
        acc[n][1] = (r >= np) ? gQuu[(r - np) + (j0 + 2 * t + 1) * NU] : 0.0;
      }
      warp_mma_band<NV, TU, NU>(
          acc, r0, [&](int ii, int l) { return sZ[ii + l * NVF]; }, [&](int l, int j) { return vQaa[l] * sZ[l + (np + j) * NVF]; });
      warp_mma_band<NFM, TU, NU>(
          acc, r0, [&](int ii, int l) { return sZ[ii + (NV + l) * NVF]; }, [&](int l, int j) { return sQuf[l + (np + j) * NFM]; });
#pragma unroll
      for (int n = 0; n < TU; ++n) {
        const int j0 = tile_off(n, NU);
        const int r = r0 + g;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          if (r < np) ex[S.e_Quup + r + (j0 + 2 * t + q) * np] = acc[n][q];
          else kkt[K.k_Quu + (r - np) + (j0 + 2 * t + q) * NU] = acc[n][q];
        }
      }
    }
  }
  // ---- gradients: lx -= R^T laf (+ Qqf r_f) ; [lu_passive ; lu] += Z[0:nv,:] laf          :108-128
  matvec_T(sR, NVF, NVF, NX, vlaf, tid, NTHR, [&](int ii, double a) {
    double v = vlx[ii] - a;
    if (ii < NV) {
      double a2 = 0.0;
      for (int l = 0; l < NFM; ++l) a2 = fma(sQqf[ii + l * NV], vr[NV + l], a2);
      v += a2;
    }
    kkt[K.k_lx + ii] = v;
  });
  if (!impact) {
    matvec_N4(sZ, NVF, NV, NVF, vlaf, tid, NTHR, [&](int ii, double a) {
      if (ii < np) ex[S.e_lup + ii] = vlup[ii] + a;
      else kkt[K.k_lu + ii - np] = vlu[ii - np] + a;
    });
  }
  // ---- state equation rows                                 contact_dynamics.cpp:130-135, impact_dynamics.cpp:71-74
  const double sdt = impact ? 1.0 : dt;
  {  // thread = (pair of rows, column phase): 16-byte stores, the rows decide the formula once, no div / mod in the loop
    constexpr int RP = NX / 2, CP = NTHR / RP;  // row pairs ; columns written per pass
    static_assert(NX % 2 == 0 && NV % 2 == 0 && NVF % 2 == 0 && CP >= 1, "row pairs never straddle the q | v boundary");
    if (tid < CP * RP) {
      const int r0 = 2 * (tid % RP), j0 = tid / RP;
      double* Fcol = kkt + K.k_Fxx + r0;
      if (r0 >= NV) {   // Fvq | Fvv = -dt R_a (+ I)
        const double* rrow = sR + (r0 - NV);
#pragma unroll 2
        for (int j = j0; j < NX; j += CP) {
          const double2 rv = *reinterpret_cast<const double2*>(rrow + j * NVF);
          *reinterpret_cast<double2*>(Fcol + j * NX) =
              make_double2(fma(-sdt, rv.x, (j == r0) ? 1.0 : 0.0), fma(-sdt, rv.y, (j == r0 + 1) ? 1.0 : 0.0));
        }
      } else if (np == 6 && r0 < 6) {  // floating base rows: Fqq = -Fqq_inv * (dSub/dqf), Fqv = -dt Fqq_inv   state_equation.cpp:80-81
#pragma unroll 2
        for (int j = j0; j < NX; j += CP) {
          double2 v = make_double2(0.0, 0.0);
          if (j < 6) v = make_double2(-FiS[r0 + j * 6], -FiS[r0 + 1 + j * 6]);
          else if (j >= NV && j < NV + 6 && !impact) v = make_double2(-dt * Fi[r0 + (j - NV) * 6], -dt * Fi[r0 + 1 + (j - NV) * 6]);
          *reinterpret_cast<double2*>(Fcol + j * NX) = v;
        }
      } else {          // Fqq = I, Fqv = dt I
        const double dtv = impact ? 0.0 : dt;
#pragma unroll 2
        for (int j = j0; j < NX; j += CP)
          *reinterpret_cast<double2*>(Fcol + j * NX) = make_double2((j == r0) ? 1.0 : ((j == r0 + NV) ? dtv : 0.0),
                                                                    (j == r0 + 1) ? 1.0 : ((j == r0 + 1 + NV) ? dtv : 0.0));
      }
    }
  }
  if (!impact)
    for (int e = tid; e < NV * NU; e += NTHR) kkt[K.k_Fvu + e] = dt * sZ[(e % NV) + (np + e / NV) * NVF];
  for (int ii = tid; ii < NX; ii += NTHR) {
    auto Fxv = [&](int l) { return l >= NV ? vFx[l] - sdt * vr[l - NV] : vFx[l]; };
    double v = Fxv(ii), f = impact ? 0.0 : vfx[ii];
    if (np == 6 && ii < 6) {  // Fq, fq head <- -Fqq_inv * (.)                                :83-85
      double a1 = 0.0, a2 = 0.0;
      for (int l = 0; l < 6; ++l) {
        a1 = fma(Fi[ii + l * 6], vFx[l], a1);
        a2 = fma(Fi[ii + l * 6], impact ? 0.0 : vfx[l], a2);
      }
      v = -a1;
      f = -a2;
    }
    kkt[K.k_Fx + ii] = v;
    if (!impact) kkt[K.k_fx + ii] = f / c.ngrids_in_phase;
  }
  // ---- switching constraint                                contact_dynamics.cpp:138-153
  if (ns > 0) {
    const double* Phia = lin + S.l_Phia;
#pragma unroll 1
    for (int e = tid; e < ns * NV; e += NTHR) ex[S.e_Phia + e] = Phia[e];
#pragma unroll 1
    for (int e = tid; e < ns * NX; e += NTHR) {
      const int q = e % ns, j = e / ns;
      double acc = 0.0;
#pragma unroll 2
      for (int l = 0; l < NV; ++l) acc = fma(Phia[q + l * ns], sR[l + j * NVF], acc);
      kkt[K.k_Phix + e] = lin[S.l_Phix + e] - acc;
    }
#pragma unroll 1
    for (int e = tid; e < ns * NU; e += NTHR) {
      const int q = e % ns, j = e / ns;
      double acc = 0.0;
#pragma unroll 2
      for (int l = 0; l < NV; ++l) acc = fma(Phia[q + l * ns], sZ[l + (np + j) * NVF], acc);
      kkt[K.k_Phiu + e] = acc;
    }
#pragma unroll 1
    for (int q = tid; q < ns; q += NTHR) {
      double acc = 0.0;
#pragma unroll 2
      for (int l = 0; l < NV; ++l) acc = fma(Phia[q + l * ns], vr[l], acc);
      kkt[K.k_p + q] = lin[S.l_p + q] - acc;
      kkt[K.k_Phit + q] = (lin[S.l_Phit + q] - acc) / c.ngrids_in_phase;  // incl. the STO scaling (intermediate_stage.cpp:146-148)
    }
  }
  // ---- STO sensitivities + scaling                         contact_dynamics.cpp:156-163, intermediate_stage.cpp:140-148
  // Only grid points of a phase whose duration is optimised carry them: the sweeps read hx, hu, h, Qtt and haf under the
  // same condition (riccati_backward.cuh: `if (sto)`, update_kernel: dts != 0), so the other grid points skip the work.
  if (!impact && (c.sto || c.sto_next)) {
    const double g1 = 1.0 / c.ngrids_in_phase;
    matvec_T(sR, NVF, NVF, NX, vhaf, tid, NTHR, [&](int ii, double a) {
      double v = vhx[ii] - a;
      if (ii < NV) {
        double a2 = 0.0;
        for (int l = 0; l < NFM; ++l) a2 = fma(sQqf[ii + l * NV], vr[NV + l], a2);
        v += a2 / dt;
      }
      kkt[K.k_hx + ii] = v * g1;
    });
    for (int ii = tid; ii < NU; ii += NTHR) {
      double acc = 0.0;
      for (int l = 0; l < NVF; ++l) acc = fma(sZ[(np + ii) + l * NVF], vhaf[l], acc);
      kkt[K.k_hu + ii] = (vhu[ii] + acc) * g1;
    }
    if (tid == NTHR - 1) {
      double h = vsc[0];
      for (int l = 0; l < NVF; ++l) h = fma(-vr[l], vhaf[l], h);
      const double Qtt = vsc[1] * g1 * g1;
      kkt[K.k_sc + 0] = Qtt;
      kkt[K.k_sc + 1] = -Qtt;
      kkt[K.k_sc + 2] = h * g1;
      kkt[K.k_sc + 3] = 0.0;
    }
  }
  if (tid == 0) tma_store_wait_read();  // the bulk stores of R | Qaf | Quf must have read shared memory before the CTA retires
}

// ------------------------------------------------------------------------------------------------------------------
// Host wire records -> linearization records (rbt_stage_layout.h: packed upper triangles of M, Qff, Qxx, Quu; Qqf and, on
// schedules without switching-time stages, the STO section do not travel and are zero-filled).  HBM streaming: one CTA per
// stage, coalesced reads of the 24 KB wire record, coalesced writes of the dense sections; the symmetric blocks are gathered
// from the packed triangle.  Only used by the PCIe-facing rbt_iteration_host_wire / _resident paths.
struct WireParams {
  const rbt_wire_layout* W;  // [n_grid] per-grid-point layouts (device memory)
  int n_grid, l_stride;
  long long ocp_stride;      // doubles of one OCP's concatenated wire records
  const double* wire;
  double* lin;
  // resident-state path: compact PDIPM residuals [record][ncp] -> the c_res section of the PDIPM records (res == nullptr: none)
  const double* res;
  double* con;
  int c_stride, c_res, ncp;
};

__global__ void __launch_bounds__(128) unpack_wire_kernel(const WireParams p) {
  const int i = int(blockIdx.x % p.n_grid);
  const size_t b = blockIdx.x / p.n_grid;
  const rbt_wire_layout& W = p.W[i];
  const double* wire = p.wire + b * size_t(p.ocp_stride) + W.ocp_off;
  double* lin = p.lin + size_t(blockIdx.x) * p.l_stride;
  const int nseg = W.nseg;
  for (int k = 0; k < W.nzero; ++k)
    for (int e = threadIdx.x; e < W.zero[k].n; e += 128) lin[W.zero[k].lin_off + e] = 0.0;
  __syncthreads();  // the diagonal / packed segments land inside zero-filled blocks
  for (int k = 0; k < nseg; ++k) {
    const rbt_wire_seg g = W.seg[k];
    const double* src = wire + g.wire_off;
    double* dst = lin + g.lin_off;
    if (!g.sym) {
      if (g.ld == g.rows) {
        for (int e = threadIdx.x; e < g.rows * g.cols; e += 128) dst[e] = src[e];
      } else {
        for (int e = threadIdx.x; e < g.rows * g.cols; e += 128) dst[(e % g.rows) + (e / g.rows) * g.ld] = src[e];
      }
    } else if (g.sym == 2) {
      for (int e = threadIdx.x; e < g.rows; e += 128) dst[e * (g.ld + 1)] = src[e];
    } else {
      for (int e = threadIdx.x; e < g.rows * g.rows; e += 128) {
        const int r = e % g.rows, c = e / g.rows;
        dst[r + c * g.ld] = (r <= c) ? src[c * (c + 1) / 2 + r] : src[r * (r + 1) / 2 + c];
      }
    }
  }
  if (p.res) {
    const double* r = p.res + size_t(blockIdx.x) * p.ncp;
    double* c = p.con + size_t(blockIdx.x) * p.c_stride + p.c_res;
    for (int e = threadIdx.x; e < p.ncp; e += 128) c[e] = r[e];
  }
}

// slack | dual of the PDIPM records (adjacent: the first 2 ncp doubles) -> compact [record][2 ncp] for one contiguous download
__global__ void __launch_bounds__(64) pack_slack_dual_kernel(const double* con, int c_stride, int c_slack, int n2, double* out) {
  const double* c = con + size_t(blockIdx.x) * c_stride + c_slack;
  double* o = out + size_t(blockIdx.x) * n2;
  for (int e = threadIdx.x; e < n2; e += 64) o[e] = c[e];
}

// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_min(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ void atomic_min_pos(double* addr, double v) {  // v > 0: IEEE order == unsigned integer order
  atomicMin(reinterpret_cast<unsigned long long*>(addr), static_cast<unsigned long long>(__double_as_longlong(v)));
}

// expand / update: one CTA of 4 warps per (OCP, stage).  The matrices of the expansion record arrive in shared memory by
// TMA bulk copies (one round trip to HBM instead of a chain of dependent column loads); each warp then owns every 4th
// column of a mat-vec (lane = row, conflict-free) and the partial sums meet in shared memory.
constexpr int XTHR = 128;

#ifndef RBT_EXP_MIN_CTAS
#define RBT_EXP_MIN_CTAS 10  // (48 registers, no spills; shared memory allows 10)
#endif
template <int NV, int NU, int NFM>
__global__ void __launch_bounds__(XTHR, RBT_EXP_MIN_CTAS) expand_kernel(const StageParams p) {
  constexpr int NX = 2 * NV, NVF = NV + NFM, NTHR = XTHR;
  constexpr int RSZ = ((NVF * NX + 1) & ~1) + ((NVF + 1) & ~1);  // R | r (adjacent in the record)
  constexpr int ZSZ = NVF * NU;
  __shared__ __align__(16) double sR[RSZ];
  __shared__ __align__(16) double sZ[ZSZ];
  __shared__ __align__(16) double sG[512];  // dgdq | dgdf of all contacts
  __shared__ __align__(16) double sC[4 * 160];  // slack | dual | res | cmpl
  __shared__ double sdx[NX], sdu[NU], sdaf[NVF], spart[4][32], smin[8];
  __shared__ __align__(8) uint64_t bar;
  const rbt_layout& K = p.K;
  const rbt_stage_layout& S = p.S;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const size_t o = blockIdx.x;
  const int i = int(o % p.n_grid), b = int(o / p.n_grid);
  const rbt_stage_ctrl c = p.ctrl[i];
  if (c.type == RBT_TERMINAL) return;  // step sizes 1.0 (terminal_stage.cpp:127-136)
  const bool impact = (c.type == RBT_IMPACT);
  const bool pdipm = !impact || p.tab.impact_friction_cone != 0;  // impact stages: cone rows only (impact_friction_cone.cpp:238-268)
  constexpr int np = NV - NU;
  const int nf = c.nf, nvf = NV + nf;
  const double* lin = p.lin + o * S.l_stride;
  const double* ex = p.ex + o * S.e_stride;
  const double* d = p.dir + o * K.d_stride;
  double* con = p.con + o * S.c_stride;
  double* xd = p.xd + o * S.x_stride;
  const int gsz = S.l_stride - S.l_dgdq;  // dgdq | dgdf | padding: the tail of the linearization record (<= 512 doubles)
  if (tid == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
    uint32_t bytes = RSZ * 8;
    if (!impact) bytes += ZSZ * 8;
    if (pdipm) bytes += gsz * 8 + 4 * S.ncp * 8;
    mbar_expect_tx(&bar, bytes);
    tma_load_1d(sR, ex + S.e_R, RSZ * 8, &bar);
    if (!impact) tma_load_1d(sZ, ex + S.e_Z + np * NVF, ZSZ * 8, &bar);
    if (pdipm) {
      tma_load_1d(sG, lin + S.l_dgdq, gsz * 8, &bar);
      tma_load_1d(sC, con + S.c_slack, 4 * S.ncp * 8, &bar);
    }
  }
  for (int e = tid; e < NX; e += NTHR) sdx[e] = d[K.d_dx + e];
  for (int e = tid; e < NU; e += NTHR) sdu[e] = impact ? 0.0 : d[K.d_du + e];
  const int nbox = p.tab.n_box, ncp = S.ncp;
  __syncthreads();
  mbar_wait(&bar, 0);
  {  // daf = -R dx + Z[:, np:np+nu] du - r ; df *= -1      contact_dynamics.cpp:167-174
    double acc = 0.0;
    if (lane < nvf) {
      for (int k = wid; k < NX; k += 4) acc = fma(-sR[lane + k * NVF], sdx[k], acc);
      if (!impact)
        for (int k = wid; k < NU; k += 4) acc = fma(sZ[lane + k * NVF], sdu[k], acc);
    }
    spart[wid][lane] = acc;
  }
  __syncthreads();
  if (tid < nvf) {
    double acc = (spart[0][tid] + spart[1][tid]) + (spart[2][tid] + spart[3][tid]);
    acc -= sR[((NVF * NX + 1) & ~1) + tid];
    if (tid >= NV) acc = -acc;
    sdaf[tid] = acc;
    xd[S.x_daf + tid] = acc;
  }
  if (!pdipm) return;
  __syncthreads();
  const double tau = p.tab.fraction_to_boundary;
  double mp = 1.0, md = 1.0;
  for (int r = tid; r < S.nc; r += NTHR) {
    if (r < nbox && (impact || __ldg(p.row_level + r) + c.ineq_gate > 2)) continue;  // row does not act here: record untouched
    const double c_sl = sC[r], c_du = sC[ncp + r], c_res = sC[2 * ncp + r], c_cm = sC[3 * ncp + r];
    double dsl, ddu;
    if (r < nbox) {
      const rbt_box_row br = p.tab.box[r];
      const double var = br.var == RBT_VAR_Q ? sdx[br.idx] : br.var == RBT_VAR_V ? sdx[NV + br.idx]
                         : br.var == RBT_VAR_A ? sdaf[br.idx] : sdu[br.idx];
      dsl = -br.sign * var - c_res;                                 // joint_*_limit.cpp:78-82
      ddu = -(c_du * dsl + c_cm) / c_sl;                            // pdipm.hxx:159-164
    } else {
      const int q = r - nbox, ci = q / 5, r5 = q % 5;
      dsl = 1.0; ddu = 1.0;                                         // friction_cone.cpp:244-245
      if ((c.contact_mask >> ci) & 1) {
        const int fstack = 3 * __popc(c.contact_mask & ((1 << ci) - 1));
        const double* dgdq = sG + size_t(ci) * 5 * NV;
        const double* dgdf = sG + (S.l_dgdf - S.l_dgdq) + size_t(ci) * 15;
        double a0 = 0.0, a1 = 0.0;
        for (int j = 0; j < NV; j += 2) {
          a0 = fma(dgdq[r5 + j * 5], sdx[j], a0);
          if (j + 1 < NV) a1 = fma(dgdq[r5 + (j + 1) * 5], sdx[j + 1], a1);
        }
        double acc = a0 + a1;
        for (int j = 0; j < 3; ++j) acc = fma(dgdf[r5 + j * 5], sdaf[NV + fstack + j], acc);
        dsl = -acc - c_res;                                         // :253-256
        ddu = -(c_du * dsl + c_cm) / c_sl;
      }
    }
    con[S.c_dslack + r] = dsl;
    con[S.c_ddual + r] = ddu;
    const double fp = -tau * (c_sl / dsl), fd = -tau * (c_du / ddu);  // pdipm.hxx:121-142
    if (fp > 0.0 && fp < 1.0) mp = fmin(mp, fp);
    if (fd > 0.0 && fd < 1.0) md = fmin(md, fd);
  }
  mp = warp_min(mp);
  md = warp_min(md);
  if (lane == 0) {
    smin[wid * 2] = mp;
    smin[wid * 2 + 1] = md;
  }
  __syncthreads();
  if (tid == 0) {  // min over the stage, then over the horizon    direct_multiple_shooting.cpp:202-209
    atomic_min_pos(&p.steps[2 * b], fmin(fmin(smin[0], smin[2]), fmin(smin[4], smin[6])));
    atomic_min_pos(&p.steps[2 * b + 1], fmin(fmin(smin[1], smin[3]), fmin(smin[5], smin[7])));
  }
}

// free-flyer part of Robot::integrateConfiguration (textbook SE(3) exponential; see oracle/condense_oracle.c)
__device__ __forceinline__ void integrate_free_flyer_dev(double* q, const double* dq, double step) {
  const double vx = step * dq[0], vy = step * dq[1], vz = step * dq[2];
  const double wx = step * dq[3], wy = step * dq[4], wz = step * dq[5];
  const double th2 = wx * wx + wy * wy + wz * wz, th = sqrt(th2);
  double bb, cc, s2 = 0.0, c2 = 1.0;  // one sincos of the half angle serves both the translation and the quaternion part
  if (th < 1e-6) {
    bb = 0.5 - th2 / 24.0; cc = 1.0 / 6.0 - th2 / 120.0;
  } else {
    sincos(0.5 * th, &s2, &c2);
    bb = 2.0 * s2 * s2 / th2; cc = (th - 2.0 * s2 * c2) / (th2 * th);
  }
  const double cx = wy * vz - wz * vy, cy = wz * vx - wx * vz, cz = wx * vy - wy * vx;
  const double ccx = wy * cz - wz * cy, ccy = wz * cx - wx * cz, ccz = wx * cy - wy * cx;
  const double tx = vx + bb * cx + cc * ccx, ty = vy + bb * cy + cc * ccy, tz = vz + bb * cz + cc * ccz;
  const double qx = q[3], qy = q[4], qz = q[5], qw = q[6];
  const double ux = qy * tz - qz * ty, uy = qz * tx - qx * tz, uz = qx * ty - qy * tx;
  const double u2x = qy * uz - qz * uy, u2y = qz * ux - qx * uz, u2z = qx * uy - qy * ux;
  q[0] += tx + 2.0 * (qw * ux + u2x);
  q[1] += ty + 2.0 * (qw * uy + u2y);
  q[2] += tz + 2.0 * (qw * uz + u2z);
  double sh, ch;
  if (th < 1e-6) { sh = 0.5 - th2 / 48.0; ch = 1.0 - th2 / 8.0; } else { sh = s2 / th; ch = c2; }
  const double ex_ = sh * wx, ey = sh * wy, ez = sh * wz, ew = ch;
  const double nx_ = qw * ex_ + qx * ew + qy * ez - qz * ey;
  const double ny = qw * ey - qx * ez + qy * ew + qz * ex_;
  const double nz = qw * ez + qx * ey - qy * ex_ + qz * ew;
  const double nw = qw * ew - qx * ex_ - qy * ey - qz * ez;
  const double nrm = 1.0 / sqrt(nx_ * nx_ + ny * ny + nz * nz + nw * nw);
  q[3] = nx_ * nrm; q[4] = ny * nrm; q[5] = nz * nrm; q[6] = nw * nrm;
}

#ifndef RBT_UPD_MIN_CTAS
#define RBT_UPD_MIN_CTAS 12  // latency-bound streaming kernel: many resident CTAs (12/SM at 40 registers) hide its load latency
#endif
template <int NV, int NU, int NFM>
__global__ void __launch_bounds__(XTHR, RBT_UPD_MIN_CTAS) update_kernel(const StageParams p) {
  constexpr int NX = 2 * NV, NVF = NV + NFM, NTHR = XTHR;
  constexpr int QSZ = NFM * NX + NFM * NV + ((NV + 1) & ~1);  // contact rows Qaf | Quf and diag(Qaa) (adjacent in the record)
  constexpr int ZSZ = (NVF * NVF + 1) & ~1;
  constexpr int PSZ = ((NX * 6 + 1) & ~1) + ((6 * NU + 1) & ~1) + 6;     // Qxup | Quup | lup (floating base: np = 6)
  __shared__ __align__(16) double sQ[QSZ];
  __shared__ __align__(16) double sZ[ZSZ];
  __shared__ __align__(16) double sP[PSZ];
  __shared__ double sdx[NX], sdu[NU], slaf[NVF], sdl[NX], sdgn[NV], spart[4][32];
  __shared__ __align__(8) uint64_t bar;
  const rbt_layout& K = p.K;
  const rbt_stage_layout& S = p.S;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const size_t o = blockIdx.x;
  const int i = int(o % p.n_grid), b = int(o / p.n_grid);
  const rbt_stage_ctrl c = p.ctrl[i];
  const bool terminal = (c.type == RBT_TERMINAL), impact = (c.type == RBT_IMPACT);
  constexpr int np = NV - NU;
  const int nf = terminal ? 0 : c.nf, nvf = NV + nf, ns = (terminal || impact) ? 0 : c.ns;
  double* ex = p.ex + o * S.e_stride;
  double* d = p.dir + o * K.d_stride;
  double* xd = p.xd + o * S.x_stride;
  double* con = p.con + o * S.c_stride;
  double* sol = p.sol + o * S.s_stride;
  const bool nup = !terminal && !impact && np == 6;
  if (tid == 0 && !terminal) {
    mbar_init(&bar, 1);
    fence_mbar_init();
    mbar_expect_tx(&bar, (QSZ + ZSZ + (nup ? PSZ : 0)) * 8);
    tma_load_1d(sQ, ex + S.e_Qaf, QSZ * 8, &bar);
    tma_load_1d(sZ, ex + S.e_Z, ZSZ * 8, &bar);
    if (nup) tma_load_1d(sP, ex + S.e_Qxup, PSZ * 8, &bar);
  }
  const double ap = p.steps[2 * b], ad = p.steps[2 * b + 1];
  for (int e = tid; e < NX; e += NTHR) {
    sdx[e] = d[K.d_dx + e];
    sdl[e] = d[K.d_dlmdgmm + e];
  }
  for (int e = tid; e < NU; e += NTHR) sdu[e] = (terminal || impact) ? 0.0 : d[K.d_du + e];
  if (!terminal)
    for (int e = tid; e < NV; e += NTHR) sdgn[e] = d[K.d_stride + K.d_dlmdgmm + NV + e];  // dgmm of stage i+1 (not modified here)
  if (!terminal && (!impact || p.tab.impact_friction_cone != 0)) {
    for (int r = tid + (impact ? p.tab.n_box : 0); r < S.nc; r += NTHR) {  // updateSlack / updateDual    constraint_component_base.hxx:25-36
      if (r < p.tab.n_box && __ldg(p.row_level + r) + c.ineq_gate > 2) continue;  // level not valid on this grid point
      con[S.c_slack + r] += ap * con[S.c_dslack + r];
      con[S.c_dual + r] += ad * con[S.c_ddual + r];
    }
  }
  __syncthreads();
  // ---- everything of SplitSolution::integrate (split_solution.cpp:58-90) that does not depend on the dual expansion runs
  //      while the bulk copies are in flight
  if (np == 6) {
    if (tid == 2 * 32) integrate_free_flyer_dev(sol + S.s_q, sdx, ap);
    if (tid < 6) {  // correctCostateDirection     state_equation.cpp:90-95
      double acc = 0.0;
      for (int l = 0; l < 6; ++l) acc = fma(ex[S.e_Fqqpi + l + tid * 6], sdl[l], acc);
      d[K.d_dlmdgmm + tid] = -acc;
      sol[S.s_lmd + tid] += ap * (-acc);
    }
  }
  for (int e = tid; e < NV; e += NTHR) {
    if (np == 6) {
      if (e >= 6) {
        sol[S.s_q + e + 1] += ap * sdx[e];
        sol[S.s_lmd + e] += ap * sdl[e];
      }
    } else {
      sol[S.s_q + e] += ap * sdx[e];
      sol[S.s_lmd + e] += ap * sdl[e];
    }
    sol[S.s_v + e] += ap * sdx[NV + e];
    sol[S.s_gmm + e] += ap * sdl[NV + e];
    if (!terminal) {
      const double da = xd[S.x_daf + e];
      if (!impact) {
        sol[S.s_a + e] += ap * da;
        sol[S.s_dv + e] = 0.0;
      } else {
        sol[S.s_a + e] = 0.0;
        sol[S.s_dv + e] += ap * da;
      }
    }
  }
  if (terminal) return;
  for (int e = tid; e < NU; e += NTHR) sol[S.s_u + e] = impact ? 0.0 : sol[S.s_u + e] + ap * sdu[e];
  for (int e = tid; e < nf; e += NTHR) sol[S.s_f + e] += ap * xd[S.x_daf + NV + e];
  for (int e = tid; e < ns; e += NTHR) sol[S.s_xi + e] += ap * d[K.d_dxi + e];
  const double dt = c.dt;
  double dts = 0.0;
  if (!impact && c.ngrids_in_phase > 0) dts = (d[K.d_dts + 1] - d[K.d_dts]) / c.ngrids_in_phase;  // intermediate_stage.cpp:167-170
  // old values of the entries this thread will update after the mat-vecs: fetched now, under the bulk copies (a load issued
  // after the barriers would sit on every warp's critical path)
  const double bm_old = (tid < nvf) ? (tid < NV ? sol[S.s_beta + tid] : sol[S.s_mu + tid - NV]) : 0.0;
  const double nup_old = (nup && wid == 3 && (lane >> 2) < 6 && (lane & 3) == 0) ? sol[S.s_nup + (lane >> 2)] : 0.0;
  double extra = 0.0;  // the per-row terms of laf that do not come from the staged matrices
  if (tid < nvf) {
    extra = ex[S.e_laf + tid];
    if (!impact) {
      if (tid < NV) {
        extra = fma(dt, sdgn[tid], extra);
        for (int q = 0; q < ns; ++q) extra = fma(ex[S.e_Phia + q + tid * ns], d[K.d_dxi + q], extra);
      }
      if (dts < -2.220446049250313e-16 || dts > 2.220446049250313e-16) extra = fma(dts, ex[S.e_haf + tid], extra);
    } else if (tid < NV) {
      extra += sdgn[tid];                                                          // impact_dynamics.cpp:94
    }
  }
  // acceleration rows of Qafqv dx + Qafu du: Qafqv_a = -diag(Qaa) R_a, Qafu_a = diag(Qaa) Z_aa, and da = -R_a dx + Z_a,u du - r_a
  // (expand_kernel; ddv on an impact stage), so they are Qaa o (da + r_a) -- no matrix needed
  const double da_r = (tid < NV) ? xd[S.x_daf + tid] + ex[S.e_r + tid] : 0.0;
  mbar_wait(&bar, 0);
  if (tid < NV) extra = fma(sQ[NFM * NX + NFM * NV + tid], da_r, extra);
  {  // laf += Qafqv dx + Qafu du (+ dt dgmm+ / Phia^T dxi / dts haf)   contact_dynamics.cpp:191-201: contact rows
    double acc = 0.0;
    if (lane >= NV && lane < nvf) {
      const double* q = sQ + (lane - NV);
      for (int k = wid; k < NX; k += 4) acc = fma(q[k * NFM], sdx[k], acc);
      if (!impact) {
        const double* qu = q + NFM * NX + np * NFM;
        for (int k = wid; k < NU; k += 4) acc = fma(qu[k * NFM], sdu[k], acc);
      }
    }
    spart[wid][lane] = acc;
  }
  if (nup && wid == 3) {  // dnu_passive: 4 lanes per row      contact_dynamics.cpp:182-190
    const int prow = lane >> 2, ppart = lane & 3;
    const double* sQxup = sP;
    const double* sQuup = sP + ((NX * 6 + 1) & ~1);
    const double* slup = sQuup + ((6 * NU + 1) & ~1);
    double pn = 0.0;
    if (prow < 6) {
      for (int k = ppart; k < NU; k += 4) pn = fma(-sQuup[prow + k * 6], sdu[k], pn);
      for (int k = ppart; k < NX; k += 4) pn = fma(-sQxup[k + prow * NX], sdx[k], pn);
      for (int k = ppart; k < NV; k += 4) pn = fma(-dt * sZ[prow + k * NVF], sdgn[k], pn);
    }
    pn += __shfl_xor_sync(0xffffffffu, pn, 1);
    pn += __shfl_xor_sync(0xffffffffu, pn, 2);
    if (prow < 6 && ppart == 0) {
      pn -= slup[prow];
      xd[S.x_dnup + prow] = pn;
      sol[S.s_nup + prow] = nup_old + ap * pn;
    }
  }
  __syncthreads();
  if (tid < nvf) {
    const double acc = extra + ((spart[0][tid] + spart[1][tid]) + (spart[2][tid] + spart[3][tid]));
    slaf[tid] = acc;
    ex[S.e_laf + tid] = acc;
  }
  __syncthreads();
  {  // dbetamu = -Z laf     :202
    double acc = 0.0;
    if (lane < nvf)
      for (int k = wid; k < nvf; k += 4) acc = fma(-sZ[lane + k * NVF], slaf[k], acc);
    spart[wid][lane] = acc;
  }
  __syncthreads();
  if (tid < nvf) {
    const double acc = (spart[0][tid] + spart[1][tid]) + (spart[2][tid] + spart[3][tid]);
    xd[S.x_dbetamu + tid] = acc;
    if (tid < NV) sol[S.s_beta + tid] = bm_old + ap * acc;
    else sol[S.s_mu + tid - NV] = bm_old + ap * acc;
  }
}

}  // namespace rbt

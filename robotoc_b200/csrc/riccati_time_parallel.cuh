// riccati_time_parallel.cuh -- time-parallel (segmented) Riccati sweeps for batches far smaller than the SM count.
//
// Without switching-time optimisation the backward sweep carries only (P, s) from grid i+1 to grid i and the forward sweep
// only dx (riccati_recursion.cpp:32-131 with every sto flag false).  Split the horizon into S contiguous segments
// [lo_j, hi_j), lo_j = floor(j N / S).  Then:
//   backward  1. tp_element_kernel: every grid point's conditional value-function element (A, b, C, eta, J) of
//                Saerkkae & Garcia-Fernandez, "Temporal parallelization of dynamic programming and linear quadratic control",
//                IEEE TAC 68(2), 2023, in robotoc's convention V(dx) = 1/2 dx^T P dx - s^T dx (a value function is an element
//                with A = b = C = 0, J = P, eta = s);
//             2. tp_combine_kernel: each segment's elements reduced to one aggregate (pairwise tree, one launch per level),
//                then a suffix scan over [aggregate_0 .. aggregate_{S-1}, terminal] (Hillis-Steele, one launch per level):
//                entry j+1 of the scan is the value function (P, s) at grid hi_j;
//             3. riccati_backward_kernel<..., SEG = true>: CTA (ocp, j) seeds P, s from the scan and sweeps [lo_j, hi_j) with
//                the serial kernel's per-stage algebra.
//   forward   4. tp_fwd_compose_kernel: the closed-loop maps dx+ = T dx + t (T = Fxx + B K, t = B k + Fx; impact: Fxx, Fx)
//                of every segment but the last, composed;
//             5. tp_fwd_boundary_kernel: the composites applied serially from dx0 give dx at every segment start;
//             6. riccati_forward_kernel<..., SEG = true>: CTA (ocp, j) sweeps its segment from that dx.
// An element needs Cholesky(Quu) (and Cholesky(W) on a switching-constraint stage), which the serial sweep does not: if one
// fails, the OCP's flag in `fail` is set and CTA (ocp, 0) of the segment kernels sweeps that OCP's whole horizon serially.
#pragma once
#include "rbt_device.cuh"
#include "riccati_backward.cuh"
#include "../../include/rbt_layout.h"

namespace rbt {

struct TpParams {
  rbt_layout L;
  const rbt_stage_ctrl* ctrl;
  int n_grid;
  int batch;
  int segs;              // S
  const double* kkt;     // [batch][n_grid][k_stride]
  const double* ric;     // [batch][n_grid][r_stride]
  double* elem;          // [batch][n_grid][TpElem::SIZE]
  const double* scan_in;  // [batch][S + 1][TpElem::SIZE]
  double* scan_out;
  double* fmap;          // [batch][S][NX * NX + NX]: composed closed-loop map of segment j
  double* dxseed;        // [batch][S][NX]: dx at the start of segment j (j >= 1)
  const double* dx0;     // [batch][NX]
  int* fail;             // [batch]
  int d;                 // combine stride of this level
  int pairs;             // reduce level: jobs per segment
  int gather;            // first scan level: read the segment aggregates and the terminal element from `elem`
};

// ---------------------------------------------------------------------------------------------------------- elements
template <int NV, int NU, int NS>
struct TpElemCfg {
  static constexpr int NX = 2 * NV, NT = 256;
  static constexpr int o_R = 0, o_dinv = o_R + NU * NU, o_Ri = o_dinv + NU, o_X = o_Ri + NU * NU, o_x = o_X + NU * NX,
                       o_Y = o_x + NU, o_W = o_Y + NU * NS, o_dinvW = o_W + NS * NS, o_D = o_dinvW + NS, o_e = o_D + NS * NX,
                       o_Z = o_e + NS, o_ze = o_Z + NS * NX, o_V = o_ze + NS, o_T = o_V + NS * NU, o_eta = o_T + NX * NX,
                       o_Rt = o_eta + NX, o_FR = o_Rt + NU * NU, o_end = o_FR + NV * NU;
};

// grid = batch x n_grid, one CTA per grid point.  Plain FMA loops: every grid point of every OCP runs concurrently, and the
// products are nx^2 nu (not nx^3).
template <int NV, int NU, int NS>
__global__ void __launch_bounds__(TpElemCfg<NV, NU, NS>::NT) tp_element_kernel(const TpParams p) {
  using C = TpElemCfg<NV, NU, NS>;
  using E = TpElem<2 * NV>;
  constexpr int NX = C::NX, NT = C::NT;
  __shared__ __align__(16) double sm[C::o_end];
  const int b = blockIdx.x / p.n_grid, i = blockIdx.x % p.n_grid;
  if (b >= p.batch) return;
  const int N = p.n_grid - 1, tid = threadIdx.x;
  const rbt_layout& L = p.L;
  const double* rec = p.kkt + (size_t(b) * p.n_grid + i) * L.k_stride;
  double* el = p.elem + (size_t(b) * p.n_grid + i) * E::SIZE;
  const rbt_stage_ctrl cs = p.ctrl[i];
  const double* Qxx = rec + L.k_Qxx;
  if (i == N || cs.type == RBT_IMPACT) {  // V_i = Qxx/2 - lx + V_{i+1}(Fxx dx + Fx);  terminal: A = b = 0
    const bool term = (i == N);
    for (int e = tid; e < NX * NX; e += NT) {
      el[E::A + e] = term ? 0.0 : rec[L.k_Fxx + e];
      el[E::C + e] = 0.0;
      el[E::J + e] = Qxx[e];
    }
    for (int r = tid; r < NX; r += NT) {
      el[E::b + r] = term ? 0.0 : rec[L.k_Fx + r];
      el[E::eta + r] = -rec[L.k_lx + r];
    }
    return;
  }
  const int ns = cs.ns;
  double *sR = sm + C::o_R, *dinv = sm + C::o_dinv, *sRi = sm + C::o_Ri, *sX = sm + C::o_X, *sx = sm + C::o_x;
  double *sY = sm + C::o_Y, *sW = sm + C::o_W, *dinvW = sm + C::o_dinvW, *sD = sm + C::o_D, *se = sm + C::o_e;
  double *sZ = sm + C::o_Z, *sze = sm + C::o_ze, *sV = sm + C::o_V, *sT = sm + C::o_T, *seta = sm + C::o_eta;
  double *sRt = sm + C::o_Rt, *sFR = sm + C::o_FR;
  const double* Qxu = rec + L.k_Qxu;  // S (nx x nu)
  const double* Fvu = rec + L.k_Fvu;  // nv x nu
  const double* lu = rec + L.k_lu;
  const double* Phx = rec + L.k_Phix;  // ns x nx (ld ns)
  const double* Phu = rec + L.k_Phiu;  // ns x nu (ld ns)
  const double* pp = rec + L.k_p;
  bool bad = false;
  for (int e = tid; e < NU * NU; e += NT) sR[e] = rec[L.k_Quu + e];
  __syncthreads();
  if (tid < 32 && !warp_cholesky<NU>(sR, NU, dinv)) bad = true;  // R = Quu = L L^T
  __syncthreads();
  if (tid < NU) {  // R^-1, column tid
    for (int k = 0; k < NU; ++k) sRi[k + tid * NU] = (k == tid) ? 1.0 : 0.0;
    chol_solve_smem(sR, dinv, NU, sRi + tid * NU, 1);
  }
  __syncthreads();
  for (int e = tid; e < NU * NX; e += NT) {  // X = R^-1 S^T
    const int u = e % NU, c = e / NU;
    double a = 0.0;
    for (int v = 0; v < NU; ++v) a = fma(sRi[u + v * NU], Qxu[c + v * NX], a);
    sX[e] = a;
  }
  if (tid < NU) {  // x = R^-1 lu
    double a = 0.0;
    for (int v = 0; v < NU; ++v) a = fma(sRi[tid + v * NU], lu[v], a);
    sx[tid] = a;
  }
  __syncthreads();
  if (ns > 0) {
    // W = Phu R^-1 Phu^T,  D = Phx - Phu X,  e = p - Phu x;  Z = W^-1 D,  ze = W^-1 e,  V = W^-1 Y^T  (Y = R^-1 Phu^T)
    for (int e = tid; e < NU * ns; e += NT) {
      const int u = e % NU, r = e / NU;
      double a = 0.0;
      for (int v = 0; v < NU; ++v) a = fma(sRi[u + v * NU], Phu[r + v * ns], a);
      sY[e] = a;
    }
    for (int e = tid; e < ns * NX; e += NT) {
      const int r = e % ns, c = e / ns;
      double a = Phx[e];
      for (int u = 0; u < NU; ++u) a = fma(-Phu[r + u * ns], sX[u + c * NU], a);
      sD[e] = a;
      sZ[e] = a;
    }
    if (tid < ns) {
      double a = pp[tid];
      for (int u = 0; u < NU; ++u) a = fma(-Phu[tid + u * ns], sx[u], a);
      se[tid] = a;
      sze[tid] = a;
    }
    __syncthreads();
    for (int e = tid; e < ns * ns; e += NT) {
      const int r = e % ns, q = e / ns;
      double a = 0.0;
      for (int u = 0; u < NU; ++u) a = fma(Phu[r + u * ns], sY[u + q * NU], a);
      sW[e] = a;
    }
    for (int e = tid; e < ns * NU; e += NT) sV[e] = sY[(e / ns) + (e % ns) * NU];  // Y^T (ns x nu, ld ns)
    __syncthreads();
    if (tid < 32 && !warp_cholesky<NS>(sW, ns, dinvW)) bad = true;
    __syncthreads();
    for (int c = tid; c < NX + 1 + NU; c += NT) {
      if (c < NX) chol_solve_smem(sW, dinvW, ns, sZ + c * ns, 1);
      else if (c == NX) chol_solve_smem(sW, dinvW, ns, sze, 1);
      else chol_solve_smem(sW, dinvW, ns, sV + (c - NX - 1) * ns, 1);
    }
    __syncthreads();
  }
  // T = S X - D^T Z  (J = Qxx - sym(T));  eta = -(lx - S x + D^T ze)
  for (int e = tid; e < NX * NX; e += NT) {
    const int r = e % NX, c = e / NX;
    double a = 0.0;
    for (int u = 0; u < NU; ++u) a = fma(Qxu[r + u * NX], sX[u + c * NU], a);
    for (int q = 0; q < ns; ++q) a = fma(-sD[q + r * ns], sZ[q + c * ns], a);
    sT[e] = a;
  }
  for (int r = tid; r < NX; r += NT) {
    double a = rec[L.k_lx + r];
    for (int u = 0; u < NU; ++u) a = fma(-Qxu[r + u * NX], sx[u], a);
    for (int q = 0; q < ns; ++q) a = fma(sD[q + r * ns], sze[q], a);
    seta[r] = -a;
  }
  __syncthreads();
  // the constrained feedback: X += Y Z, x += Y ze;  projected inverse Rt = R^-1 - Y W^-1 Y^T  (riccati_factorizer.cpp:58-77)
  for (int e = tid; e < NU * NX; e += NT) {
    const int u = e % NU, c = e / NU;
    double a = sX[e];
    for (int q = 0; q < ns; ++q) a = fma(sY[u + q * NU], sZ[q + c * ns], a);
    sX[e] = a;
  }
  for (int e = tid; e < NU * NU; e += NT) {
    const int u = e % NU, v = e / NU;
    double a = sRi[e];
    for (int q = 0; q < ns; ++q) a = fma(-sY[u + q * NU], sV[q + v * ns], a);
    sRt[e] = a;
  }
  __syncthreads();
  if (tid < NU) {
    double a = sx[tid];
    for (int q = 0; q < ns; ++q) a = fma(sY[tid + q * NU], sze[q], a);
    sx[tid] = a;
  }
  for (int e = tid; e < NV * NU; e += NT) {  // FR = Fvu Rt
    const int r = e % NV, u = e / NV;
    double a = 0.0;
    for (int v = 0; v < NU; ++v) a = fma(Fvu[r + v * NV], 0.5 * (sRt[v + u * NU] + sRt[u + v * NU]), a);
    sFR[e] = a;
  }
  __syncthreads();
  // A = Fxx - B X,  b = Fx - B x,  C = B Rt B^T,  J = Qxx - sym(T)      (B = [0; Fvu])
  for (int e = tid; e < NX * NX; e += NT) {
    const int r = e % NX, c = e / NX;
    double a = rec[L.k_Fxx + e], cc = 0.0;
    if (r >= NV) {
      for (int u = 0; u < NU; ++u) a = fma(-Fvu[(r - NV) + u * NV], sX[u + c * NU], a);
      if (c >= NV)
        for (int u = 0; u < NU; ++u) cc = fma(sFR[(r - NV) + u * NV], Fvu[(c - NV) + u * NV], cc);
    }
    el[E::A + e] = a;
    el[E::C + e] = cc;
    el[E::J + e] = Qxx[e] - 0.5 * (sT[e] + sT[c + r * NX]);
  }
  for (int r = tid; r < NX; r += NT) {
    double a = rec[L.k_Fx + r];
    if (r >= NV)
      for (int u = 0; u < NU; ++u) a = fma(-Fvu[(r - NV) + u * NV], sx[u], a);
    el[E::b + r] = a;
    el[E::eta + r] = seta[r];
  }
  if (tid < 32) {
    bad = __any_sync(0xffffffffu, bad);
    if (bad && tid == 0) atomicExch(&p.fail[b], 1);
  }
}

// --------------------------------------------------------------------------------------------------------- combine
// 3 groups of TX warps; each group computes one NX x NX product at a time on the fp64 tensor pipe (GEMM warp w of a group
// owns the 8-row band w; the last band is pulled back, as in the backward sweep).
template <int NX>
struct TpCombCfg {
  static constexpr int TX = num_tiles(NX);
  static constexpr int NGRP = 3, NT = NGRP * TX * 32;
  static constexpr int MM = NX * NX, LDA = 2 * NX;
  static constexpr int o_Ai = 0, o_Ci = o_Ai + MM, o_Jj = o_Ci + MM, o_Aj = o_Jj + MM, o_Mi = o_Aj + MM,
                       o_R = o_Mi + MM,  // 4 MM: the two Gauss-Jordan buffers [M | I] (NX x 2NX), later T1 | T2 | U | W2
                       o_bi = o_R + 4 * MM, o_etaj = o_bi + NX, o_v = o_etaj + NX, o_w = o_v + NX, o_r = o_w + NX,
                       o_ew = o_r + NX, o_piv = o_ew + NX, o_end = o_piv + NX;
  static constexpr size_t SMEM_BYTES = size_t(o_end) * 8;
  static_assert(2 * NX * LDA <= 4 * MM, "Gauss-Jordan buffers fit the product region");
};

// One band of an NX x NX x NX product by GEMM warp gw (0..TX-1) of a group: epi(r, c, value) for every element it owns.
template <int NX, class FA, class FB, class Epi>
__device__ __forceinline__ void tp_gemm_band(int gw, FA fa, FB fb, Epi epi) {
  constexpr int TX = num_tiles(NX);
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int i0 = tile_off(gw, NX);
  double acc[TX][2];
#pragma unroll
  for (int n = 0; n < TX; ++n) acc[n][0] = acc[n][1] = 0.0;
  warp_mma_band<NX, TX, NX, true>(acc, i0, fa, fb);
  const bool mine = !(NX % 8 != 0 && gw == TX - 1 && i0 + g < 8 * (TX - 1));
  if (mine) {
#pragma unroll
    for (int n = 0; n < TX; ++n) {
      const int j0 = tile_off(n, NX);
      epi(i0 + g, j0 + 2 * t, acc[n][0]);
      epi(i0 + g, j0 + 2 * t + 1, acc[n][1]);
    }
  }
}

// out = (element i) followed by (element j):
//   A = A_j M^-1 A_i,  b = A_j M^-1 (b_i + C_i eta_j) + b_j,  C = A_j M^-1 C_i A_j^T + C_j,   M = I + C_i J_j
//   eta = A_i^T M^-T (eta_j - J_j b_i) + eta_i,  J = A_i^T M^-T J_j A_i + J_i                 (M^T = I + J_j C_i)
// M^-1 by Gauss-Jordan with partial pivoting (M is not symmetric); with T1 = M^-1 A_i the J and eta updates are T1^T (...).
// `out` may alias `ei` (in-place reduction): every block of ei is read into shared memory, or read by the thread that then
// overwrites the same word, before it is written.
template <int NX>
__device__ __forceinline__ void tp_combine(const double* ei, const double* ej, double* out, double* sm) {
  using C = TpCombCfg<NX>;
  using E = TpElem<NX>;
  constexpr int MM = C::MM, LDA = C::LDA, NT = C::NT, TX = C::TX;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int grp = warp / TX, gw = warp % TX, gtid = tid % (TX * 32);
  constexpr int GT = TX * 32;
  double *sAi = sm + C::o_Ai, *sCi = sm + C::o_Ci, *sJj = sm + C::o_Jj, *sAj = sm + C::o_Aj, *sMi = sm + C::o_Mi;
  double *sR = sm + C::o_R, *sbi = sm + C::o_bi, *setaj = sm + C::o_etaj, *sv = sm + C::o_v, *sw = sm + C::o_w;
  double *sr = sm + C::o_r, *sew = sm + C::o_ew;
  int* piv = reinterpret_cast<int*>(sm + C::o_piv);
  for (int e = tid; e < MM / 2; e += NT) {
    reinterpret_cast<double2*>(sAi)[e] = reinterpret_cast<const double2*>(ei + E::A)[e];
    reinterpret_cast<double2*>(sCi)[e] = reinterpret_cast<const double2*>(ei + E::C)[e];
    reinterpret_cast<double2*>(sJj)[e] = reinterpret_cast<const double2*>(ej + E::J)[e];
    reinterpret_cast<double2*>(sAj)[e] = reinterpret_cast<const double2*>(ej + E::A)[e];
  }
  for (int r = tid; r < NX; r += NT) {
    sbi[r] = ei[E::b + r];
    setaj[r] = ej[E::eta + r];
  }
  __syncthreads();
  double* aug0 = sR;
  double* aug1 = sR + NX * LDA;
  // ---- [M | I] with M = I + C_i J_j ;  v = C_i eta_j,  w = J_j b_i
  if (grp == 0) {
    tp_gemm_band<NX>(gw, [&](int r, int k) { return sCi[r + k * NX]; }, [&](int k, int c) { return sJj[k + c * NX]; },
                     [&](int r, int c, double v) { aug0[r * LDA + c] = v + (r == c ? 1.0 : 0.0); });
  } else if (grp == 1) {
    for (int e = gtid; e < MM; e += GT) aug0[(e / NX) * LDA + NX + (e % NX)] = ((e / NX) == (e % NX)) ? 1.0 : 0.0;
  } else {
    matvec_N4(sCi, NX, NX, NX, setaj, gtid, GT, [&](int r, double a) { sv[r] = a; });
    matvec_N4(sJj, NX, NX, NX, sbi, gtid, GT, [&](int r, double a) { sw[r] = a; });
  }
  __syncthreads();
  // ---- Gauss-Jordan on [M | I], partial pivoting without row swaps: pivot row p_k is the unused row with the largest
  // |entry| in column k (every warp finds it redundantly with shuffles, so a step costs one barrier); ping-pong buffers.
  // At the end row p_k holds row k of M^-1 in its right half.
  unsigned long long used = 0ull;
  for (int k = 0; k < NX; ++k) {
    const double* src = (k & 1) ? aug1 : aug0;
    double* dst = (k & 1) ? aug0 : aug1;
    double bv = -1.0;
    int bi = NX;
    for (int r = lane; r < NX; r += 32) {
      const double v = ((used >> r) & 1ull) ? -1.0 : fabs(src[r * LDA + k]);
      if (v > bv) {
        bv = v;
        bi = r;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) {
        bv = ov;
        bi = oi;
      }
    }
    const int pr = bi;
    used |= 1ull << pr;
    if (tid == 0) piv[k] = pr;
    const double inv = 1.0 / src[pr * LDA + k];
    for (int e = tid; e < NX * LDA; e += NT) {
      const int r = e / LDA, c = e - r * LDA;
      const double pv = src[pr * LDA + c] * inv;
      dst[e] = (r == pr) ? pv : fma(-src[r * LDA + k], pv, src[e]);
    }
    __syncthreads();
  }
  const double* fin = (NX & 1) ? aug1 : aug0;
  for (int e = tid; e < MM; e += NT) {
    const int k = e % NX, c = e / NX;
    sMi[e] = fin[piv[k] * LDA + NX + c];  // M^-1 col-major
  }
  __syncthreads();
  double *sT1 = sR, *sT2 = sR + MM, *sU = sR + 2 * MM, *sW2 = sR + 3 * MM;
  // ---- T1 = M^-1 A_i,  T2 = M^-1 C_i,  U = J_j A_i ;  r = M^-1 (b_i + v),  ew = eta_j - w
  if (grp == 0) {
    tp_gemm_band<NX>(gw, [&](int r, int k) { return sMi[r + k * NX]; }, [&](int k, int c) { return sAi[k + c * NX]; },
                     [&](int r, int c, double v) { sT1[r + c * NX] = v; });
  } else if (grp == 1) {
    tp_gemm_band<NX>(gw, [&](int r, int k) { return sMi[r + k * NX]; }, [&](int k, int c) { return sCi[k + c * NX]; },
                     [&](int r, int c, double v) { sT2[r + c * NX] = v; });
  } else {
    tp_gemm_band<NX>(gw, [&](int r, int k) { return sJj[r + k * NX]; }, [&](int k, int c) { return sAi[k + c * NX]; },
                     [&](int r, int c, double v) { sU[r + c * NX] = v; });
    for (int r = gtid; r < NX; r += GT) {
      sew[r] = setaj[r] - sw[r];
      sv[r] += sbi[r];
    }
    __syncwarp();
    named_bar_sync(1, GT);
    matvec_N4(sMi, NX, NX, NX, sv, gtid, GT, [&](int r, double a) { sr[r] = a; });
  }
  __syncthreads();
  // ---- A = A_j T1 (-> out),  W2 = A_j T2,  X = T1^T U (-> the dead A_i buffer)
  double* sX = sAi;
  if (grp == 0) {
    tp_gemm_band<NX>(gw, [&](int r, int k) { return sAj[r + k * NX]; }, [&](int k, int c) { return sT1[k + c * NX]; },
                     [&](int r, int c, double v) { out[E::A + r + c * NX] = v; });
  } else if (grp == 1) {
    tp_gemm_band<NX>(gw, [&](int r, int k) { return sAj[r + k * NX]; }, [&](int k, int c) { return sT2[k + c * NX]; },
                     [&](int r, int c, double v) { sW2[r + c * NX] = v; });
  } else {
    tp_gemm_band<NX>(gw, [&](int r, int k) { return sT1[k + r * NX]; }, [&](int k, int c) { return sU[k + c * NX]; },
                     [&](int r, int c, double v) { sX[r + c * NX] = v; });
  }
  __syncthreads();
  // ---- C = W2 A_j^T (-> T2's buffer, symmetrised below) ;  b = A_j r + b_j ;  eta = T1^T ew + eta_i
  double* sCo = sT2;
  if (grp == 0) {
    tp_gemm_band<NX>(gw, [&](int r, int k) { return sW2[r + k * NX]; }, [&](int k, int c) { return sAj[c + k * NX]; },
                     [&](int r, int c, double v) { sCo[r + c * NX] = v; });
  } else if (grp == 1) {
    matvec_N4(sAj, NX, NX, NX, sr, gtid, GT, [&](int r, double a) { out[E::b + r] = a + ej[E::b + r]; });
  } else {
    matvec_T(sT1, NX, NX, NX, sew, gtid, GT, [&](int c, double a) { out[E::eta + c] = a + ei[E::eta + c]; });
  }
  __syncthreads();
  for (int e = tid; e < MM; e += NT) {
    const int r = e % NX, c = e / NX;
    out[E::J + e] = 0.5 * (sX[e] + sX[c + r * NX]) + ei[E::J + e];
    out[E::C + e] = 0.5 * (sCo[e] + sCo[c + r * NX]) + ej[E::C + e];
  }
}

// mode 0 (p.gather < 0): one level of the in-segment tree reduction, job (ocp, segment j, m): element k = lo_j + 2 d m absorbs
//   element k + d (in place) if k + d < hi_j.  After ceil(log2(max segment length)) levels, element lo_j is the aggregate.
// mode 1: one level of the suffix scan over q = 0..S (q < S: aggregate of segment q, q = S: terminal), job (ocp, q):
//   out[q] = in[q] followed by in[q + d] (or a copy of in[q]).
template <int NX>
__global__ void __launch_bounds__(TpCombCfg<NX>::NT) tp_combine_kernel(const TpParams p) {
  using E = TpElem<NX>;
  extern __shared__ __align__(16) double sm[];
  const int N = p.n_grid - 1, S = p.segs;
  if (p.gather < 0) {
    const int per = S * p.pairs;
    const int b = blockIdx.x / per, j = (blockIdx.x % per) / p.pairs, m = blockIdx.x % p.pairs;
    if (b >= p.batch || p.fail[b]) return;
    const int k = tp_seg_lo(j, N, S) + 2 * p.d * m;
    if (k + p.d >= tp_seg_lo(j + 1, N, S)) return;
    double* eb = p.elem + size_t(b) * p.n_grid * E::SIZE;
    tp_combine<NX>(eb + size_t(k) * E::SIZE, eb + size_t(k + p.d) * E::SIZE, eb + size_t(k) * E::SIZE, sm);
    return;
  }
  const int b = blockIdx.x / (S + 1), q = blockIdx.x % (S + 1);
  if (b >= p.batch || p.fail[b]) return;
  auto src = [&](int qq) {
    return p.gather ? p.elem + (size_t(b) * p.n_grid + (qq < S ? tp_seg_lo(qq, N, S) : N)) * E::SIZE
                    : p.scan_in + (size_t(b) * (S + 1) + qq) * E::SIZE;
  };
  double* dst = p.scan_out + (size_t(b) * (S + 1) + q) * E::SIZE;
  if (q + p.d <= S) {
    tp_combine<NX>(src(q), src(q + p.d), dst, sm);
  } else {
    const double2* s2 = reinterpret_cast<const double2*>(src(q));
    for (int e = threadIdx.x; e < E::SIZE / 2; e += blockDim.x) reinterpret_cast<double2*>(dst)[e] = s2[e];
  }
}

// --------------------------------------------------------------------------------------------------------- forward
template <int NV, int NU>
struct TpFwdCfg {
  static constexpr int NX = 2 * NV, TX = num_tiles(NX), NT = 32 * TX;
  static constexpr int o_T = 0, o_Phi = o_T + NX * NX, o_Phi2 = o_Phi + NX * NX, o_t = o_Phi2 + NX * NX, o_phi = o_t + NX,
                       o_phi2 = o_phi + NX, o_end = o_phi2 + NX;
  static constexpr size_t SMEM_BYTES = size_t(o_end) * 8;
};

// grid = batch x (S - 1): CTA (ocp, j) composes the closed-loop maps of segment j: Phi = T_{hi-1} ... T_lo, phi likewise.
template <int NV, int NU>
__global__ void __launch_bounds__(TpFwdCfg<NV, NU>::NT) tp_fwd_compose_kernel(const TpParams p) {
  using C = TpFwdCfg<NV, NU>;
  constexpr int NX = C::NX, NT = C::NT;
  extern __shared__ __align__(16) double sm[];
  const int S = p.segs, N = p.n_grid - 1;
  const int b = blockIdx.x / (S - 1), j = blockIdx.x % (S - 1);
  if (b >= p.batch || p.fail[b]) return;
  const rbt_layout& L = p.L;
  const int tid = threadIdx.x, warp = tid >> 5;
  const int lo = tp_seg_lo(j, N, S), hi = tp_seg_lo(j + 1, N, S);
  double *sT = sm + C::o_T, *st = sm + C::o_t;
  double* Phi[2] = {sm + C::o_Phi, sm + C::o_Phi2};
  double* phi[2] = {sm + C::o_phi, sm + C::o_phi2};
  int cur = 0;
  for (int i = lo; i < hi; ++i) {
    const double* rec = p.kkt + (size_t(b) * p.n_grid + i) * L.k_stride;
    const double* ric = p.ric + (size_t(b) * p.n_grid + i) * L.r_stride;
    const bool impact = p.ctrl[i].type == RBT_IMPACT;
    const double* Fvu = rec + L.k_Fvu;
    double* dT = (i == lo) ? Phi[0] : sT;
    double* dt = (i == lo) ? phi[0] : st;
    for (int e = tid; e < NX * NX; e += NT) {  // T = Fxx + [0; Fvu] K   (K^T is stored col-major nx x nu)
      const int r = e % NX, c = e / NX;
      double a = rec[L.k_Fxx + e];
      if (!impact && r >= NV)
        for (int u = 0; u < NU; ++u) a = fma(Fvu[(r - NV) + u * NV], ric[L.r_K + c + u * NX], a);
      dT[e] = a;
    }
    for (int r = tid; r < NX; r += NT) {  // t = Fx + [0; Fvu] k
      double a = rec[L.k_Fx + r];
      if (!impact && r >= NV)
        for (int u = 0; u < NU; ++u) a = fma(Fvu[(r - NV) + u * NV], ric[L.r_k + u], a);
      dt[r] = a;
    }
    __syncthreads();
    if (i > lo) {
      const double* P0 = Phi[cur];
      double* P1 = Phi[cur ^ 1];
      tp_gemm_band<NX>(warp, [&](int r, int k) { return sT[r + k * NX]; }, [&](int k, int c) { return P0[k + c * NX]; },
                       [&](int r, int c, double v) { P1[r + c * NX] = v; });
      matvec_N4(sT, NX, NX, NX, phi[cur], tid, NT, [&](int r, double a) { phi[cur ^ 1][r] = a + st[r]; });
      cur ^= 1;
      __syncthreads();
    }
  }
  double* out = p.fmap + (size_t(b) * S + j) * (NX * NX + NX);
  for (int e = tid; e < NX * NX; e += NT) out[e] = Phi[cur][e];
  for (int r = tid; r < NX; r += NT) out[NX * NX + r] = phi[cur][r];
}

// grid = batch, one warp pair per OCP: dx at segment j + 1 = Phi_j dx_j + phi_j, serially over j from dx0.
template <int NX>
__global__ void __launch_bounds__(64) tp_fwd_boundary_kernel(const TpParams p) {
  __shared__ double sdx[2][NX];
  const int b = blockIdx.x, tid = threadIdx.x, S = p.segs;
  if (b >= p.batch || p.fail[b]) return;
  for (int r = tid; r < NX; r += 64) sdx[0][r] = p.dx0[size_t(b) * NX + r];
  __syncthreads();
  int cur = 0;
  for (int j = 0; j + 1 < S; ++j) {
    const double* m = p.fmap + (size_t(b) * S + j) * (NX * NX + NX);
    for (int r = tid; r < NX; r += 64) {
      double a = m[NX * NX + r];
      for (int k = 0; k < NX; ++k) a = fma(m[r + k * NX], sdx[cur][k], a);
      sdx[cur ^ 1][r] = a;
      p.dxseed[(size_t(b) * S + j + 1) * NX + r] = a;
    }
    cur ^= 1;
    __syncthreads();
  }
}

}  // namespace rbt

// ustage_kernels.cuh -- stage layer of the UNCONSTRAINED path (fixed base, no contacts; iiwa14: nv = 7).
//
//   ucondense_kernel   tail of UnconstrIntermediateStage::evalKKT           src/unconstr/unconstr_intermediate_stage.cpp:96-98
//                        Constraints::condenseSlackAndDual (joint limits)    pdipm.hxx:27-100, joint_*_limit.cpp:68-83
//                        UnconstrDynamics::condenseUnconstrDynamics          src/dynamics/unconstr_dynamics.cpp:67-87
//                      UnconstrTerminalStage::evalKKT (copy of Qxx, lx)      src/unconstr/unconstr_terminal_stage.cpp:69-94
//   uexpand_kernel     UnconstrDirectMultipleShooting::computeStepSizes      src/unconstr/unconstr_direct_multiple_shooting.cpp:128-146
//                        expandPrimal / expandDual                           unconstr_dynamics.cpp:90-104
//                        expandSlackAndDual, fraction to boundary            joint_*_limit.cpp:78-83, pdipm.hxx:121-164
//   uupdate_kernel     UnconstrDirectMultipleShooting::integrateSolution     unconstr_direct_multiple_shooting.cpp:159-179
//
// The blocks are 7x7: a whole stage is ~5 kFLOP against ~7 KB of records, i.e. HBM-bound streaming work.  One warp owns
// one (OCP, stage) pair; the linearization record is pulled into shared memory with coalesced loads, everything is done
// in place there, and the KKT / expansion records leave with coalesced stores.  No tensor cores: nothing here reaches
// an 8x8x4 DMMA tile without padding 7 -> 8, and the kernel is bound by the record traffic anyway.
//
// Joint limits act from the grid point the reference gives them: UnconstrOCPSolver sets GridInfo::stage = i, and
// ConstraintsData::setTimeStage (src/constraints/constraints_data.cpp:20-45) turns the position level off on stages 0 and 1
// and the velocity level off on stage 0.  A row of level urow_level(var) acts on grid point i iff i >= that level; a row
// that does not act adds nothing to the KKT / expansion records, takes no part in the step sizes, and its PDIPM record is
// left untouched.
#pragma once
#include "rbt_device.cuh"
#include "stage_kernels.cuh"  // warp_min, atomic_min_pos
#include "../../include/rbt_ustage_layout.h"

namespace rbt {

struct UStageParams {
  rbt_ulayout K;
  rbt_ustage_layout S;
  rbt_constraint_table tab;
  int N, batch;
  double dt;
  const double* lin;
  double* con;
  double* kkt;
  double* ex;
  const double* dir;
  double* xd;
  double* sol;
  double* steps;
};

__device__ __forceinline__ int urow_level(int var) { return var == RBT_VAR_Q ? 2 : var == RBT_VAR_V ? 1 : 0; }

template <int NV>
struct UStageCfg {
  static constexpr int NX = 2 * NV;
  static constexpr int up2(int x) { return (x + 1) & ~1; }
  static constexpr int LSTRIDE = ((3 * up2(NV * NV) + up2(NV) + up2(NX * NX) + 2 * up2(NV * NV) + up2(NX) + 2 * up2(NV) + up2(NX)) + 15) & ~15;
  static constexpr int QXU = up2(NX * NV), VEC = up2(NV);
  static constexpr int XTRA = QXU + 2 * VEC;  // Qxu, w, luc
  static constexpr int WARPS = 4;
  static constexpr int PER_WARP = LSTRIDE + XTRA;
};

template <int NV>
__global__ void __launch_bounds__(32 * UStageCfg<NV>::WARPS) ucondense_kernel(const UStageParams p) {
  using C = UStageCfg<NV>;
  constexpr int NX = C::NX;
  __shared__ __align__(16) double smem[C::WARPS * C::PER_WARP];
  const rbt_ulayout& K = p.K;
  const rbt_ustage_layout& S = p.S;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const size_t o = size_t(blockIdx.x) * C::WARPS + wid;
  const size_t total = size_t(p.batch) * (p.N + 1);
  if (o >= total) return;
  const int i = int(o % (p.N + 1));
  const bool terminal = (i == p.N);
  double* s = smem + wid * C::PER_WARP;
  double* sQxu = s + C::LSTRIDE;
  double* w = sQxu + C::QXU;
  double* luc = w + C::VEC;
  const double* lin = p.lin + o * S.l_stride;
  double* kkt = p.kkt + o * K.k_stride;
  double* ex = p.ex + o * S.e_stride;
  double* con = p.con + o * S.c_stride;
  if (terminal) {  // Qxx, lx only; the rest of the records is zero (as the oracle leaves it)
    for (int e = lane; e < K.k_stride; e += 32) {
      double v = 0.0;
      if (e >= K.k_Qxx && e < K.k_Qxx + NX * NX) v = lin[S.l_Qxx + e - K.k_Qxx];
      else if (e >= K.k_lx && e < K.k_lx + NX) v = lin[S.l_lx + e - K.k_lx];
      kkt[e] = v;
    }
    for (int e = lane; e < S.e_stride; e += 32) ex[e] = 0.0;
    return;
  }
  {  // coalesced 16-byte loads of the whole linearization record
    const double2* src = reinterpret_cast<const double2*>(lin);
    double2* dst = reinterpret_cast<double2*>(s);
    for (int e = lane; e < S.l_stride / 2; e += 32) dst[e] = src[e];
  }
  __syncwarp();
  double* Qxx = s + S.l_Qxx;
  double* Qaa = s + S.l_Qaa;
  double* Quu = s + S.l_Quu;
  double* lx = s + S.l_lx;
  double* la = s + S.l_la;
  double* lu = s + S.l_lu;
  const double* Dq = s + S.l_dIDdq;
  const double* Dv = s + S.l_dIDdv;
  const double* Da = s + S.l_dIDda;
  const double* ID = s + S.l_ID;
  // ---- PDIPM rows: cmpl, cond per row (parallel), then one lane per target variable gathers its rows in table order
  const int nbox = p.tab.n_box;
  for (int r = lane; r < nbox; r += 32) {
    if (i < urow_level(p.tab.box[r].var)) continue;
    const double sl = con[S.c_slack + r], du = con[S.c_dual + r], rs = con[S.c_res + r];
    const double cm = sl * du - p.tab.barrier;
    con[S.c_cmpl + r] = cm;
    con[S.c_cond + r] = (du * rs - cm) / sl;
  }
  __syncwarp();
  if (lane < 4 * NV && i >= urow_level(lane / NV)) {
    const int var = lane / NV, idx = lane % NV;
    double dacc = 0.0, gacc = 0.0;
    double* dptr = var == RBT_VAR_Q ? &Qxx[idx + idx * NX] : var == RBT_VAR_V ? &Qxx[(NV + idx) * (NX + 1)]
                 : var == RBT_VAR_A ? &Qaa[idx * (NV + 1)] : &Quu[idx * (NV + 1)];
    double* gptr = var == RBT_VAR_Q ? &lx[idx] : var == RBT_VAR_V ? &lx[NV + idx] : var == RBT_VAR_A ? &la[idx] : &lu[idx];
    dacc = *dptr;
    gacc = *gptr;
    for (int r = 0; r < nbox; ++r) {
      const rbt_box_row br = p.tab.box[r];
      if (br.var == var && br.idx == idx) {
        dacc += con[S.c_dual + r] / con[S.c_slack + r];
        gacc += br.sign * con[S.c_cond + r];
      }
    }
    *dptr = dacc;
    *gptr = gacc;
  }
  __syncwarp();
  // expansion record: lu, Quu as they stand after the constraints
  for (int e = lane; e < S.e_stride; e += 32) {
    double v = 0.0;
    if (e >= S.e_lu && e < S.e_lu + NV) v = lu[e - S.e_lu];
    else if (e >= S.e_Quu && e < S.e_Quu + NV * NV) v = Quu[e - S.e_Quu];
    ex[e] = v;
  }
  // ---- condenseUnconstrDynamics
  if (lane < NV) {
    w[lane] = Quu[lane * (NV + 1)];
    luc[lane] = lu[lane] + w[lane] * ID[lane];
  }
  __syncwarp();
  if (lane < 3 * NV) {  // lq, lv, la += dID_d*^T lu_condensed
    const int which = lane / NV, j = lane % NV;
    const double* D = which == 0 ? Dq : which == 1 ? Dv : Da;
    double acc = 0.0;
#pragma unroll
    for (int l = 0; l < NV; ++l) acc += D[l + j * NV] * luc[l];
    double* g = which == 0 ? &lx[j] : which == 1 ? &lx[NV + j] : &la[j];
    *g += acc;
  }
  // six NV x NV products A^T diag(w) B
  for (int e = lane; e < 6 * NV * NV; e += 32) {
    const int prod = e / (NV * NV), ij = e % (NV * NV), ii = ij % NV, jj = ij / NV;
    const double* A = (prod == 0 || prod == 1 || prod == 4) ? Dq : (prod == 2 || prod == 5) ? Dv : Da;
    const double* B = (prod == 0) ? Dq : (prod == 1 || prod == 2) ? Dv : Da;
    double acc = 0.0;
#pragma unroll
    for (int l = 0; l < NV; ++l) acc += A[l + ii * NV] * w[l] * B[l + jj * NV];
    switch (prod) {
      case 0: Qxx[ii + jj * NX] += acc; break;                 // Qqq
      case 1: Qxx[ii + (NV + jj) * NX] += acc; break;          // Qqv
      case 2: Qxx[NV + ii + (NV + jj) * NX] += acc; break;     // Qvv
      case 3: Qaa[ii + jj * NV] += acc; break;                 // Qaa
      case 4: sQxu[ii + jj * NX] = acc; break;                 // Qqu() (really Qqa)
      default: sQxu[NV + ii + jj * NX] = acc; break;           // Qvu()
    }
  }
  __syncwarp();
  for (int e = lane; e < NV * NV; e += 32) {  // Qvq = Qqv^T
    const int ii = e % NV, jj = e / NV;
    Qxx[NV + ii + jj * NX] = Qxx[jj + (NV + ii) * NX];
  }
  __syncwarp();
  for (int e = lane; e < K.k_stride; e += 32) {
    double v = 0.0;
    if (e < K.k_Qxu) { if (e < NX * NX) v = Qxx[e]; }
    else if (e < K.k_Qaa) { if (e - K.k_Qxu < NX * NV) v = sQxu[e - K.k_Qxu]; }
    else if (e < K.k_Fx) { if (e - K.k_Qaa < NV * NV) v = Qaa[e - K.k_Qaa]; }
    else if (e < K.k_lx) { if (e - K.k_Fx < NX) v = s[S.l_Fx + e - K.k_Fx]; }
    else if (e < K.k_la) { if (e - K.k_lx < NX) v = lx[e - K.k_lx]; }
    else if (e - K.k_la < NV) v = la[e - K.k_la];
    kkt[e] = v;
  }
}

template <int NV>
__global__ void __launch_bounds__(128) uexpand_kernel(const UStageParams p) {
  constexpr int NX = 2 * NV;
  __shared__ double sm[4][NX + 2 * NV + 2];
  const rbt_ulayout& K = p.K;
  const rbt_ustage_layout& S = p.S;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const size_t oo = size_t(blockIdx.x) * 4 + wid;  // over batch * N (terminal stages skipped)
  if (oo >= size_t(p.batch) * p.N) return;
  const int b = int(oo / p.N), i = int(oo % p.N);
  const size_t o = size_t(b) * (p.N + 1) + i;
  const double* lin = p.lin + o * S.l_stride;
  const double* ex = p.ex + o * S.e_stride;
  const double* d = p.dir + o * K.d_stride;
  double* con = p.con + o * S.c_stride;
  double* xd = p.xd + o * S.x_stride;
  double* dx = sm[wid];
  double* da = dx + NX;
  double* du = da + NV;
  if (lane < NX) dx[lane] = d[K.d_dx + lane];
  if (lane < NV) da[lane] = d[K.d_da + lane];
  __syncwarp();
  if (lane < NV) {
    double acc = lin[S.l_ID + lane];
#pragma unroll
    for (int j = 0; j < NV; ++j)
      acc += lin[S.l_dIDdq + lane + j * NV] * dx[j] + lin[S.l_dIDdv + lane + j * NV] * dx[NV + j] +
             lin[S.l_dIDda + lane + j * NV] * da[j];
    du[lane] = acc;
    xd[S.x_du + lane] = acc;
  }
  __syncwarp();
  if (lane < NV) {
    double acc = ex[S.e_lu + lane];
#pragma unroll
    for (int j = 0; j < NV; ++j) acc += ex[S.e_Quu + lane + j * NV] * du[j];
    xd[S.x_dbeta + lane] = acc / p.dt;
  }
  double mp = 1.0, md = 1.0;
  const double rate = p.tab.fraction_to_boundary;
  for (int r = lane; r < p.tab.n_box; r += 32) {
    const rbt_box_row br = p.tab.box[r];
    if (i < urow_level(br.var)) continue;
    const double* var = br.var == RBT_VAR_Q ? dx : br.var == RBT_VAR_V ? dx + NV : br.var == RBT_VAR_A ? da : du;
    const double sl = con[S.c_slack + r], dl = con[S.c_dual + r];
    const double ds = -br.sign * var[br.idx] - con[S.c_res + r];
    const double dd = -(dl * ds + con[S.c_cmpl + r]) / sl;
    con[S.c_dslack + r] = ds;
    con[S.c_ddual + r] = dd;
    const double fp = -rate * (sl / ds), fd = -rate * (dl / dd);
    if (fp > 0 && fp < 1 && fp < mp) mp = fp;
    if (fd > 0 && fd < 1 && fd < md) md = fd;
  }
  mp = warp_min(mp);
  md = warp_min(md);
  if (lane == 0) {
    atomic_min_pos(&p.steps[2 * b], mp);
    atomic_min_pos(&p.steps[2 * b + 1], md);
  }
}

template <int NV>
__global__ void __launch_bounds__(128) uupdate_kernel(const UStageParams p) {
  const rbt_ulayout& K = p.K;
  const rbt_ustage_layout& S = p.S;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const size_t o = size_t(blockIdx.x) * 4 + wid;
  if (o >= size_t(p.batch) * (p.N + 1)) return;
  const int b = int(o / (p.N + 1)), i = int(o % (p.N + 1));
  const bool terminal = (i == p.N);
  const double ps = p.steps[2 * b], ds = p.steps[2 * b + 1];
  const double* d = p.dir + o * K.d_stride;
  const double* xd = p.xd + o * S.x_stride;
  double* sol = p.sol + o * S.s_stride;
  double* con = p.con + o * S.c_stride;
  if (lane < NV) {
    sol[S.s_q + lane] += ps * d[K.d_dx + lane];
    sol[S.s_v + lane] += ps * d[K.d_dx + NV + lane];
    sol[S.s_lmd + lane] += ps * d[K.d_dlmdgmm + lane];
    sol[S.s_gmm + lane] += ps * d[K.d_dlmdgmm + NV + lane];
    if (!terminal) {
      sol[S.s_a + lane] += ps * d[K.d_da + lane];
      sol[S.s_u + lane] += ps * xd[S.x_du + lane];
      sol[S.s_beta + lane] += ps * xd[S.x_dbeta + lane];
    }
  }
  if (terminal) return;
  for (int r = lane; r < p.tab.n_box; r += 32) {
    if (i < urow_level(p.tab.box[r].var)) continue;
    con[S.c_slack + r] += ps * con[S.c_dslack + r];
    con[S.c_dual + r] += ds * con[S.c_ddual + r];
  }
}

}  // namespace rbt

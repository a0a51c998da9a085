// riccati_forward.cuh -- batched forward Riccati recursion (state / control / costate / multiplier directions).
//
// Behaviour of   RiccatiRecursion::forwardRiccatiRecursion     src/riccati/riccati_recursion.cpp:83-131
//                forwardRiccatiRecursion / computeSwitchingTimeDirection / computeCostateDirection /
//                computeLagrangeMultiplierDirection            src/riccati/riccati_factorizer.cpp:200-281
//
// One CTA (3 warps) per OCP walks i = 0..N.  The sweep is matrix-vector work at ~0.25 FLOP/B, i.e. pure HBM
// streaming: per stage [Fxx|Fvu|Fx] (KKT record) and [P|s|K|k] (Riccati record) arrive by two cp.async.bulk
// copies into a 2-deep ring (stage i+1 in flight while stage i computes), completion on one mbarrier per slot.
// The ring is sized for the plain stage (53.9 KB of shared memory, 4 CTAs/SM).  The extras of a switching-constraint
// or STO stage i ([M|m], [Psi|Phi|T|W], ...: 2 of 47 grid points in a trot) are copied into the OTHER slot instead,
// and stage i+1 is issued once stage i is done: one exposed load latency on those stages only.
#pragma once
#include "rbt_device.cuh"
#include "../../include/rbt_layout.h"

namespace rbt {

struct FwdParams {
  rbt_layout L;
  const rbt_stage_ctrl* ctrl;
  int n_grid;
  int batch;
  const double* kkt;
  const double* ric;
  const double* dx0;  // [batch][nx]
  double* dir;        // [batch][n_grid][d_stride]
  // time-parallel sweep (SEG instance only, riccati_time_parallel.cuh)
  int segs;
  const double* dxseed;  // [batch][segs][nx]: dx at the first grid point of segment j >= 1
  const int* tp_fail;    // [batch]: nonzero = CTA (ocp, 0) sweeps the whole horizon from dx0
};

template <int NV, int NU, int NS>
struct FwdCfg {
  static constexpr int NX = 2 * NV;
  static constexpr int NTHREADS = 96;
  static constexpr int KPART = NX * NX + ((NV * NU + 1) & ~1) + ((NX + 1) & ~1);          // Fxx|Fvu|Fx
  static constexpr int RPART = NX * NX + ((NX + 1) & ~1) + ((NU * NX + 1) & ~1) + ((NU + 1) & ~1);  // P|s|K|k
  // extras (in the slot after the stage's own): [M|m] [Psi|Phi|T|W] [mt|mtn] [dtsdx|stosc] [fx]
  static constexpr int e_M = 0;
  static constexpr int e_m = e_M + ((NS * NX + 1) & ~1);
  static constexpr int e_Psi = e_m + ((NS + 1) & ~1);
  static constexpr int e_Phi = e_Psi + ((NX + 1) & ~1);
  static constexpr int e_T = e_Phi + ((NX + 1) & ~1);
  static constexpr int e_W = e_T + ((NU + 1) & ~1);
  static constexpr int e_mt = e_W + ((NU + 1) & ~1);
  static constexpr int e_mtn = e_mt + ((NS + 1) & ~1);
  static constexpr int e_pol = e_mtn + ((NS + 1) & ~1);  // dtsdx (nx) | dtsdts, dts0
  static constexpr int e_fx = e_pol + ((NX + 1) & ~1) + 2;
  static constexpr int ESZ = e_fx + ((NX + 1) & ~1);
  static constexpr int SLOT = KPART + RPART;
  static_assert(ESZ <= SLOT, "the extras of a stage must fit one ring slot");
  static constexpr int o_dx = 2 * SLOT;  // dx ping-pong (2 x NX), du (NU)
  static constexpr int o_du = o_dx + 2 * NX;
  static constexpr int o_bar = o_du + ((NU + 1) & ~1);
  static constexpr int SMEM_DOUBLES = o_bar + 2;
  static constexpr size_t SMEM_BYTES = size_t(SMEM_DOUBLES) * 8;
};

// SEG: the time-parallel instance -- CTA (ocp, j) sweeps grid points lo_j .. hi_j - 1 (the last segment through N) from
// p.dxseed.  Ring slots and the dx ping-pong count from the segment's first grid point.
template <int NV, int NU, int NS, bool SEG = false>
__global__ void __launch_bounds__(FwdCfg<NV, NU, NS>::NTHREADS, 4) riccati_forward_kernel(const FwdParams p) {
  using C = FwdCfg<NV, NU, NS>;
  constexpr int NX = C::NX, NTHR = C::NTHREADS;
  constexpr int CO = ((NX + 15) / 16) * 16;  // first thread of the costate group
  static_assert(CO + NX <= NTHR, "costate thread group must fit");
  extern __shared__ __align__(16) double smem[];
  const rbt_layout& L = p.L;
  const int tid = threadIdx.x;
  const int b = SEG ? int(blockIdx.x) / p.segs : int(blockIdx.x);
  if (b >= p.batch) return;
  const int N = p.n_grid - 1;
  int lo = 0, last = N, seg = 0;
  if constexpr (SEG) {
    seg = int(blockIdx.x) % p.segs;
    if (p.tp_fail[b] != 0) {
      if (seg != 0) return;
    } else {
      lo = tp_seg_lo(seg, N, p.segs);
      last = (seg == p.segs - 1) ? N : tp_seg_lo(seg + 1, N, p.segs) - 1;
    }
  }
  const double* kkt_b = p.kkt + size_t(b) * p.n_grid * L.k_stride;
  const double* ric_b = p.ric + size_t(b) * p.n_grid * L.r_stride;
  double* dir_b = p.dir + size_t(b) * p.n_grid * L.d_stride;
  double* sdx = smem + C::o_dx;
  double* sdu = smem + C::o_du;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + C::o_bar);  // one per ring slot

  auto needs_pol = [&](int st) {
    const rbt_stage_ctrl c = p.ctrl[st];
    return (st == 0 && c.sto) || ((c.type == RBT_IMPACT || c.type == RBT_LIFT) && c.sto_next);
  };
  auto has_extras = [&](int st) {
    const rbt_stage_ctrl c = p.ctrl[st];
    return st < N && (c.ns > 0 || c.sto || needs_pol(st));
  };
  // one elected thread: the main copies of grid point st into ring slot (st - lo) & 1
  auto issue_main = [&](int st) {
    const int slot = (st - lo) & 1;
    double* base = smem + slot * C::SLOT;
    const double* krec = kkt_b + size_t(st) * L.k_stride;
    const double* rrec = ric_b + size_t(st) * L.r_stride;
    fence_proxy_async();
    if (st < N) {
      mbar_expect_tx(&bars[slot], uint32_t(C::KPART + C::RPART) * 8u);
      tma_load_1d(base, krec + L.k_Fxx, uint32_t(C::KPART) * 8u, &bars[slot]);
      tma_load_1d(base + C::KPART, rrec + L.r_P, uint32_t(C::RPART) * 8u, &bars[slot]);
    } else {  // terminal: only P|s
      const uint32_t by = uint32_t(NX * NX + ((NX + 1) & ~1)) * 8u;
      mbar_expect_tx(&bars[slot], by);
      tma_load_1d(base + C::KPART, rrec + L.r_P, by, &bars[slot]);
    }
  };
  // one elected thread: the extras of grid point st into the other slot, (st - lo + 1) & 1
  auto issue_extras = [&](int st) {
    const int slot = (st - lo + 1) & 1;
    double* ex = smem + slot * C::SLOT;
    const rbt_stage_ctrl c = p.ctrl[st];
    const double* krec = kkt_b + size_t(st) * L.k_stride;
    const double* rrec = ric_b + size_t(st) * L.r_stride;
    fence_proxy_async();
    uint32_t bytes = 0;
    if (c.ns > 0) bytes += uint32_t(C::e_Psi - C::e_M) * 8u;
    if (c.sto) bytes += uint32_t(C::e_mt - C::e_Psi) * 8u + uint32_t(C::ESZ - C::e_fx) * 8u;
    if (c.sto && c.ns > 0) bytes += uint32_t(C::e_pol - C::e_mt) * 8u;
    if (needs_pol(st)) bytes += uint32_t(C::e_fx - C::e_pol) * 8u;
    mbar_expect_tx(&bars[slot], bytes);
    if (c.ns > 0) tma_load_1d(ex + C::e_M, rrec + L.r_M, uint32_t(C::e_Psi - C::e_M) * 8u, &bars[slot]);
    if (c.sto) {
      tma_load_1d(ex + C::e_Psi, rrec + L.r_Psi, uint32_t(C::e_mt - C::e_Psi) * 8u, &bars[slot]);
      tma_load_1d(ex + C::e_fx, krec + L.k_fx, uint32_t(C::ESZ - C::e_fx) * 8u, &bars[slot]);
    }
    if (c.sto && c.ns > 0) tma_load_1d(ex + C::e_mt, rrec + L.r_mt, uint32_t(C::e_pol - C::e_mt) * 8u, &bars[slot]);
    if (needs_pol(st)) tma_load_1d(ex + C::e_pol, rrec + L.r_dtsdx, uint32_t(C::e_fx - C::e_pol) * 8u, &bars[slot]);
  };
  // Ring invariant at the top of stage i: slot (i - lo) & 1 holds (or receives) stage i; the other slot receives the
  // extras of stage i if it has any, else stage i + 1.  Every copy into a slot is matched by exactly one wait on its
  // mbarrier, so each slot's phase parity is the count of its waits mod 2 (bit s of `ph`, identical in every thread).
  auto issue_after = [&](int i) {  // stage i's copies are done; i + 1 is in flight unless stage i had extras
    if (has_extras(i) && i + 1 <= last) issue_main(i + 1);
    if (i + 1 <= last && has_extras(i + 1)) issue_extras(i + 1);
    else if (i + 2 <= last) issue_main(i + 2);
  };

  if (tid == 0) {
    for (int q = 0; q < 2; ++q) mbar_init(&bars[q], 1);
    fence_mbar_init();
  }
  if (tid < NX) sdx[tid] = (SEG && lo > 0) ? p.dxseed[(size_t(b) * p.segs + seg) * NX + tid] : p.dx0[size_t(b) * NX + tid];
  __syncthreads();
  if (tid == 0) {
    issue_main(lo);
    if (has_extras(lo)) issue_extras(lo);
    else if (last >= lo + 1) issue_main(lo + 1);
  }
  uint32_t ph = 0;             // mbarrier parity per slot
  double dts = 0.0, dtsn = 0.0;  // final switching-time directions of the previous stage

  for (int i = lo; i <= last; ++i) {
    const int slot = (i - lo) & 1;
    const rbt_stage_ctrl c = p.ctrl[i];
    const double* base = smem + slot * C::SLOT;
    const double* sA = base;
    const double* sB = base + NX * NX;
    const double* sFx = sB + ((NV * NU + 1) & ~1);
    const double* sPm = base + C::KPART;
    const double* ss = sPm + NX * NX;
    const double* sKt = ss + ((NX + 1) & ~1);
    const double* sk = sKt + ((NU * NX + 1) & ~1);
    const double* ex = smem + (slot ^ 1) * C::SLOT;  // extras (only read when `extras`)
    double* dx = sdx + ((i - lo) & 1) * NX;
    double* dxn = sdx + ((i - lo + 1) & 1) * NX;
    double* drec = dir_b + size_t(i) * L.d_stride;
    const bool terminal = (i == N);
    const bool impact = (!terminal && c.type == RBT_IMPACT);
    const bool lift = (!terminal && c.type == RBT_LIFT);
    const bool sto = !terminal && c.sto, sto_next = !terminal && c.sto_next;
    const bool extras = !terminal && has_extras(i);

    mbar_wait(&bars[slot], (ph >> slot) & 1u);
    ph ^= 1u << slot;
    if (extras) {
      mbar_wait(&bars[slot ^ 1], (ph >> (slot ^ 1)) & 1u);
      ph ^= 1u << (slot ^ 1);
    }

    // ---- switching-time bookkeeping (riccati_recursion.cpp:88-118); entry state = final state of stage i-1
    if (i == 0 && sto) {  // :90-93, has_prev_sto_phase = false
      dtsn = dot_serial(ex + C::e_pol, dx, NX) + ex[C::e_pol + ((NX + 1) & ~1) + 1];
    }
    if (lift) {
      dts = dtsn;
      dtsn = 0.0;
      if (sto_next) {
        dtsn = dot_serial(ex + C::e_pol, dx, NX) + ex[C::e_pol + ((NX + 1) & ~1) + 1];
        if (sto) dtsn += ex[C::e_pol + ((NX + 1) & ~1)] * dts;
      }
    }
    if (impact) {
      dts = dtsn;
      dtsn = 0.0;
    }
    const double delta = dtsn - dts;

    if (!terminal && !impact) {
      // du = K dx + k (+ T (dts_next - dts) - W dts_next)           riccati_factorizer.cpp:205-212
      matvec_T(sKt, NX, NX, NU, dx, tid, NTHR, [&](int u, double a) {
        double v = a + sk[u];
        if (sto) {
          v += ex[C::e_T + u] * delta;
          if (sto_next) v -= ex[C::e_W + u] * dtsn;
        }
        sdu[u] = v;
        drec[L.d_du + u] = v;
      });
      __syncthreads();
    }
    if (tid < NX) {
      const int r = tid;
      drec[L.d_dx + r] = dx[r];
      if (!terminal) {
        // dx+ = Fx + A dx (+ [0; Bv du]) (+ fx (dts_next - dts))      :213-218 / :227-229
        double a = sFx[r];
        for (int k = 0; k < NX; ++k) a = fma(sA[r + k * NX], dx[k], a);
        if (!impact) {
          if (r >= NV)
            for (int u = 0; u < NU; ++u) a = fma(sB[(r - NV) + u * NV], sdu[u], a);
          if (sto) a = fma(ex[C::e_fx + r], delta, a);
        }
        dxn[r] = a;
      }
    } else if (tid >= CO && tid < CO + NX && !(impact && sto_next)) {
      // dlmdgmm = P dx - s (+ Psi (dts_next-dts) - Phi dts_next)       :246-266
      const int r = tid - CO;
      double a = -ss[r];
      for (int k = 0; k < NX; ++k) a = fma(sPm[r + k * NX], dx[k], a);
      if (sto) {
        if (impact) {
          a -= ex[C::e_Phi + r] * dtsn;
        } else {
          a += ex[C::e_Psi + r] * delta;
          if (sto_next) a -= ex[C::e_Phi + r] * dtsn;
        }
      }
      drec[L.d_dlmdgmm + r] = a;
    }
    // dx+ is complete.  A plain stage has read its slot for the last time (so has every thread the dx of this stage):
    // the slot is refilled right away, and the next stage starts without another barrier.
    __syncthreads();

    if (extras) {
      if (impact && sto_next) {
        // impact with an STO phase after it: dts_next comes from the NEW state dx+      riccati_recursion.cpp:100-106
        const double e_dts = dts;  // d[i+1].dts = d[i-1].dts_next
        double e_dtsn = dot_serial(ex + C::e_pol, dxn, NX) + ex[C::e_pol + ((NX + 1) & ~1) + 1];
        if (sto) e_dtsn += ex[C::e_pol + ((NX + 1) & ~1)] * e_dts;
        dts = e_dts;
        dtsn = e_dtsn;
        if (tid >= CO && tid < CO + NX) {
          const int r = tid - CO;
          double a = -ss[r];
          for (int k = 0; k < NX; ++k) a = fma(sPm[r + k * NX], dx[k], a);
          if (sto) a -= ex[C::e_Phi + r] * dtsn;
          drec[L.d_dlmdgmm + r] = a;
        }
      }
      if (!terminal && !impact && c.ns > 0) {
        // dxi = M dx + m (+ mt (dts_next-dts) - mt_next dts_next)        riccati_factorizer.cpp:269-281
        const int ns = c.ns;
        for (int q = tid; q < ns; q += NTHR) {
          double a = ex[C::e_m + q];
          for (int k = 0; k < NX; ++k) a = fma(ex[C::e_M + q + k * ns], dx[k], a);
          if (sto) {
            a += ex[C::e_mt + q] * delta;
            if (sto_next) a -= ex[C::e_mtn + q] * dtsn;
          }
          drec[L.d_dxi + q] = a;
        }
      }
      __syncthreads();  // everyone is done with the slot and the extras of this stage
    }
    if (tid == 0) {
      drec[L.d_dts + 0] = dts;
      drec[L.d_dts + 1] = dtsn;
      issue_after(i);
    }
  }
}

}  // namespace rbt

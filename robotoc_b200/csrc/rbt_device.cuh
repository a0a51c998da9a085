// rbt_device.cuh -- sm_90a device helpers: 1-D TMA bulk copies + mbarrier, fp64 tensor-pipe tiles
// (mma.sync.m8n8k4.f64, DMMA), small warp-parallel dense helpers.  fp64 has no wgmma kind, so the
// tensor pipe is reached through DMMA (tools/fp64_microbench.cu compares it with DFMA).
#pragma once
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

namespace rbt {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---- mbarrier / TMA (cp.async.bulk, 1-D) -------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Spins on try_wait (HW-suspended wait).  A bulk copy that never completes would hang the GPU box, so the spin is
// bounded: after ~2^24 failed probes (seconds) the kernel traps and the host sees a CUDA error instead of a hang.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  uint32_t tries = 0;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    if (!ok && ++tries > (1u << 24)) {
      if ((threadIdx.x & 31) == 0)
        printf("[rbt] mbarrier wait timed out: block %d thread %d bar %u parity %u\n", blockIdx.x, threadIdx.x,
               smem_u32(bar), parity);
      __trap();
    }
  } while (!ok);
}
// global -> shared bulk copy; bytes % 16 == 0, both addresses 16-B aligned.  SASS: UBLKCP.
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- 1-D TMA bulk store shared -> global (bulk async-group completion).  The issuing thread must (a) order the CTA's generic-
// proxy writes to the source before the copy: barrier, then tma_store_fence(); (b) keep the source alive until the copy has READ
// it: tma_store_wait_read() before the buffer is reused or the CTA exits.
__device__ __forceinline__ void tma_store_fence() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_store_1d(void* gmem_dst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

// ---- DMMA m8n8k4: D(8x8) += A(8x4) * B(4x8), fp64.  lane = 4*g + t:
//   a = A[g][t],  b = B[t][g],  c0 = C[g][2t], c1 = C[g][2t+1]
__device__ __forceinline__ void dmma884(double& c0, double& c1, double a, double b) {
  // volatile: the instruction is warp-convergent; it must never be cloned into the arms of a per-thread branch
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

// Bulk L2 prefetch (no shared-memory destination, no completion tracking): bytes multiple of 16, 16-byte aligned source.
__device__ __forceinline__ void l2_prefetch_bulk(const void* gmem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gmem_src), "r"(bytes) : "memory");
}

// Tile origin for an extent M covered by 8-wide tiles: full tiles, then one tile pulled back to end at M
// (overlapping rows/cols are simply computed twice with identical operands -> identical bits).
__host__ __device__ constexpr int tile_off(int t, int M) { return (8 * t + 8 <= M) ? 8 * t : (M >= 8 ? M - 8 : 0); }
__host__ __device__ constexpr int num_tiles(int M) { return (M + 7) / 8; }

// One warp accumulates NT 8x8 tiles of one 8-row band:  acc[n] += sum_k A(i0+g, k) * B(k, joff(n)+g).
//   fa(i, k) / fb(k, j) return the operand element (shared-memory loads).  K need not be a multiple of 4.
// n_begin (warp-uniform): tiles n < n_begin are skipped (symmetric products: only the tiles on/above the diagonal band).
// PIPE = false: one fragment set, the loads of k-step ks issued right before its MMAs (NT + 1 fewer live doubles) -- for the
// register-starved backward sweep (80-register cap: the second fragment set only adds spills there).
template <int K, int NT, int N, bool PIPE = true, class FA, class FB>
__device__ __forceinline__ void warp_mma_band(double (&acc)[NT][2], int i0, FA fa, FB fb, int n_begin = 0) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  constexpr int KS = (K + 3) / 4;
  // Software-pipelined by hand: the operands of k-step ks+1 are loaded BEFORE the NT tensor instructions of k-step ks are
  // issued.  (The volatile MMA statements are scheduling barriers for ptxas: with the natural "load b, mma, load b, mma"
  // order every DMMA would wait a full shared-memory latency for its own operand.)
  auto load = [&](int ks, double& a, double (&b)[NT]) {
    const int k0 = 4 * ks;
    // K tail: load from a clamped (valid) index and zero the A operand arithmetically -- no per-thread branch
    // may surround the warp-convergent MMA.
    const int k = (K % 4 == 0) ? (k0 + t) : min(k0 + t, K - 1);
    const double msk = ((K % 4 == 0) || (k0 + t < K)) ? 1.0 : 0.0;
    a = fa(i0 + g, k) * msk;
#pragma unroll
    for (int n = 0; n < NT; ++n)
      if (n >= n_begin) b[n] = fb(k, tile_off(n, N) + g);
  };
  if constexpr (!PIPE) {
    double a, b[NT];
#pragma unroll
    for (int ks = 0; ks < KS; ++ks) {
      load(ks, a, b);
#pragma unroll
      for (int n = 0; n < NT; ++n)
        if (n >= n_begin) dmma884(acc[n][0], acc[n][1], a, b[n]);
    }
    return;
  }
  double a0, b0[NT], a1, b1[NT];
  load(0, a0, b0);
#pragma unroll
  for (int ks = 0; ks < KS; ks += 2) {
    if (ks + 1 < KS) load(ks + 1, a1, b1);
#pragma unroll
    for (int n = 0; n < NT; ++n)
      if (n >= n_begin) dmma884(acc[n][0], acc[n][1], a0, b0[n]);
    if (ks + 1 < KS) {
      if (ks + 2 < KS) load(ks + 2, a0, b0);
#pragma unroll
      for (int n = 0; n < NT; ++n)
        if (n >= n_begin) dmma884(acc[n][0], acc[n][1], a1, b1[n]);
    }
  }
}

// ---- small dense helpers over shared memory (all threads of the CTA cooperate; tid/nthr given) ----
// y[c] = sum_k A[k + c*lda] * x[k]  (A^T x), 4 lanes per column, conflict-free for lda % 4 == 0 or 2.
// Call with all threads; uses shuffles inside aligned groups of 4 lanes.  Result written by lane q==0.
template <class Epi>
__device__ __forceinline__ void matvec_T(const double* A, int lda, int K, int C, const double* x, int tid, int nthr,
                                         Epi epi) {
  const int q = tid & 3;
  const int ngroups = nthr >> 2;
  const int Cpad = (C + ngroups - 1) / ngroups * ngroups;
  for (int c = tid >> 2; c < Cpad; c += ngroups) {
    double acc = 0.0;
    if (c < C)
      for (int k = q; k < K; k += 4) acc = fma(A[k + c * lda], x[k], acc);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    if (q == 0 && c < C) epi(c, acc);
  }
}

// y[r] = sum_k A[r + k*lda] * x[k]  (A x), one thread per row (conflict-free: consecutive lanes, consecutive rows).
template <class Epi>
__device__ __forceinline__ void matvec_N(const double* A, int lda, int R, int K, const double* x, int tid, int nthr,
                                         Epi epi) {
  for (int r = tid; r < R; r += nthr) {
    double acc = 0.0;
    for (int k = 0; k < K; ++k) acc = fma(A[r + k * lda], x[k], acc);
    epi(r, acc);
  }
}

// y[r] = sum_k A[r + k*lda] * x[k]  (A x) with 4 lanes per row (k interleaved) + 2 shuffles: 4x shorter dependent chain
// than matvec_N.  Call with whole warps (nthr multiple of 32).
template <class Epi>
__device__ __forceinline__ void matvec_N4(const double* A, int lda, int R, int K, const double* x, int tid, int nthr,
                                          Epi epi) {
  const int q = tid & 3;
  const int ngroups = nthr >> 2;
  const int Rpad = (R + ngroups - 1) / ngroups * ngroups;
  for (int r = tid >> 2; r < Rpad; r += ngroups) {
    double acc = 0.0;
    if (r < R)
      for (int k = q; k < K; k += 4) acc = fma(A[r + k * lda], x[k], acc);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    if (q == 0 && r < R) epi(r, acc);
  }
}

// ---- fast fp64 reciprocal / reciprocal square root: MUFU seed (rel. error 2^-23) + two Newton steps -> ~1 ulp.  The seeds
// flush subnormals; pivots of the factorizations here are O(1e-6 .. 1e12).
__device__ __forceinline__ double fast_rcp(double d) {
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(d));
  r = fma(r, fma(-d, r, 1.0), r);
  r = fma(r, fma(-d, r, 1.0), r);
  return r;
}
__device__ __forceinline__ double fast_rsqrt(double d) {
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
  double h = 0.5 * d;
  y = y * fma(-h * y, y, 1.5);
  y = y * fma(-h * y, y, 1.5);
  return y;
}

// Cholesky factor AND its inverse of an N x N (N <= 16) SPD matrix held in registers by ONE warp, N doubles per lane:
//   lane r < N       holds ROW r of the matrix in c[0..N-1] (entries k <= r are read; the others are scratch),
//   lane 16 + q      builds COLUMN q of the inverse of the unit-lower factor (starts as the unit vector e_q).
// Square-root-free elimination A = L_u D L_u^T.  With the inverse kept column-wise, step j is the SAME statement on both
// half-warps:  w = c[j] / d_j ;  c[s] -= w * a_sj  (s > j),  where a_sj = slot j of matrix lane s comes from ONE shuffle that
// serves both halves (matrix lane r: a_rs -= (a_rj / d_j) a_sj;  inverse lane q: e_s[q] -= (a_sj / d_j) e_j[q]).
// No shared-memory round trip, no __syncwarp, no per-element predicate.  The pivot chain is shuffle -> reciprocal (MUFU seed
// + 2 Newton steps) -> multiply -> fma; the column shuffles are issued under the reciprocal (tools/lat_microbench.cu
// measures these latencies).  Square roots are taken once at the end, one per lane.
// On exit:  lane r < N:   c[k] = L[r][k]      (k <= r; Cholesky factor, A = L L^T)
//           lane 16 + q:  c[k] = (L^-1)[k][q] (k >= q; exactly 0 above the diagonal)
//           rs (every lane l): 1 / L[l & 15][l & 15] on lanes with (l & 15) < N.
// Returns false (on every lane) if a pivot was not positive.
template <int N>
__device__ __forceinline__ bool warp_chol_inv_reg(double (&c)[N], double& rs) {
  static_assert(N <= 16, "two half-warps");
  const int lane = threadIdx.x & 31;
  const int idx = lane & 15;
  bool ok = true;
  double dsave = 1.0;
  if (lane >= 16) {
#pragma unroll
    for (int k = 0; k < N; ++k) c[k] = (k == idx) ? 1.0 : 0.0;
  }
#pragma unroll
  for (int j = 0; j < N; ++j) {
    const double dj = __shfl_sync(0xffffffffu, c[j], j);  // pivot
    double v[N];
#pragma unroll
    for (int s = j + 1; s < N; ++s) v[s] = __shfl_sync(0xffffffffu, c[j], s);  // unscaled column j: a_sj
    ok = ok && (dj > 0.0);
    if (idx == j) dsave = dj;
    const double w = c[j] * fast_rcp(dj);
#pragma unroll
    for (int s = j + 1; s < N; ++s) c[s] = fma(-w, v[s], c[s]);
  }
  rs = fast_rsqrt(dsave);  // lanes (l & 15) == j hold 1 / sqrt(d_j)
#pragma unroll
  for (int j = 0; j < N; ++j) c[j] *= __shfl_sync(0xffffffffu, rs, j);  // L[r][j] = a_rj / sqrt(d_j) | (L^-1)[j][q] = e_j[q] / sqrt(d_j)
  return ok;
}

__device__ __forceinline__ double dot_serial(const double* a, const double* b, int n) {
  double s = 0.0;
  for (int i = 0; i < n; ++i) s = fma(a[i], b[i], s);
  return s;
}

}  // namespace rbt

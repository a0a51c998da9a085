// rbt_api.cu -- C ABI of librobotoc_b200.so (see include/robotoc_b200.h for the reference interfaces replaced).
// Plumbing only: handles, device buffers, stream-ordered copies and kernel launches.  No CPU compute path.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <cstdint>
#include <cstdlib>
#include <string>
#include <vector>

#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <cstdlib>

#include "../../include/robotoc_b200.h"
#include "riccati_backward.cuh"
#include "riccati_forward.cuh"
#include "riccati_time_parallel.cuh"
#include "riccati_unconstr.cuh"
#include "stage_kernels.cuh"
#include "ustage_kernels.cuh"
#include "eval_kernels.cuh"
#include "line_search_kernels.cuh"
#include "rnea_kernels.cuh"

namespace {

struct Err {
  std::string msg;
};

#define RBT_CUDA(h, call)                                                                     \
  do {                                                                                        \
    cudaError_t e_ = (call);                                                                  \
    if (e_ != cudaSuccess) {                                                                  \
      (h)->err = std::string(#call) + ": " + cudaGetErrorString(e_);                          \
      return RBT_ERR_CUDA;                                                                    \
    }                                                                                         \
  } while (0)

template <class K>
int set_smem(K kernel, size_t bytes) {
  return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) == cudaSuccess ? 0 : 1;
}

}  // namespace

struct rbt_handle {
  rbt_dims dims;
  rbt_layout L;
  int n_grid_max = 0, n_grid = 0, batch = 0, device = 0;
  double max_dts0 = 0.1;
  rbt_stage_ctrl* d_ctrl = nullptr;
  std::vector<rbt_stage_ctrl> ctrl;  // host copy
  double *d_kkt = nullptr, *d_ric = nullptr, *d_fact = nullptr, *d_dir = nullptr, *d_dx0 = nullptr;
  double* own[12] = {};  // the handle's own allocation of a buffer that the caller re-bound (freed in destroy)
  int* d_info = nullptr;
  int* d_arrivals = nullptr;  // per-SM CTA arrival counters (CTA de-phasing in the backward kernel)
  int* d_struct = nullptr;    // [0]: 1 = every Fxx of the KKT buffer has the mechanical structure (see rbt_set_fxx_structure)
  int fxx_mode = RBT_FXX_AUTO;
  // time-parallel sweeps (riccati_time_parallel.cuh): requested segment count (0 = automatic, 1 = serial) and scratch,
  // allocated on the first segmented sweep; the S-dependent buffers grow with the largest S used
  int tsegs = 0, n_sm = 0, tp_cap = 0;
  double *d_tp_elem = nullptr, *d_tp_scan[2] = {nullptr, nullptr}, *d_tp_fmap = nullptr, *d_tp_dx = nullptr;
  int* d_tp_fail = nullptr;
  const double* tp_seeds = nullptr;  // the scan buffer the last segmented backward sweep read its seeds from
  bool kkt_from_condense = false;  // the KKT records were just written by rbt_condense: structure holds by construction
  int stagger_ns = 0;
  long long* d_timeline = nullptr;  // bring-up instrumentation (RBT_TIMELINE_CTA)
  // stage layer
  bool stage_ready = false;
  bool keep_info = false;  // condense's Cholesky flags survive the following backward launch
  rbt_stage_dims sdims;
  rbt_stage_layout S;
  rbt_constraint_table table;
  double *d_lin = nullptr, *d_con = nullptr, *d_ex = nullptr, *d_sol = nullptr, *d_xd = nullptr, *d_steps = nullptr,
         *d_ones = nullptr;
  double *d_stage_perf = nullptr, *d_perf = nullptr, *d_x0in = nullptr;  // eval_kernels.cuh
  // line search (line_search_kernels.cuh): trial buffers sized on first use, filter state per OCP
  int ls_trials = 0;
  double *d_ls_alphas = nullptr, *d_ls_trial = nullptr, *d_ls_stage_barrier = nullptr, *d_ls_barrier = nullptr;
  double *d_ls_in = nullptr, *d_ls_filt = nullptr, *d_ls_step = nullptr;
  int *d_ls_nfilt = nullptr, *d_ls_k = nullptr;
  double* d_step_pack = nullptr;  // packed Newton step of this rank (rbt_allgather_step), allocated on first use
  int timeline_cta = -1;
  long long launches = 0;
  // batch window [cb0, cb0 + cnb) the launch helpers work on (cnb == 0: the whole batch); used by rbt_iteration_host to
  // pipeline uploads, kernels and downloads over chunks of the batch
  int cb0 = 0, cnb = 0;
  double* d_wire = nullptr;  // packed host wire records (rbt_iteration_host_wire), allocated on first use
  int* d_tgt = nullptr;           // box rows per PDIPM target (stage_kernels.cuh: StageParams::tgt)
  double* d_bound = nullptr;      // joint limits per box row (rbt_set_joint_limits)
  rbt::RneaModel* d_model = nullptr;  // robot model of rbt_linearize_inverse_dynamics (rbt_set_robot_model)
  double* d_res_stage = nullptr;  // rbt_iteration_host_resident: compact residuals in, compact slack|dual out
  double* d_sd_stage = nullptr;
  std::vector<rbt_wire_layout> Wv;   // per grid point (the wire record of a grid point depends on its control word)
  rbt_wire_layout* d_W = nullptr;
  long long w_ocp = 0;               // doubles of one OCP's concatenated wire records
  int cost_structure = RBT_COST_GENERAL;  // what the host's wire records hold (rbt_set_wire_cost_structure)
  bool wire_dirty = true;                 // per-grid-point wire layouts on the device are stale (schedule / cost structure changed)
  bool attr_bwd = false, attr_fwd = false, attr_cond = false, attr_tp = false;  // MaxDynamicSharedMemorySize set on THIS handle's device
  cudaEvent_t ev_condense_mid = nullptr;  // caller-owned event recorded between the two kernels of rbt_condense (timing)
  cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
  std::vector<cudaEvent_t> ev;
  std::string err;
};

static inline int win_b0(const rbt_handle* h) { return h->cnb ? h->cb0 : 0; }
static inline int win_nb(const rbt_handle* h) { return h->cnb ? h->cnb : h->batch; }

struct rbt_uhandle {
  int nv = 0, N = 0, batch = 0, device = 0;
  double dt = 0;
  rbt_ulayout L;
  double *d_kkt = nullptr, *d_ric = nullptr, *d_fact = nullptr, *d_dir = nullptr, *d_dx0 = nullptr;
  int* d_info = nullptr;
  // stage layer
  bool stage_ready = false;
  rbt_ustage_layout S;
  rbt_constraint_table table;
  double *d_lin = nullptr, *d_con = nullptr, *d_ex = nullptr, *d_sol = nullptr, *d_xd = nullptr, *d_steps = nullptr,
         *d_ones = nullptr;
  long long launches = 0;
  std::string err;
};

// ---- compiled instances ------------------------------------------------------------------------------------------
// ANYmal (floating base + 4 point contacts): nv=18, nu=12, max_dimf=12     src/robot/robot.cpp:33-60
#define RBT_INSTANCES(X) X(18, 12, 12)

static bool instance_supported(const rbt_dims& d) {
#define X(NV, NU, NS) \
  if (d.nv == NV && d.nu == NU && d.ns_max == NS) return true;
  RBT_INSTANCES(X)
#undef X
  return false;
}

// All functions below are declared extern "C" in include/robotoc_b200.h; the definitions inherit that linkage.

const char* rbt_version(void) { return "robotoc_b200 0.1 (sm_90a; instances: constrained nv18/nu12/ns12; unconstr nv7)"; }

int rbt_layout_get(const rbt_dims* dims, const char* field) {
  if (!dims || !field) return -1;
  rbt_layout L;
  rbt_make_layout(dims, &L);
  return rbt_layout_field(&L, field);
}

int rbt_ulayout_get(int nv, const char* field) {
  if (nv <= 0 || !field) return -1;
  rbt_ulayout L;
  rbt_make_ulayout(nv, &L);
  return rbt_ulayout_field(&L, field);
}

int rbt_device_info(int device, int* sm, int* n_sm, char* name, int name_len) {
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) {
    cudaGetLastError();
    return RBT_ERR_CUDA;
  }
  if (sm) *sm = prop.major * 10 + prop.minor;
  if (n_sm) *n_sm = prop.multiProcessorCount;
  if (name && name_len > 0) {
    std::strncpy(name, prop.name, name_len - 1);
    name[name_len - 1] = 0;
  }
  return RBT_OK;
}

int rbt_create(const rbt_dims* dims, int n_grid_max, int batch, int device, rbt_handle** out) {
  if (!dims || !out || n_grid_max < 2 || batch < 1 || dims->nv < 1 || dims->nu < 1 || dims->ns_max < 0) return RBT_ERR_ARG;
  if (!instance_supported(*dims)) return RBT_ERR_ARG;
  rbt_handle* h = new rbt_handle();
  h->dims = *dims;
  rbt_make_layout(dims, &h->L);
  h->n_grid_max = n_grid_max;
  h->batch = batch;
  h->device = device;
  *out = h;
  RBT_CUDA(h, cudaSetDevice(device));
  const size_t per = size_t(batch) * n_grid_max;
  RBT_CUDA(h, cudaMalloc(&h->d_ctrl, sizeof(rbt_stage_ctrl) * n_grid_max));
  RBT_CUDA(h, cudaMalloc(&h->d_kkt, per * h->L.k_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_ric, per * h->L.r_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_fact, per * h->L.f_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_dir, per * h->L.d_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_dx0, size_t(batch) * h->L.nx * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_info, size_t(batch) * sizeof(int)));
  RBT_CUDA(h, cudaMalloc(&h->d_arrivals, 1024 * sizeof(int)));
  RBT_CUDA(h, cudaMalloc(&h->d_struct, 4 * sizeof(int)));
  RBT_CUDA(h, cudaMemset(h->d_struct, 0, 4 * sizeof(int)));
  h->stagger_ns = getenv("RBT_STAGGER_NS") ? atoi(getenv("RBT_STAGGER_NS")) : 0;
  if (getenv("RBT_TIMELINE_CTA")) {
    h->timeline_cta = atoi(getenv("RBT_TIMELINE_CTA"));
    RBT_CUDA(h, cudaMalloc(&h->d_timeline, size_t(n_grid_max) * 32 * sizeof(long long)));
    RBT_CUDA(h, cudaMemset(h->d_timeline, 0, size_t(n_grid_max) * 32 * sizeof(long long)));
  }
  RBT_CUDA(h, cudaMemset(h->d_kkt, 0, per * h->L.k_stride * 8));  // condensing skips the switching rows a stage lacks: keep them defined
  RBT_CUDA(h, cudaMemset(h->d_ric, 0, per * h->L.r_stride * 8));
  RBT_CUDA(h, cudaMemset(h->d_fact, 0, per * h->L.f_stride * 8));
  RBT_CUDA(h, cudaMemset(h->d_dir, 0, per * h->L.d_stride * 8));
  RBT_CUDA(h, cudaMemset(h->d_info, 0, size_t(batch) * sizeof(int)));
  RBT_CUDA(h, cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, device));
  return RBT_OK;
}

static double** buf_slot(rbt_handle* h, int which);

// The stage kernels are compiled for nf_max / n_contacts of the constraint table: every grid of the schedule must fit.
static int check_contacts(rbt_handle* h, const rbt_stage_ctrl* ctrl, int n_grid) {
  if (!h->stage_ready) return RBT_OK;
  for (int i = 0; i < n_grid; ++i)
    if (ctrl[i].nf > h->sdims.nf_max || ctrl[i].contact_mask >= (1 << h->sdims.n_contacts)) {
      h->err = "[rbt_set_schedule] invalid argument: grid " + std::to_string(i) + " has more contacts than the stage layer was set up for";
      return RBT_ERR_ARG;
    }
  return RBT_OK;
}

int rbt_destroy(rbt_handle* h) {
  if (h) {
    cudaFree(h->d_wire);
    cudaFree(h->d_W);
    cudaFree(h->d_tgt);
    cudaFree(h->d_bound);
    cudaFree(h->d_model);
    cudaFree(h->d_res_stage);
    cudaFree(h->d_sd_stage);
    if (h->s_h2d) cudaStreamDestroy(h->s_h2d);
    if (h->s_d2h) cudaStreamDestroy(h->s_d2h);
    for (cudaEvent_t e : h->ev) cudaEventDestroy(e);
  }
  if (!h) return RBT_ERR_ARG;
  cudaSetDevice(h->device);
  cudaFree(h->d_ctrl);
  for (int q = 0; q <= RBT_BUF_XDIR; ++q) {
    double** slot = buf_slot(h, q);
    if (slot) cudaFree(h->own[q] ? h->own[q] : *slot);  // never free a caller-owned buffer
  }
  cudaFree(h->d_info);
  cudaFree(h->d_arrivals);
  cudaFree(h->d_struct);
  cudaFree(h->d_timeline);
  cudaFree(h->d_steps);
  cudaFree(h->d_ones);
  cudaFree(h->d_step_pack);
  cudaFree(h->d_ls_alphas); cudaFree(h->d_ls_trial); cudaFree(h->d_ls_stage_barrier); cudaFree(h->d_ls_barrier);
  cudaFree(h->d_ls_in); cudaFree(h->d_ls_filt); cudaFree(h->d_ls_step); cudaFree(h->d_ls_nfilt); cudaFree(h->d_ls_k);
  cudaFree(h->d_stage_perf);
  cudaFree(h->d_perf);
  cudaFree(h->d_x0in);
  cudaFree(h->d_tp_elem); cudaFree(h->d_tp_scan[0]); cudaFree(h->d_tp_scan[1]); cudaFree(h->d_tp_fmap); cudaFree(h->d_tp_dx);
  cudaFree(h->d_tp_fail);
  delete h;
  return RBT_OK;
}

int rbt_set_schedule(rbt_handle* h, const rbt_stage_ctrl* ctrl, int n_grid, double max_dts0) {
  if (!h || !ctrl) return RBT_ERR_ARG;
  if (n_grid < 2 || n_grid > h->n_grid_max) {
    h->err = "[rbt_set_schedule] invalid argument: n_grid must be in [2, n_grid_max]";
    return RBT_ERR_ARG;
  }
  if (!(max_dts0 > 0)) {
    h->err = "[rbt_set_schedule] invalid argument: max_dts0 must be positive";
    return RBT_ERR_ARG;
  }
  for (int i = 0; i < n_grid; ++i) {
    const rbt_stage_ctrl& c = ctrl[i];
    const bool last = (i == n_grid - 1);
    if ((c.type == RBT_TERMINAL) != last || c.type < 0 || c.type > 3 || c.ns < 0 || c.ns > h->dims.ns_max ||
        (c.type == RBT_IMPACT && (i == 0 || last)) || (c.type == RBT_LIFT && i == 0)) {
      h->err = "[rbt_set_schedule] invalid argument: inconsistent stage control table at grid " + std::to_string(i);
      return RBT_ERR_ARG;
    }
    // contact bookkeeping: the stage kernels index fixed-size shared arrays with nv + nf and use popc(contact_mask) offsets
    // into the stacked force block, so a table that lies about either is rejected here, not discovered on the device
    const int nf_max = 3 * RBT_MAX_CONTACTS;
    if (c.nf < 0 || c.nf > nf_max || c.nf % 3 != 0 || c.contact_mask < 0 || c.contact_mask >= (1 << RBT_MAX_CONTACTS) ||
        3 * __builtin_popcount((unsigned)c.contact_mask) != c.nf || c.ngrids_in_phase < 0 || !(c.dt >= 0.0) ||
        !(c.dt < 1.0e300) || (c.sto != 0 && c.sto != 1) || (c.sto_next != 0 && c.sto_next != 1) || c.ineq_gate < 0 ||
        c.ineq_gate > 2) {
      h->err = "[rbt_set_schedule] invalid argument: grid " + std::to_string(i) +
               ": need 0 <= nf <= 12, nf % 3 == 0, 3 * popcount(contact_mask) == nf, ngrids_in_phase >= 0, finite dt >= 0, "
               "ineq_gate in {0, 1, 2}";
      return RBT_ERR_ARG;
    }
    if (c.type == RBT_IMPACT && c.ns != 0) {
      h->err = "[rbt_set_schedule] invalid argument: an impact grid carries no switching constraint (grid " + std::to_string(i) + ")";
      return RBT_ERR_ARG;
    }
  }
  if (check_contacts(h, ctrl, n_grid) != RBT_OK) return RBT_ERR_ARG;
  RBT_CUDA(h, cudaSetDevice(h->device));
  RBT_CUDA(h, cudaMemcpy(h->d_ctrl, ctrl, sizeof(rbt_stage_ctrl) * n_grid, cudaMemcpyHostToDevice));
  // stage-conditional outputs (M, STO terms, policies) must not leak from a previous schedule
  RBT_CUDA(h, cudaMemset(h->d_ric, 0, size_t(h->batch) * n_grid * h->L.r_stride * 8));
  RBT_CUDA(h, cudaMemset(h->d_dir, 0, size_t(h->batch) * n_grid * h->L.d_stride * 8));
  h->n_grid = n_grid;
  h->max_dts0 = max_dts0;
  h->ctrl.assign(ctrl, ctrl + n_grid);
  h->wire_dirty = true;
  return RBT_OK;
}

static double* buf_ptr(rbt_handle* h, int which) {
  switch (which) {
    case RBT_BUF_KKT: return h->d_kkt;
    case RBT_BUF_RIC: return h->d_ric;
    case RBT_BUF_FACT: return h->d_fact;
    case RBT_BUF_DIR: return h->d_dir;
    case RBT_BUF_DX0: return h->d_dx0;
    case RBT_BUF_LIN: return h->d_lin;
    case RBT_BUF_CON: return h->d_con;
    case RBT_BUF_EXP: return h->d_ex;
    case RBT_BUF_SOL: return h->d_sol;
    case RBT_BUF_XDIR: return h->d_xd;
    case RBT_BUF_STEPS: return h->d_steps;
    case RBT_BUF_PERF: return h->d_perf;
    default: return nullptr;
  }
}

long long rbt_buf_doubles(rbt_handle* h, int which) {
  if (!h) return -1;
  const long long per = (long long)h->batch * h->n_grid;
  if (which >= RBT_BUF_LIN && !h->stage_ready) return -1;
  switch (which) {
    case RBT_BUF_LIN: return per * h->S.l_stride;
    case RBT_BUF_CON: return per * h->S.c_stride;
    case RBT_BUF_EXP: return per * h->S.e_stride;
    case RBT_BUF_SOL: return per * h->S.s_stride;
    case RBT_BUF_XDIR: return per * h->S.x_stride;
    case RBT_BUF_STEPS: return 2LL * h->batch;
    case RBT_BUF_PERF: return 8LL * h->batch;
    case RBT_BUF_KKT: return per * h->L.k_stride;
    case RBT_BUF_RIC: return per * h->L.r_stride;
    case RBT_BUF_FACT: return per * h->L.f_stride;
    case RBT_BUF_DIR: return per * h->L.d_stride;
    case RBT_BUF_DX0: return (long long)h->batch * h->L.nx;
    default: return -1;
  }
}

double* rbt_dev_ptr(rbt_handle* h, int which) { return h ? buf_ptr(h, which) : nullptr; }

static double** buf_slot(rbt_handle* h, int which) {
  switch (which) {
    case RBT_BUF_KKT: return &h->d_kkt;
    case RBT_BUF_RIC: return &h->d_ric;
    case RBT_BUF_FACT: return &h->d_fact;
    case RBT_BUF_DIR: return &h->d_dir;
    case RBT_BUF_DX0: return &h->d_dx0;
    case RBT_BUF_LIN: return &h->d_lin;
    case RBT_BUF_CON: return &h->d_con;
    case RBT_BUF_EXP: return &h->d_ex;
    case RBT_BUF_SOL: return &h->d_sol;
    case RBT_BUF_XDIR: return &h->d_xd;
    default: return nullptr;
  }
}

int rbt_bind_buffer(rbt_handle* h, int which, double* dev) {
  if (!h) return RBT_ERR_ARG;
  double** slot = buf_slot(h, which);
  if (!slot || (which >= RBT_BUF_LIN && !h->stage_ready)) return RBT_ERR_ARG;
  if (!h->own[which]) h->own[which] = *slot;  // remember the handle's own allocation the first time it is replaced
  double* q = dev ? dev : h->own[which];
  if ((reinterpret_cast<uintptr_t>(q) & 15u) != 0) {
    h->err = "[rbt_bind_buffer] invalid argument: device buffer must be 16-byte aligned";
    return RBT_ERR_ARG;
  }
  *slot = q;
  return RBT_OK;
}

static long long stage_xfer(rbt_handle* h, int which, bool up, const double* host_c, double* host_m, int b0, int nb,
                            cudaStream_t st, bool do_copy, int* rc_out);
enum { RBT_XFER_WIRE = 100, RBT_XFER_SWITCHING = 101, RBT_XFER_RES = 102, RBT_XFER_SD = 103 };
// the STO section of the linearization records is read on switching-time stages only (riccati_backward.cuh: cs.sto)
static int ctrl_has_sto(const rbt_stage_ctrl* ctrl, int n_grid) {
  for (int i = 0; i < n_grid; ++i)
    if (ctrl[i].sto || ctrl[i].sto_next) return 1;
  return 0;
}
// wire layouts of all grid points of a schedule; returns the OCP stride in doubles
static long long make_wire_layouts(const rbt_stage_layout& S, const rbt_stage_ctrl* ctrl, int n_grid, int cost_structure,
                                   std::vector<rbt_wire_layout>& out) {
  const int with_sto = ctrl_has_sto(ctrl, n_grid);
  out.resize(n_grid);
  long long off = 0;
  for (int i = 0; i < n_grid; ++i) {
    rbt_make_wire_layout(&S, &ctrl[i], with_sto, cost_structure, &out[i]);
    out[i].ocp_off = int(off);
    off += out[i].w_doubles;
  }
  return off;
}
static int ensure_wire_layouts(rbt_handle* h) {  // rebuilt only when the schedule or the cost structure changed
  if (!h->wire_dirty && h->d_W) return RBT_OK;
  h->w_ocp = make_wire_layouts(h->S, h->ctrl.data(), h->n_grid, h->cost_structure, h->Wv);
  if (!h->d_W) RBT_CUDA(h, cudaMalloc(&h->d_W, size_t(h->n_grid_max) * sizeof(rbt_wire_layout)));
  RBT_CUDA(h, cudaMemcpy(h->d_W, h->Wv.data(), size_t(h->n_grid) * sizeof(rbt_wire_layout), cudaMemcpyHostToDevice));
  h->wire_dirty = false;
  return RBT_OK;
}

// KKT upload plan: one strided copy of the core section [Fxx|Fvu|Fx|lx|lu|Qxx|Qxu|Quu] of every record (record padding and
// unused switching/STO sections never cross PCIe), plus one strided copy per stage that carries extras.
static long long kkt_upload(rbt_handle* h, const double* host, cudaStream_t st, bool do_copy, int* rc_out) {
  const rbt_layout& L = h->L;
  const size_t pitch = size_t(L.k_stride) * 8;
  int n_extra = 0;
  for (const auto& c : h->ctrl) n_extra += (c.ns > 0 || c.sto) ? 1 : 0;
  const bool wide = n_extra * 2 > h->n_grid;  // most stages carry extras (STO horizons): copy core+extras in one go
  const size_t width = size_t(wide ? L.k_core_size + L.k_extra_size : L.k_core_size) * 8;
  const size_t rows = size_t(h->batch) * h->n_grid;
  long long bytes = (long long)(width * rows);
  if (do_copy && cudaMemcpy2DAsync(h->d_kkt, pitch, host, pitch, width, rows, cudaMemcpyHostToDevice, st) != cudaSuccess) {
    *rc_out = RBT_ERR_CUDA;
    return 0;
  }
  if (!wide) {
    const size_t opitch = pitch * h->n_grid;
    for (int i = 0; i < h->n_grid; ++i) {
      const rbt_stage_ctrl& c = h->ctrl[i];
      if (!(c.ns > 0 || c.sto)) continue;
      const size_t off = size_t(i) * L.k_stride + L.k_Phix;
      bytes += (long long)(size_t(L.k_extra_size) * 8 * h->batch);
      if (do_copy && cudaMemcpy2DAsync(h->d_kkt + off, opitch, host + off, opitch, size_t(L.k_extra_size) * 8, h->batch,
                                       cudaMemcpyHostToDevice, st) != cudaSuccess) {
        *rc_out = RBT_ERR_CUDA;
        return 0;
      }
    }
  }
  return bytes;
}

long long rbt_upload_bytes(rbt_handle* h, int which) {
  if (!h || h->n_grid == 0) return -1;
  int rc = RBT_OK;
  if (which == RBT_BUF_DX0) return rbt_buf_doubles(h, which) * 8;
  if (which == RBT_BUF_LIN || which == RBT_BUF_CON || which == RBT_BUF_SOL)
    return h->stage_ready ? stage_xfer(h, which, true, nullptr, nullptr, 0, h->batch, nullptr, false, &rc) : -1;
  if (which != RBT_BUF_KKT) return -1;
  return kkt_upload(h, nullptr, nullptr, false, &rc);
}

int rbt_upload(rbt_handle* h, int which, const double* host, void* stream) {
  if (!h || !host) return RBT_ERR_ARG;
  if (which != RBT_BUF_KKT && which != RBT_BUF_DX0 && which != RBT_BUF_LIN && which != RBT_BUF_CON && which != RBT_BUF_SOL)
    return RBT_ERR_ARG;
  if (which >= RBT_BUF_LIN && !h->stage_ready) return RBT_ERR_STATE;
  if (h->n_grid == 0) return RBT_ERR_STATE;
  RBT_CUDA(h, cudaSetDevice(h->device));
  if (which == RBT_BUF_KKT) {
    int rc = RBT_OK;
    h->kkt_from_condense = false;
    kkt_upload(h, host, (cudaStream_t)stream, true, &rc);
    if (rc != RBT_OK) {
      h->err = std::string("rbt_upload(KKT): ") + cudaGetErrorString(cudaGetLastError());
      return rc;
    }
    return RBT_OK;
  }
  if (which != RBT_BUF_DX0) {  // trimmed strided copies (see stage_xfer)
    int rc = RBT_OK;
    stage_xfer(h, which, true, host, nullptr, 0, h->batch, (cudaStream_t)stream, true, &rc);
    if (rc != RBT_OK) {
      h->err = std::string("rbt_upload: ") + cudaGetErrorString(cudaGetLastError());
      return rc;
    }
    return RBT_OK;
  }
  RBT_CUDA(h, cudaMemcpyAsync(buf_ptr(h, which), host, size_t(rbt_buf_doubles(h, which)) * 8, cudaMemcpyHostToDevice,
                              (cudaStream_t)stream));
  return RBT_OK;
}

int rbt_download(rbt_handle* h, int which, double* host, void* stream) {
  if (!h || !host || !buf_ptr(h, which)) return RBT_ERR_ARG;
  if (h->n_grid == 0) return RBT_ERR_STATE;
  RBT_CUDA(h, cudaSetDevice(h->device));
  RBT_CUDA(h, cudaMemcpyAsync(host, buf_ptr(h, which), size_t(rbt_buf_doubles(h, which)) * 8, cudaMemcpyDeviceToHost,
                              (cudaStream_t)stream));
  return RBT_OK;
}

int rbt_download_info(rbt_handle* h, int* host_flags, void* stream) {
  if (!h || !host_flags) return RBT_ERR_ARG;
  RBT_CUDA(h, cudaSetDevice(h->device));
  RBT_CUDA(h, cudaMemcpyAsync(host_flags, h->d_info, size_t(h->batch) * sizeof(int), cudaMemcpyDeviceToHost,
                              (cudaStream_t)stream));
  return RBT_OK;
}

int rbt_check_info(rbt_handle* h, int* first_bad, void* stream) {
  if (!h) return RBT_ERR_ARG;
  RBT_CUDA(h, cudaSetDevice(h->device));
  std::vector<int> flags(size_t(h->batch), 0);
  RBT_CUDA(h, cudaMemcpyAsync(flags.data(), h->d_info, flags.size() * sizeof(int), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  RBT_CUDA(h, cudaStreamSynchronize((cudaStream_t)stream));
  if (first_bad) *first_bad = -1;
  for (int b = 0; b < h->batch; ++b)
    if (flags[size_t(b)]) {
      if (first_bad) *first_bad = b;
      h->err = "numerical failure: OCP " + std::to_string(b) + " flag " + std::to_string(flags[size_t(b)]) +
               " (1: Quu + B^T P B not positive definite, 2: switching-constraint Schur complement, 4: M, 8: J M^-1 J^T in the condensing)";
      return RBT_ERR_NUMERIC;
    }
  return RBT_OK;
}

// ---- time-parallel sweeps (riccati_time_parallel.cuh) ------------------------------------------------------------------
// Segment count of the next sweep: 1 (serial) on any schedule with switching-time optimisation, whose phase transitions are
// serial; otherwise the request of rbt_set_time_segments (clamped to N), or the automatic choice from the HANDLE's batch (not
// the chunk a pipelined host path works on), so one handle always takes the same path at every chunk size.
static int tp_auto_segments(int batch, int n_sm, int N) {
  // Serial everywhere: on an H100 SXM (BASELINE.md section 6, tools/time_parallel_latency.py) the segmented sweeps were
  // faster at no batch size from 1 to 1024 and no segment count from 2 to N (at batch 1 the best, S = 23, ties the serial
  // sweeps).  Kept as the one place where a faster combine would enable them.
  (void)batch; (void)n_sm; (void)N;
  return 1;
}

static int tp_segments(const rbt_handle* h) {
  const int N = h->n_grid - 1;
  if (N < 2 || ctrl_has_sto(h->ctrl.data(), h->n_grid)) return 1;
  if (h->tsegs == 1) return 1;
  if (h->tsegs > 1) return std::min(h->tsegs, N);
  return std::min(tp_auto_segments(h->batch, h->n_sm, N), N);
}

int rbt_set_time_segments(rbt_handle* h, int segments) {
  if (!h || segments < 0) return RBT_ERR_ARG;
  if (segments > 1) {
    if (segments > h->n_grid - 1) {
      h->err = "[rbt_set_time_segments] invalid argument: more segments than stages (set the schedule first)";
      return RBT_ERR_ARG;
    }
    if (ctrl_has_sto(h->ctrl.data(), h->n_grid)) {
      h->err = "[rbt_set_time_segments] invalid argument: a schedule with switching-time optimisation is swept serially";
      return RBT_ERR_ARG;
    }
  }
  h->tsegs = segments;
  return RBT_OK;
}

static int tp_ensure(rbt_handle* h, int S) {
  const size_t esz = rbt::TpElem<2 * 18>::SIZE;  // every compiled instance has nx = 36
  if (h->L.nx != 36) {
    h->err = "internal: time-parallel element size";
    return RBT_ERR_STATE;
  }
  if (!h->d_tp_elem) {
    RBT_CUDA(h, cudaMalloc(&h->d_tp_elem, size_t(h->batch) * h->n_grid_max * esz * 8));
    RBT_CUDA(h, cudaMalloc(&h->d_tp_fail, size_t(h->batch) * sizeof(int)));
    RBT_CUDA(h, cudaMemset(h->d_tp_fail, 0, size_t(h->batch) * sizeof(int)));
  }
  if (S > h->tp_cap) {
    for (int q = 0; q < 2; ++q) {
      cudaFree(h->d_tp_scan[q]);
      h->d_tp_scan[q] = nullptr;
      RBT_CUDA(h, cudaMalloc(&h->d_tp_scan[q], size_t(h->batch) * (S + 1) * esz * 8));
    }
    cudaFree(h->d_tp_fmap);
    cudaFree(h->d_tp_dx);
    h->d_tp_fmap = h->d_tp_dx = nullptr;
    RBT_CUDA(h, cudaMalloc(&h->d_tp_fmap, size_t(h->batch) * S * (h->L.nx * h->L.nx + h->L.nx) * 8));
    RBT_CUDA(h, cudaMalloc(&h->d_tp_dx, size_t(h->batch) * S * h->L.nx * 8));
    h->tp_cap = S;
  }
  return RBT_OK;
}

static rbt::TpParams tp_params(rbt_handle* h, int S) {
  rbt::TpParams q{};
  const int b0 = win_b0(h), nb = win_nb(h);
  const size_t go = size_t(b0) * h->n_grid;
  const size_t esz = rbt::TpElem<2 * 18>::SIZE;
  q.L = h->L;
  q.ctrl = h->d_ctrl;
  q.n_grid = h->n_grid;
  q.batch = nb;
  q.segs = S;
  q.kkt = h->d_kkt + go * h->L.k_stride;
  q.ric = h->d_ric + go * h->L.r_stride;
  q.elem = h->d_tp_elem + go * esz;
  q.fmap = h->d_tp_fmap + size_t(b0) * S * (h->L.nx * h->L.nx + h->L.nx);
  q.dxseed = h->d_tp_dx + size_t(b0) * S * h->L.nx;
  q.dx0 = h->d_dx0 + size_t(b0) * h->L.nx;
  q.fail = h->d_tp_fail + b0;
  return q;
}

// Elements, in-segment reduction and suffix scan: returns (in h->tp_seeds) the scan buffer whose entry j + 1 is (P, s) at hi_j.
template <int NV, int NU, int NS>
static int tp_backward_boundaries(rbt_handle* h, int S, cudaStream_t st) {
  constexpr int NX = 2 * NV;
  using CC = rbt::TpCombCfg<NX>;
  const size_t esz = rbt::TpElem<NX>::SIZE;
  if (!h->attr_tp) {
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::tp_combine_kernel<NX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CC::SMEM_BYTES));
    h->attr_tp = true;
  }
  const int b0 = win_b0(h), nb = win_nb(h), N = h->n_grid - 1;
  rbt::TpParams q = tp_params(h, S);
  RBT_CUDA(h, cudaMemsetAsync(h->d_tp_fail + b0, 0, size_t(nb) * sizeof(int), st));
  rbt::tp_element_kernel<NV, NU, NS><<<nb * h->n_grid, rbt::TpElemCfg<NV, NU, NS>::NT, 0, st>>>(q);
  h->launches += 1;
  int lmax = 0;
  for (int j = 0; j < S; ++j) lmax = std::max(lmax, rbt::tp_seg_lo(j + 1, N, S) - rbt::tp_seg_lo(j, N, S));
  q.gather = -1;
  for (int d = 1; d < lmax; d *= 2) {  // tree reduction inside every segment, in place
    q.d = d;
    q.pairs = (lmax + 2 * d - 1) / (2 * d);
    rbt::tp_combine_kernel<NX><<<nb * S * q.pairs, CC::NT, CC::SMEM_BYTES, st>>>(q);
    h->launches += 1;
  }
  int cur = 0;
  q.gather = 1;
  for (int d = 1; d < S + 1; d *= 2) {  // suffix scan over the aggregates and the terminal element
    q.d = d;
    q.scan_in = h->d_tp_scan[cur ^ 1] + size_t(b0) * (S + 1) * esz;
    q.scan_out = h->d_tp_scan[cur] + size_t(b0) * (S + 1) * esz;
    rbt::tp_combine_kernel<NX><<<nb * (S + 1), CC::NT, CC::SMEM_BYTES, st>>>(q);
    h->launches += 1;
    q.gather = 0;
    cur ^= 1;
  }
  h->tp_seeds = h->d_tp_scan[cur ^ 1];
  RBT_CUDA(h, cudaGetLastError());
  return RBT_OK;
}

template <int NV, int NU, int NS>
static int launch_backward(rbt_handle* h, int write_fact, cudaStream_t st) {
  constexpr int NP = 6;
  using C = rbt::BwdCfg<NV, NU, NS, NP>;
  if (C::STAGE != h->L.k_stage_size || C::EXTRA != h->L.k_extra_size) {
    h->err = "internal: shared-memory staging size does not match rbt_layout";
    return RBT_ERR_STATE;
  }
  const int S = tp_segments(h);
  auto kern_s = S > 1 ? rbt::riccati_backward_kernel<NV, NU, NS, NP, true, true>   // Fqq = I, Fqv = dt I outside the floating-base blocks
                      : rbt::riccati_backward_kernel<NV, NU, NS, NP, true>;
  auto kern_g = S > 1 ? rbt::riccati_backward_kernel<NV, NU, NS, NP, false, true>  // any Fxx
                      : rbt::riccati_backward_kernel<NV, NU, NS, NP, false>;
  if (!h->attr_bwd) {  // the attribute is per device: tracked per handle (a handle lives on one device)
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::riccati_backward_kernel<NV, NU, NS, NP, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::riccati_backward_kernel<NV, NU, NS, NP, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::riccati_backward_kernel<NV, NU, NS, NP, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::riccati_backward_kernel<NV, NU, NS, NP, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    h->attr_bwd = true;
  }
  rbt::BwdParams p;
  p.L = h->L;
  p.ctrl = h->d_ctrl;
  const int b0 = win_b0(h), nb = win_nb(h);
  const size_t go = size_t(b0) * h->n_grid;
  p.n_grid = h->n_grid;
  p.batch = nb;
  p.max_dts0 = h->max_dts0;
  p.kkt = h->d_kkt + go * h->L.k_stride;
  p.ric = h->d_ric + go * h->L.r_stride;
  p.fact = write_fact ? h->d_fact + go * h->L.f_stride : nullptr;
  p.info = h->d_info + b0;
  p.sm_arrivals = h->d_arrivals;
  p.stagger_ns = h->stagger_ns;
  p.timeline = h->d_timeline;
  p.timeline_cta = h->timeline_cta;
  p.struct_flag = nullptr;
  p.segs = S;
  p.seeds = nullptr;
  p.tp_fail = nullptr;
  const int grid = nb * S;
  if (S > 1) {
    int rc = tp_ensure(h, S);
    if (!rc) rc = tp_backward_boundaries<NV, NU, NS>(h, S, st);
    if (rc) return rc;
    p.seeds = h->tp_seeds + size_t(b0) * (S + 1) * rbt::TpElem<2 * NV>::SIZE;
    p.tp_fail = h->d_tp_fail + b0;
  }
  if (!h->keep_info) RBT_CUDA(h, cudaMemsetAsync(h->d_info + b0, 0, size_t(nb) * sizeof(int), st));
  h->keep_info = false;
  if (h->stagger_ns > 0) RBT_CUDA(h, cudaMemsetAsync(h->d_arrivals, 0, 1024 * sizeof(int), st));
  // Which instance: the condensing kernel writes Fqq = I, Fqv = dt I outside the floating-base blocks by construction
  // (state_equation.cpp:52-55,68-87), a caller can declare it (rbt_set_fxx_structure), otherwise (RBT_FXX_AUTO) the records are
  // inspected on the device and BOTH instances are launched -- the one the flag does not select returns at once.
  const bool known_struct = h->kkt_from_condense || h->fxx_mode == RBT_FXX_MECHANICAL;
  h->kkt_from_condense = false;
  if (known_struct) {
    kern_s<<<grid, C::NTHREADS, C::SMEM_BYTES, st>>>(p);
    h->launches += 1;
  } else if (h->fxx_mode == RBT_FXX_GENERAL) {
    kern_g<<<grid, C::NTHREADS, C::SMEM_BYTES, st>>>(p);
    h->launches += 1;
  } else {
    RBT_CUDA(h, cudaMemsetAsync(h->d_struct, 0, 2 * sizeof(int), st));
    rbt::check_fxx_structure_kernel<NV, NP><<<(nb * (h->n_grid - 1) + 7) / 8, 256, 0, st>>>(p, h->d_struct);
    p.struct_flag = h->d_struct;
    kern_s<<<grid, C::NTHREADS, C::SMEM_BYTES, st>>>(p);
    kern_g<<<grid, C::NTHREADS, C::SMEM_BYTES, st>>>(p);
    h->launches += 3;
  }
  RBT_CUDA(h, cudaGetLastError());
  return RBT_OK;
}

int rbt_set_fxx_structure(rbt_handle* h, int mode) {
  if (!h || (mode != RBT_FXX_AUTO && mode != RBT_FXX_MECHANICAL && mode != RBT_FXX_GENERAL)) return RBT_ERR_ARG;
  h->fxx_mode = mode;
  return RBT_OK;
}

template <int NV, int NU, int NS>
static int launch_forward(rbt_handle* h, cudaStream_t st) {
  using C = rbt::FwdCfg<NV, NU, NS>;
  const int S = tp_segments(h);
  auto kern = S > 1 ? rbt::riccati_forward_kernel<NV, NU, NS, true> : rbt::riccati_forward_kernel<NV, NU, NS>;
  if (!h->attr_fwd) {
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::riccati_forward_kernel<NV, NU, NS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::riccati_forward_kernel<NV, NU, NS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::tp_fwd_compose_kernel<NV, NU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)rbt::TpFwdCfg<NV, NU>::SMEM_BYTES));
    h->attr_fwd = true;
  }
  rbt::FwdParams p;
  p.L = h->L;
  p.ctrl = h->d_ctrl;
  const int b0 = win_b0(h), nb = win_nb(h);
  const size_t go = size_t(b0) * h->n_grid;
  p.n_grid = h->n_grid;
  p.batch = nb;
  p.kkt = h->d_kkt + go * h->L.k_stride;
  p.ric = h->d_ric + go * h->L.r_stride;
  p.dx0 = h->d_dx0 + size_t(b0) * h->L.nx;
  p.dir = h->d_dir + go * h->L.d_stride;
  p.segs = S;
  p.dxseed = nullptr;
  p.tp_fail = nullptr;
  if (S > 1) {
    // the backward sweep of this handle ran segmented too (same rule, same handle): its failure flags are current
    if (int rc = tp_ensure(h, S)) return rc;
    rbt::TpParams q = tp_params(h, S);
    rbt::tp_fwd_compose_kernel<NV, NU><<<nb * (S - 1), rbt::TpFwdCfg<NV, NU>::NT, rbt::TpFwdCfg<NV, NU>::SMEM_BYTES, st>>>(q);
    rbt::tp_fwd_boundary_kernel<2 * NV><<<nb, 64, 0, st>>>(q);
    h->launches += 2;
    p.dxseed = q.dxseed;
    p.tp_fail = q.fail;
  }
  kern<<<nb * S, C::NTHREADS, C::SMEM_BYTES, st>>>(p);
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

int rbt_riccati_backward(rbt_handle* h, int write_fact, void* stream) {
  if (!h) return RBT_ERR_ARG;
  if (h->n_grid == 0) {
    h->err = "[rbt_riccati_backward] no schedule set";
    return RBT_ERR_STATE;
  }
  RBT_CUDA(h, cudaSetDevice(h->device));
#define X(NV, NU, NS) \
  if (h->dims.nv == NV && h->dims.nu == NU && h->dims.ns_max == NS) return launch_backward<NV, NU, NS>(h, write_fact, (cudaStream_t)stream);
  RBT_INSTANCES(X)
#undef X
  return RBT_ERR_ARG;
}

int rbt_riccati_forward(rbt_handle* h, void* stream) {
  if (!h) return RBT_ERR_ARG;
  if (h->n_grid == 0) {
    h->err = "[rbt_riccati_forward] no schedule set";
    return RBT_ERR_STATE;
  }
  RBT_CUDA(h, cudaSetDevice(h->device));
#define X(NV, NU, NS) \
  if (h->dims.nv == NV && h->dims.nu == NU && h->dims.ns_max == NS) return launch_forward<NV, NU, NS>(h, (cudaStream_t)stream);
  RBT_INSTANCES(X)
#undef X
  return RBT_ERR_ARG;
}

// ---- stage layer ---------------------------------------------------------------------------------------------------
int rbt_stage_layout_get(const rbt_stage_dims* sdims, const char* field) {
  if (!sdims || !field) return -1;
  rbt_stage_layout S;
  rbt_make_stage_layout(sdims, &S);
  return rbt_stage_layout_field(&S, field);
}

int rbt_stage_setup(rbt_handle* h, const rbt_stage_dims* sd, const rbt_constraint_table* table) {
  if (!h || !sd || !table) return RBT_ERR_ARG;
  if (sd->nv != h->dims.nv || sd->nu != h->dims.nu || sd->ns_max != h->dims.ns_max || sd->n_passive != h->dims.n_passive ||
      sd->n_passive != sd->nv - sd->nu /* dim_passive = dimv - dimu (robot.cpp): compiled into the stage kernels */ ||
      sd->nf_max != 12 || table->n_box != sd->n_box || table->n_contacts != sd->n_contacts || sd->n_box > RBT_MAX_BOX_ROWS ||
      sd->n_contacts > RBT_MAX_CONTACTS || !(table->barrier > 0) || !(table->fraction_to_boundary > 0) ||
      !(table->fraction_to_boundary <= 1)) {
    h->err = "[rbt_stage_setup] invalid argument: stage dims / constraint table inconsistent with the handle";
    return RBT_ERR_ARG;
  }
  for (int r = 0; r < table->n_box; ++r) {
    const rbt_box_row& b = table->box[r];
    const int lim = (b.var == RBT_VAR_U) ? sd->nu : sd->nv;
    if (b.var < 0 || b.var > 3 || b.idx < 0 || b.idx >= lim || (b.sign != 1 && b.sign != -1)) {
      h->err = "[rbt_stage_setup] invalid argument: bad box row " + std::to_string(r);
      return RBT_ERR_ARG;
    }
  }
  {
    if (3 * sd->nv + sd->nu > RBT_MAX_TARGETS) {
      h->err = "[rbt_stage_setup] invalid argument: too many limit targets";
      return RBT_ERR_ARG;
    }
    std::vector<int> cnt(RBT_MAX_TARGETS, 0);
    for (int r = 0; r < table->n_box; ++r) {
      const rbt_box_row& b = table->box[r];
      const int t = (b.var == RBT_VAR_U) ? 3 * sd->nv + b.idx : b.var * sd->nv + b.idx;
      if (++cnt[t] > 4) {
        h->err = "[rbt_stage_setup] invalid argument: more than 4 box rows on one variable";
        return RBT_ERR_ARG;
      }
    }
  }
  if (h->stage_ready) {  // a second call would leak every stage buffer and leave stale own[] pointers behind a re-bound one
    h->err = "[rbt_stage_setup] already set up on this handle (create a new handle for another constraint table)";
    return RBT_ERR_STATE;
  }
  h->sdims = *sd;
  h->table = *table;
  h->stage_ready = true;  // (for check_contacts; reset below on failure)
  if (h->n_grid > 0 && check_contacts(h, h->ctrl.data(), h->n_grid) != RBT_OK) {
    h->stage_ready = false;
    return RBT_ERR_ARG;
  }
  h->stage_ready = false;
  rbt_make_stage_layout(sd, &h->S);
  {  // condense_kernel lands [l_D, l_Phix) and [l_ha, l_dgdq) of the record in place: the static mirror must match
    using C = rbt::CondCfg<18, 12, 12>;
    const rbt_stage_layout& S = h->S;
    const int gsz = (S.l_dgdf - S.l_dgdq) + ((15 * S.ncon + 1) & ~1);
    const int q0 = S.l_Quu - C::IN1A;  // record offset that maps onto the second in-place mirror
    const bool ok = S.l_Qxx - S.l_D == C::IN1A && S.l_Phix - S.l_Quu == C::IN1B && S.l_IDC - S.l_D == C::i_IDC &&
                    S.l_Qaa - S.l_D == C::i_Qaa && S.l_Qff - S.l_D == C::i_Qff && S.l_Qqf - S.l_D == C::i_Qqf &&
                    S.l_lx - q0 == C::i_lx && S.l_la - q0 == C::i_la && S.l_lf - q0 == C::i_lf && S.l_lu - q0 == C::i_lu &&
                    S.l_Fx - q0 == C::i_Fx && S.l_lup - q0 == C::i_lup && S.l_se3 - q0 == C::i_se3 && S.l_dgdq - S.l_ha == C::IN2 &&
                    S.l_hf - S.l_ha == C::j_hf && S.l_hx - S.l_ha == C::j_hx && S.l_hu - S.l_ha == C::j_hu &&
                    S.l_fx - S.l_ha == C::j_fx && S.l_sc - S.l_ha == C::j_sc &&
                    5 * S.ncp + gsz <= C::NVF * C::NX &&  // PDIPM staging fits in the R buffer
                    S.l_J - S.l_M == rbt::MjtjCfg<18, 12>::o_J && S.l_D - S.l_M == rbt::MjtjCfg<18, 12>::MJ;
    if (!ok) {
      h->err = "[rbt_stage_setup] invalid argument: stage layout not supported by the compiled condensing kernel";
      return RBT_ERR_ARG;
    }
  }
  if (h->S.ncp > 160 || h->S.l_stride - h->S.l_dgdq > 512) {  // shared-memory staging areas of expand_kernel
    h->err = "[rbt_stage_setup] invalid argument: more than 160 inequality rows or more than 4 friction cones";
    return RBT_ERR_ARG;
  }
  RBT_CUDA(h, cudaSetDevice(h->device));
  const size_t per = size_t(h->batch) * h->n_grid_max;
  RBT_CUDA(h, cudaMalloc(&h->d_lin, per * h->S.l_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_con, per * h->S.c_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_ex, per * h->S.e_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_sol, per * h->S.s_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_xd, per * h->S.x_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_steps, size_t(h->batch) * 2 * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_ones, size_t(h->batch) * 2 * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_stage_perf, per * 4 * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_perf, size_t(h->batch) * 8 * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_x0in, size_t(h->batch) * 2 * h->dims.nv * 8));
  {  // box rows acting on each target entry (var, idx), in ascending row order (deterministic accumulation on the device):
     // entry = (row + 1) * sign, 0 = none.  Device memory, not kernel parameters: the lanes of a warp look up different targets,
     // and a divergent constant-bank access is serialised.
    int tg[RBT_MAX_TARGETS][4] = {};
    for (int r = 0; r < h->table.n_box; ++r) {
      const rbt_box_row& b = h->table.box[r];
      const int t = (b.var == RBT_VAR_U) ? 3 * h->sdims.nv + b.idx : b.var * h->sdims.nv + b.idx;
      for (int q = 0; q < 4; ++q)
        if (tg[t][q] == 0) {
          tg[t][q] = (r + 1) * (b.sign < 0 ? -1 : 1);
          break;
        }
    }
    // ... followed by the level of every box row (2 = position, 1 = velocity, 0 = acceleration / torque): a row acts on a grid
    // point iff level + ineq_gate <= 2 (ConstraintsData::setTimeStage)
    int lvl[RBT_MAX_BOX_ROWS] = {};
    for (int r = 0; r < h->table.n_box; ++r) lvl[r] = h->table.box[r].var == RBT_VAR_Q ? 2 : (h->table.box[r].var == RBT_VAR_V ? 1 : 0);
    RBT_CUDA(h, cudaMalloc(&h->d_tgt, sizeof(tg) + sizeof(lvl)));
    RBT_CUDA(h, cudaMemcpy(h->d_tgt, tg, sizeof(tg), cudaMemcpyHostToDevice));
    RBT_CUDA(h, cudaMemcpy(h->d_tgt + RBT_MAX_TARGETS * 4, lvl, sizeof(lvl), cudaMemcpyHostToDevice));
  }
  RBT_CUDA(h, cudaMemset(h->d_perf, 0, size_t(h->batch) * 8 * 8));
  RBT_CUDA(h, cudaMemset(h->d_lin, 0, per * h->S.l_stride * 8));  // uploads skip record padding: keep it defined
  RBT_CUDA(h, cudaMemset(h->d_sol, 0, per * h->S.s_stride * 8));
  RBT_CUDA(h, cudaMemset(h->d_ex, 0, per * h->S.e_stride * 8));
  RBT_CUDA(h, cudaMemset(h->d_xd, 0, per * h->S.x_stride * 8));
  RBT_CUDA(h, cudaMemset(h->d_con, 0, per * h->S.c_stride * 8));
  std::vector<double> ones(size_t(h->batch) * 2, 1.0);
  RBT_CUDA(h, cudaMemcpy(h->d_ones, ones.data(), ones.size() * 8, cudaMemcpyHostToDevice));
  RBT_CUDA(h, cudaMemcpy(h->d_steps, ones.data(), ones.size() * 8, cudaMemcpyHostToDevice));
  h->stage_ready = true;
  return RBT_OK;
}

static rbt::StageParams make_stage_params(rbt_handle* h) {
  rbt::StageParams p;
  p.K = h->L;
  p.S = h->S;
  p.tab = h->table;
  p.ctrl = h->d_ctrl;
  const int b0 = win_b0(h);
  const size_t go = size_t(b0) * h->n_grid;
  p.n_grid = h->n_grid;
  p.batch = win_nb(h);
  p.lin = h->d_lin + go * h->S.l_stride;
  p.con = h->d_con + go * h->S.c_stride;
  p.kkt = h->d_kkt + go * h->L.k_stride;
  p.ex = h->d_ex + go * h->S.e_stride;
  p.dir = h->d_dir + go * h->L.d_stride;
  p.xd = h->d_xd + go * h->S.x_stride;
  p.sol = h->d_sol + go * h->S.s_stride;
  p.steps = h->d_steps + 2 * size_t(b0);
  p.info = h->d_info + b0;
  p.tgt = reinterpret_cast<const int4*>(h->d_tgt);
  p.row_level = h->d_tgt + RBT_MAX_TARGETS * 4;
  return p;
}

#define RBT_STAGE_CHECK(h, what)                                  \
  if (!(h)) return RBT_ERR_ARG;                                   \
  if (!(h)->stage_ready || (h)->n_grid == 0) {                    \
    (h)->err = "[" what "] stage layer not set up / no schedule"; \
    return RBT_ERR_STATE;                                         \
  }                                                               \
  RBT_CUDA(h, cudaSetDevice((h)->device));

int rbt_condense(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_condense");
  using C = rbt::CondCfg<18, 12, 12>;
  auto kern = rbt::condense_kernel<18, 12, 12>;
  if (!h->attr_cond) {
    RBT_CUDA(h, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    h->attr_cond = true;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int nb = win_nb(h);
  RBT_CUDA(h, cudaMemsetAsync(h->d_info + win_b0(h), 0, size_t(nb) * sizeof(int), st));
  rbt::mjtjinv_kernel<18, 12><<<(nb * h->n_grid + 1) / 2, 64, 0, st>>>(make_stage_params(h));  // K1: Z = [[M,J^T],[J,0]]^-1
  RBT_CUDA(h, cudaGetLastError());
  if (h->ev_condense_mid) RBT_CUDA(h, cudaEventRecord(h->ev_condense_mid, st));
  kern<<<nb * h->n_grid, C::NTHREADS, C::SMEM_BYTES, st>>>(make_stage_params(h));     // K2: condensing (DMMA)
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 2;
  h->keep_info = true;
  h->kkt_from_condense = true;
  return RBT_OK;
}

int rbt_set_condense_event(rbt_handle* h, void* cuda_event) {
  if (!h) return RBT_ERR_ARG;
  h->ev_condense_mid = (cudaEvent_t)cuda_event;
  return RBT_OK;
}

int rbt_expand_and_step_sizes(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_expand_and_step_sizes");
  cudaStream_t st = (cudaStream_t)stream;
  RBT_CUDA(h, cudaMemcpyAsync(h->d_steps + 2 * size_t(win_b0(h)), h->d_ones, size_t(win_nb(h)) * 2 * 8, cudaMemcpyDeviceToDevice, st));
  rbt::expand_kernel<18, 12, 12><<<win_nb(h) * h->n_grid, rbt::XTHR, 0, st>>>(make_stage_params(h));
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

int rbt_update(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_update");
  rbt::update_kernel<18, 12, 12><<<win_nb(h) * h->n_grid, rbt::XTHR, 0, (cudaStream_t)stream>>>(make_stage_params(h));
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

static rbt::EvalParams make_eval_params(rbt_handle* h) {
  rbt::EvalParams q;
  q.sp = make_stage_params(h);
  const int b0 = win_b0(h);
  q.stage_perf = h->d_stage_perf + size_t(b0) * h->n_grid * 4;
  q.perf = h->d_perf + size_t(b0) * 8;
  q.x0in = h->d_x0in + size_t(b0) * 2 * h->dims.nv;
  q.dx0 = h->d_dx0 + size_t(b0) * h->L.nx;
  return q;
}

int rbt_eval_kkt(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_eval_kkt");
  cudaStream_t st = (cudaStream_t)stream;
  const rbt::EvalParams q = make_eval_params(h);
  const int nb = win_nb(h);
  rbt::perf_index_kernel<<<(nb * h->n_grid + 3) / 4, 128, 0, st>>>(q);
  rbt::perf_reduce_kernel<<<(nb + 127) / 128, 128, 0, st>>>(q);
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 2;
  return RBT_OK;
}

int rbt_set_slack_and_dual_positive(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_set_slack_and_dual_positive");
  const rbt::EvalParams q = make_eval_params(h);
  const long long total = (long long)win_nb(h) * h->n_grid * h->S.ncp;
  rbt::slack_dual_positive_kernel<<<unsigned((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(q);
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

int rbt_set_joint_limits(rbt_handle* h, const double* bound_host) {
  if (!h || !bound_host) return RBT_ERR_ARG;
  if (!h->stage_ready) {
    h->err = "[rbt_set_joint_limits] stage layer not set up";
    return RBT_ERR_STATE;
  }
  RBT_CUDA(h, cudaSetDevice(h->device));
  if (!h->d_bound) RBT_CUDA(h, cudaMalloc(&h->d_bound, sizeof(double) * RBT_MAX_BOX_ROWS));
  RBT_CUDA(h, cudaMemcpy(h->d_bound, bound_host, sizeof(double) * h->table.n_box, cudaMemcpyHostToDevice));
  return RBT_OK;
}

int rbt_linearize_joint_limits(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_linearize_joint_limits");
  if (!h->d_bound) {
    h->err = "[rbt_linearize_joint_limits] call rbt_set_joint_limits first";
    return RBT_ERR_STATE;
  }
  const rbt::EvalParams q = make_eval_params(h);
  const long long total = (long long)win_nb(h) * h->n_grid * (3 * h->S.nv + h->S.nu);
  rbt::linearize_joint_limits_kernel<<<unsigned((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(q, h->d_bound);
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

int rbt_set_robot_model(rbt_handle* h, const rbt_robot_model* m) {
  if (!h || !m) return RBT_ERR_ARG;
  if (!h->stage_ready) {
    h->err = "[rbt_set_robot_model] stage layer not set up";
    return RBT_ERR_STATE;
  }
  auto bad = [&](const std::string& what) {
    h->err = "[rbt_set_robot_model] invalid argument: " + what;
    return RBT_ERR_ARG;
  };
  if (m->nv != h->S.nv || m->n_bodies != m->nv - 5 || m->n_bodies > RBT_MAX_BODIES) return bad("nv / n_bodies disagree with the handle");
  if (m->n_contacts != h->S.ncon) return bad("n_contacts disagrees with the stage layer");
  rbt::RneaModel d = {};
  d.nb = m->n_bodies;
  d.ncon = m->n_contacts;
  for (int b = 0; b < m->n_bodies; ++b) {
    const std::string tag = "body " + std::to_string(b) + ": ";
    if (b == 0 ? m->parent[b] != -1 : (m->parent[b] < 0 || m->parent[b] >= b)) return bad(tag + "parent must come earlier in the order");
    if (!(m->mass[b] > 0.0)) return bad(tag + "mass must be positive");
    const double* I = m->inertia[b];
    double imax = 0.0;
    for (int e = 0; e < 9; ++e) imax = std::max(imax, std::fabs(I[e]));
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < i; ++j)
        if (!(std::fabs(I[i + 3 * j] - I[j + 3 * i]) <= 1e-12 * imax)) return bad(tag + "inertia is not symmetric");
    // Sylvester: leading minors of a symmetric 3x3
    const double m1 = I[0], m2 = I[0] * I[4] - I[1] * I[3];
    const double m3 = I[0] * (I[4] * I[8] - I[5] * I[7]) - I[3] * (I[1] * I[8] - I[2] * I[7]) + I[6] * (I[1] * I[5] - I[2] * I[4]);
    if (!(m1 > 0.0 && m2 > 0.0 && m3 > 0.0)) return bad(tag + "inertia is not positive definite");
    if (b > 0) {
      const double* u = m->axis[b];
      if (!(std::fabs(std::sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2]) - 1.0) <= 1e-12)) return bad(tag + "axis is not a unit vector");
    }
    d.parent[b] = m->parent[b];
    for (int e = 0; e < 3; ++e) {
      d.axis[b][e] = m->axis[b][e];
      d.p[b][e] = m->placement[b][9 + e];
      d.com[b][e] = m->com[b][e];
    }
    for (int e = 0; e < 9; ++e) {
      d.R[b][e] = m->placement[b][e];
      d.Ic[b][e] = I[e];
    }
    d.mass[b] = m->mass[b];
  }
  for (int c = 0; c < m->n_contacts; ++c) {
    if (m->contact_parent[c] < 0 || m->contact_parent[c] >= m->n_bodies) return bad("contact " + std::to_string(c) + ": no such parent body");
    d.cparent[c] = m->contact_parent[c];
    for (int e = 0; e < 9; ++e) d.cR[c][e] = m->contact_placement[c][e];
    for (int e = 0; e < 3; ++e) d.cp[c][e] = m->contact_placement[c][9 + e];
  }
  for (int e = 0; e < 3; ++e) d.gravity[e] = m->gravity[e];
  RBT_CUDA(h, cudaSetDevice(h->device));
  if (!h->d_model) RBT_CUDA(h, cudaMalloc(&h->d_model, sizeof(rbt::RneaModel)));
  RBT_CUDA(h, cudaMemcpy(h->d_model, &d, sizeof(rbt::RneaModel), cudaMemcpyHostToDevice));
  return RBT_OK;
}

int rbt_linearize_inverse_dynamics(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_linearize_inverse_dynamics");
  if (!h->d_model) {
    h->err = "[rbt_linearize_inverse_dynamics] call rbt_set_robot_model first";
    return RBT_ERR_STATE;
  }
  rbt::linearize_inverse_dynamics_kernel<18><<<win_nb(h) * h->n_grid, rbt::RneaCfg<18>::NTHR, 0, (cudaStream_t)stream>>>(
      make_stage_params(h), h->d_model);
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

int rbt_initial_state_direction(rbt_handle* h, const double* dq0_v0_host, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_initial_state_direction");
  if (!dq0_v0_host) return RBT_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  RBT_CUDA(h, cudaMemcpyAsync(h->d_x0in, dq0_v0_host, size_t(h->batch) * 2 * h->dims.nv * 8, cudaMemcpyHostToDevice, st));
  const rbt::EvalParams q = make_eval_params(h);
  const int total = win_nb(h) * h->L.nx;
  rbt::initial_state_direction_kernel<<<(total + 127) / 128, 128, 0, st>>>(q);
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

// ---- line search: trial step sizes as an extra batch axis -------------------------------------------------------------------
enum { RBT_LS_FILTER_CAP = 16 };

static int ls_ensure(rbt_handle* h, int n_trials) {
  if (n_trials <= h->ls_trials) return RBT_OK;
  cudaFree(h->d_ls_alphas); cudaFree(h->d_ls_trial); cudaFree(h->d_ls_stage_barrier); cudaFree(h->d_ls_barrier); cudaFree(h->d_ls_in);
  h->d_ls_alphas = h->d_ls_trial = h->d_ls_stage_barrier = h->d_ls_barrier = h->d_ls_in = nullptr;
  const size_t kb = size_t(n_trials) * h->batch;
  RBT_CUDA(h, cudaMalloc(&h->d_ls_alphas, kb * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_ls_barrier, kb * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_ls_stage_barrier, kb * h->n_grid_max * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_ls_trial, kb * h->n_grid_max * rbt::T_STRIDE * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_ls_in, (2 * kb + 2 * size_t(h->batch)) * 8));  // cost | viol of the trials, cost0 | viol0
  if (!h->d_ls_filt) {
    RBT_CUDA(h, cudaMalloc(&h->d_ls_filt, size_t(h->batch) * 2 * RBT_LS_FILTER_CAP * 8));
    RBT_CUDA(h, cudaMalloc(&h->d_ls_nfilt, size_t(h->batch) * sizeof(int)));
    RBT_CUDA(h, cudaMalloc(&h->d_ls_step, size_t(h->batch) * 8));
    RBT_CUDA(h, cudaMalloc(&h->d_ls_k, size_t(h->batch) * sizeof(int)));
    RBT_CUDA(h, cudaMemset(h->d_ls_nfilt, 0, size_t(h->batch) * sizeof(int)));
  }
  h->ls_trials = n_trials;
  return RBT_OK;
}

int rbt_trial_doubles(void) { return rbt::T_STRIDE; }

int rbt_line_search_trials(rbt_handle* h, int n_trials, double step_size_reduction_rate, double* alphas_host, double* barrier_host,
                           double* trial_host, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_line_search_trials");
  if (n_trials < 1 || n_trials > 64 || !(step_size_reduction_rate > 0.0 && step_size_reduction_rate < 1.0)) {
    h->err = "[rbt_line_search_trials] invalid argument: 1 <= n_trials <= 64, 0 < step_size_reduction_rate < 1";
    return RBT_ERR_ARG;
  }
  if (int rc = ls_ensure(h, n_trials)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  rbt::TrialParams q;
  q.sp = make_stage_params(h);
  q.n_trials = n_trials;
  q.rate = step_size_reduction_rate;
  q.alphas = h->d_ls_alphas;
  q.trial = h->d_ls_trial;
  q.stage_barrier = h->d_ls_stage_barrier;
  q.barrier = h->d_ls_barrier;
  const long long warps = (long long)n_trials * h->batch * h->n_grid;
  rbt::trial_solution_kernel<<<unsigned((warps + 3) / 4), 128, 0, st>>>(q);
  rbt::trial_reduce_kernel<<<(n_trials * h->batch + 127) / 128, 128, 0, st>>>(q);
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 2;
  const size_t kb = size_t(n_trials) * h->batch;
  if (alphas_host) RBT_CUDA(h, cudaMemcpyAsync(alphas_host, h->d_ls_alphas, kb * 8, cudaMemcpyDeviceToHost, st));
  if (barrier_host) RBT_CUDA(h, cudaMemcpyAsync(barrier_host, h->d_ls_barrier, kb * 8, cudaMemcpyDeviceToHost, st));
  if (trial_host) RBT_CUDA(h, cudaMemcpyAsync(trial_host, h->d_ls_trial, kb * h->n_grid * rbt::T_STRIDE * 8, cudaMemcpyDeviceToHost, st));
  return RBT_OK;
}

double* rbt_line_search_trial_dev(rbt_handle* h) { return h ? h->d_ls_trial : nullptr; }

int rbt_line_search_clear_history(rbt_handle* h, void* stream) {
  if (!h) return RBT_ERR_ARG;
  if (h->d_ls_nfilt) RBT_CUDA(h, cudaMemsetAsync(h->d_ls_nfilt, 0, size_t(h->batch) * sizeof(int), (cudaStream_t)stream));
  return RBT_OK;
}

int rbt_line_search_filter(rbt_handle* h, int n_trials, double step_size_reduction_rate, double min_step_size,
                           double filter_cost_reduction_rate, double filter_constraint_violation_reduction_rate,
                           const double* cost0_host, const double* violation0_host, const double* cost_host,
                           const double* violation_host, double* step_host, int* accepted_trial_host, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_line_search_filter");
  if (n_trials < 1 || n_trials > h->ls_trials || !cost0_host || !violation0_host || !cost_host || !violation_host ||
      !(filter_cost_reduction_rate > 0.0) || !(filter_constraint_violation_reduction_rate > 0.0)) {
    h->err = "[rbt_line_search_filter] invalid argument (call rbt_line_search_trials with at least n_trials first; the reduction "
             "rates must be positive like LineSearchFilter's, line_search_filter.cpp:15-20)";
    return RBT_ERR_ARG;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t kb = size_t(n_trials) * h->batch;
  double* d_cost = h->d_ls_in;
  double* d_viol = h->d_ls_in + size_t(h->ls_trials) * h->batch;
  double* d_c0 = h->d_ls_in + 2 * size_t(h->ls_trials) * h->batch;
  double* d_v0 = d_c0 + h->batch;
  RBT_CUDA(h, cudaMemcpyAsync(d_cost, cost_host, kb * 8, cudaMemcpyHostToDevice, st));
  RBT_CUDA(h, cudaMemcpyAsync(d_viol, violation_host, kb * 8, cudaMemcpyHostToDevice, st));
  RBT_CUDA(h, cudaMemcpyAsync(d_c0, cost0_host, size_t(h->batch) * 8, cudaMemcpyHostToDevice, st));
  RBT_CUDA(h, cudaMemcpyAsync(d_v0, violation0_host, size_t(h->batch) * 8, cudaMemcpyHostToDevice, st));
  rbt::FilterParams q;
  q.batch = h->batch; q.n_trials = n_trials; q.cap = RBT_LS_FILTER_CAP;
  q.rate = step_size_reduction_rate; q.min_step = min_step_size;
  q.cost_rate = filter_cost_reduction_rate; q.viol_rate = filter_constraint_violation_reduction_rate;
  q.steps = h->d_steps; q.cost0 = d_c0; q.viol0 = d_v0; q.cost = d_cost; q.barrier = h->d_ls_barrier; q.viol = d_viol;
  q.filt = h->d_ls_filt; q.nfilt = h->d_ls_nfilt; q.out_step = h->d_ls_step; q.out_k = h->d_ls_k;
  rbt::line_search_filter_kernel<<<(h->batch + 127) / 128, 128, 0, st>>>(q);
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  if (step_host) RBT_CUDA(h, cudaMemcpyAsync(step_host, h->d_ls_step, size_t(h->batch) * 8, cudaMemcpyDeviceToHost, st));
  if (accepted_trial_host) RBT_CUDA(h, cudaMemcpyAsync(accepted_trial_host, h->d_ls_k, size_t(h->batch) * sizeof(int), cudaMemcpyDeviceToHost, st));
  return RBT_OK;
}

// Host <-> device traffic of the stage layer, for the batch window [b0, b0 + nb).  Only what the kernels read / what
// persists crosses PCIe: record padding never does, the switching-constraint section of the linearization record only for
// the stages that carry one, of the PDIPM record slack | dual | residual go up and slack | dual come back.
static long long stage_xfer(rbt_handle* h, int which, bool up, const double* host_c, double* host_m, int b0, int nb,
                            cudaStream_t st, bool do_copy, int* rc_out) {
  const rbt_stage_layout& S = h->S;
  const size_t rows = size_t(nb) * h->n_grid, go = size_t(b0) * h->n_grid;
  long long bytes = 0;
  auto copy2d = [&](double* dev, const double* hc, double* hm, size_t off, size_t stride, size_t width, size_t pitch_rows,
                    size_t nrows) {
    bytes += (long long)(width * 8 * nrows);
    if (!do_copy || *rc_out != RBT_OK) return;
    const size_t pitch = stride * pitch_rows * 8;
    if (pitch == width * 8) {  // contiguous: one linear DMA
      cudaError_t e1 = up ? cudaMemcpyAsync(dev + off, hc + off, width * 8 * nrows, cudaMemcpyHostToDevice, st)
                          : cudaMemcpyAsync(hm + off, dev + off, width * 8 * nrows, cudaMemcpyDeviceToHost, st);
      if (e1 != cudaSuccess) *rc_out = RBT_ERR_CUDA;
      return;
    }
    cudaError_t e = up ? cudaMemcpy2DAsync(dev + off, pitch, hc + off, pitch, width * 8, nrows, cudaMemcpyHostToDevice, st)
                       : cudaMemcpy2DAsync(hm + off, pitch, dev + off, pitch, width * 8, nrows, cudaMemcpyDeviceToHost, st);
    if (e != cudaSuccess) *rc_out = RBT_ERR_CUDA;
  };
  if (which == RBT_XFER_WIRE) {  // packed wire records: contiguous
    copy2d(h->d_wire, host_c, host_m, size_t(b0) * h->w_ocp, h->w_ocp, h->w_ocp, 1, nb);
  } else if (which == RBT_XFER_SWITCHING) {  // only the switching-constraint sections of the classic record
    const size_t base = go * S.l_stride;
    for (int i = 0; i < h->n_grid; ++i)
      if (h->ctrl[i].ns > 0 && h->ctrl[i].type != RBT_IMPACT)
        copy2d(h->d_lin, host_c, host_m, base + size_t(i) * S.l_stride + S.l_Phix, S.l_stride, S.l_ha - S.l_Phix, h->n_grid, nb);
  } else if (which == RBT_BUF_LIN) {
    const size_t base = go * S.l_stride;
    const size_t tail = size_t(S.l_dgdf) + ((15 * S.ncon + 1) & ~1) - S.l_ha;
    copy2d(h->d_lin, host_c, host_m, base, S.l_stride, S.l_Phix, 1, rows);            // M .. se3
    copy2d(h->d_lin, host_c, host_m, base + S.l_ha, S.l_stride, tail, 1, rows);       // ha .. dgdf
    for (int i = 0; i < h->n_grid; ++i)
      if (h->ctrl[i].ns > 0 && h->ctrl[i].type != RBT_IMPACT)                         // Phix, Phia, p, Phit
        copy2d(h->d_lin, host_c, host_m, base + size_t(i) * S.l_stride + S.l_Phix, S.l_stride, S.l_ha - S.l_Phix, h->n_grid, nb);
  } else if (which == RBT_XFER_RES) {  // compact PDIPM residuals [batch][n_grid][ncp]: one contiguous copy into the staging buffer
    copy2d(h->d_res_stage, host_c, host_m, go * S.ncp, S.ncp, S.ncp, 1, rows);   // (unpack_wire_kernel scatters them into c_res)
  } else if (which == RBT_XFER_SD) {   // compact slack | dual [batch][n_grid][2 ncp] (packed by pack_slack_dual_kernel): contiguous
    copy2d(h->d_sd_stage, host_c, host_m, go * 2 * S.ncp, 2 * S.ncp, 2 * S.ncp, 1, rows);

  } else if (which == RBT_BUF_CON) {
    copy2d(h->d_con, host_c, host_m, go * S.c_stride + S.c_slack, S.c_stride, size_t(up ? 3 : 2) * S.ncp, 1, rows);
  } else if (which == RBT_BUF_SOL) {
    // whole records incl. the few padding doubles: ONE contiguous DMA instead of a strided 2-D copy of 1.4 KB rows (the copy
    // engine spends as long per row as on ~4 KB of payload)
    copy2d(h->d_sol, host_c, host_m, go * S.s_stride, S.s_stride, S.s_stride, 1, rows);
  } else if (which == RBT_BUF_DX0) {
    copy2d(h->d_dx0, host_c, host_m, size_t(b0) * h->L.nx, h->L.nx, h->L.nx, 1, nb);
  } else if (which == RBT_BUF_STEPS) {
    copy2d(h->d_steps, host_c, host_m, 2 * size_t(b0), 2, 2, 1, nb);
  }
  return bytes;
}

int rbt_iteration_host_bytes(rbt_handle* h, int wire, long long* h2d, long long* d2h) {
  if (!h || !h->stage_ready || h->n_grid == 0) return RBT_ERR_STATE;
  int rc = RBT_OK;
  long long up = 0, down = 0;
  h->w_ocp = make_wire_layouts(h->S, h->ctrl.data(), h->n_grid, h->cost_structure, h->Wv);
  if (wire == 2) {  // rbt_iteration_host_resident: wire records + residuals + dx0 up
    up += stage_xfer(h, RBT_XFER_WIRE, true, nullptr, nullptr, 0, h->batch, nullptr, false, &rc);
    up += stage_xfer(h, RBT_XFER_SWITCHING, true, nullptr, nullptr, 0, h->batch, nullptr, false, &rc);
    up += stage_xfer(h, RBT_XFER_RES, true, nullptr, nullptr, 0, h->batch, nullptr, false, &rc);
    up += stage_xfer(h, RBT_BUF_DX0, true, nullptr, nullptr, 0, h->batch, nullptr, false, &rc);
    for (int w : {int(RBT_BUF_SOL), int(RBT_XFER_SD), int(RBT_BUF_STEPS)}) down += stage_xfer(h, w, false, nullptr, nullptr, 0, h->batch, nullptr, false, &rc);
    if (h2d) *h2d = up;
    if (d2h) *d2h = down;
    return RBT_OK;
  }
  if (wire) {
    up += stage_xfer(h, RBT_XFER_WIRE, true, nullptr, nullptr, 0, h->batch, nullptr, false, &rc);
    up += stage_xfer(h, RBT_XFER_SWITCHING, true, nullptr, nullptr, 0, h->batch, nullptr, false, &rc);
  } else {
    up += stage_xfer(h, RBT_BUF_LIN, true, nullptr, nullptr, 0, h->batch, nullptr, false, &rc);
  }
  for (int w : {RBT_BUF_CON, RBT_BUF_SOL, RBT_BUF_DX0}) up += stage_xfer(h, w, true, nullptr, nullptr, 0, h->batch, nullptr, false, &rc);
  for (int w : {RBT_BUF_SOL, RBT_BUF_CON, RBT_BUF_STEPS}) down += stage_xfer(h, w, false, nullptr, nullptr, 0, h->batch, nullptr, false, &rc);
  if (h2d) *h2d = up;
  if (d2h) *d2h = down;
  return RBT_OK;
}

// res_host != NULL: resident mode (solution, slack and dual stay where the previous iteration left them on the device; only the
// PDIPM residuals come from the host), con_host / sol_host are not read.
static int iteration_host_impl(rbt_handle* h, const double* wire_host, const double* lin_host, const double* con_host,
                               const double* sol_host, const double* res_host, const double* dx0_host, double* sol_out,
                               double* con_out, double* steps_out, void* stream) {
  if (!h || (!lin_host && !wire_host) || !dx0_host) return RBT_ERR_ARG;
  if (!res_host && (!con_host || !sol_host)) return RBT_ERR_ARG;
  RBT_STAGE_CHECK(h, "rbt_iteration_host");
  if (wire_host) {
    int rcw = ensure_wire_layouts(h);
    if (rcw != RBT_OK) return rcw;
    bool sw = false;
    for (int i = 0; i < h->n_grid; ++i) sw = sw || (h->ctrl[i].ns > 0 && h->ctrl[i].type != RBT_IMPACT);
    if ((h->cost_structure & RBT_WIRE_DEVICE_ID) && !h->d_model) {
      h->err = "[rbt_iteration_host_wire] the wire records leave the inverse dynamics to the device: call rbt_set_robot_model first";
      return RBT_ERR_STATE;
    }
    if (sw && !lin_host) {
      h->err = "[rbt_iteration_host_wire] invalid argument: the schedule has switching-constraint stages, their sections come from lin_host_switching";
      return RBT_ERR_ARG;
    }
    if (!h->d_wire) {  // sized for the largest possible record at every grid point
      rbt_wire_layout wmax;
      rbt_stage_ctrl cmax = {};
      cmax.type = RBT_INTERMEDIATE; cmax.nf = h->S.nfm; cmax.contact_mask = (1 << h->S.ncon) - 1;
      rbt_make_wire_layout(&h->S, &cmax, 1, RBT_COST_GENERAL, &wmax);
      RBT_CUDA(h, cudaMalloc(&h->d_wire, size_t(h->batch) * h->n_grid_max * wmax.w_doubles * 8));
    }
    if (res_host && !h->d_res_stage) {
      RBT_CUDA(h, cudaMalloc(&h->d_res_stage, size_t(h->batch) * h->n_grid_max * h->S.ncp * 8));
      RBT_CUDA(h, cudaMalloc(&h->d_sd_stage, size_t(h->batch) * h->n_grid_max * 2 * h->S.ncp * 8));
    }
  }
  cudaStream_t st = (cudaStream_t)stream;
  // chunks of the batch: the upload of chunk c+1, the kernels of chunk c and the download of chunk c-1 overlap
  int n_chunks = h->batch >= 512 ? 8 : (h->batch >= 128 ? 4 : 1);
  if (const char* e = getenv("RBT_E2E_CHUNKS")) n_chunks = std::max(1, std::min(atoi(e), h->batch));
  if (!h->s_h2d) {
    RBT_CUDA(h, cudaStreamCreateWithFlags(&h->s_h2d, cudaStreamNonBlocking));
    RBT_CUDA(h, cudaStreamCreateWithFlags(&h->s_d2h, cudaStreamNonBlocking));
  }
  while ((int)h->ev.size() < 2 * n_chunks + 2) {
    cudaEvent_t e;
    RBT_CUDA(h, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    h->ev.push_back(e);
  }
  cudaEvent_t ev_entry = h->ev[2 * n_chunks], ev_exit = h->ev[2 * n_chunks + 1];
  RBT_CUDA(h, cudaEventRecord(ev_entry, st));            // device buffers may still be read by earlier work on `stream`
  RBT_CUDA(h, cudaStreamWaitEvent(h->s_h2d, ev_entry, 0));
  RBT_CUDA(h, cudaStreamWaitEvent(h->s_d2h, ev_entry, 0));
  int rc = RBT_OK;
  for (int c = 0; c < n_chunks && rc == RBT_OK; ++c) {
    const int b0 = int((long long)h->batch * c / n_chunks), b1 = int((long long)h->batch * (c + 1) / n_chunks), nb = b1 - b0;
    if (nb <= 0) continue;
    if (wire_host) {
      stage_xfer(h, RBT_XFER_WIRE, true, wire_host, nullptr, b0, nb, h->s_h2d, true, &rc);
      if (lin_host) stage_xfer(h, RBT_XFER_SWITCHING, true, lin_host, nullptr, b0, nb, h->s_h2d, true, &rc);
    } else {
      stage_xfer(h, RBT_BUF_LIN, true, lin_host, nullptr, b0, nb, h->s_h2d, true, &rc);
    }
    if (res_host) {
      stage_xfer(h, RBT_XFER_RES, true, res_host, nullptr, b0, nb, h->s_h2d, true, &rc);
    } else {
      stage_xfer(h, RBT_BUF_CON, true, con_host, nullptr, b0, nb, h->s_h2d, true, &rc);
      stage_xfer(h, RBT_BUF_SOL, true, sol_host, nullptr, b0, nb, h->s_h2d, true, &rc);
    }
    stage_xfer(h, RBT_BUF_DX0, true, dx0_host, nullptr, b0, nb, h->s_h2d, true, &rc);
    if (rc != RBT_OK) break;
    RBT_CUDA(h, cudaEventRecord(h->ev[2 * c], h->s_h2d));
    RBT_CUDA(h, cudaStreamWaitEvent(st, h->ev[2 * c], 0));
    h->cb0 = b0;
    h->cnb = nb;
    if (wire_host) {  // expand the packed records of this chunk into the linearization records
      rbt::WireParams wp;
      wp.W = h->d_W;
      wp.n_grid = h->n_grid;
      wp.ocp_stride = h->w_ocp;
      wp.l_stride = h->S.l_stride;
      wp.wire = h->d_wire + size_t(b0) * h->w_ocp;
      wp.lin = h->d_lin + size_t(b0) * h->n_grid * h->S.l_stride;
      wp.res = res_host ? h->d_res_stage + size_t(b0) * h->n_grid * h->S.ncp : nullptr;
      wp.con = h->d_con + size_t(b0) * h->n_grid * h->S.c_stride;
      wp.c_stride = h->S.c_stride; wp.c_res = h->S.c_res; wp.ncp = h->S.ncp;
      rbt::unpack_wire_kernel<<<nb * h->n_grid, 128, 0, st>>>(wp);
      h->launches += 1;
      if ((h->cost_structure & RBT_WIRE_DEVICE_ID) && (rc = rbt_linearize_inverse_dynamics(h, stream)) != RBT_OK) break;
    }
    if (!(rc = rbt_condense(h, stream)) && !(rc = rbt_riccati_backward(h, 0, stream)) && !(rc = rbt_riccati_forward(h, stream)) &&
        !(rc = rbt_expand_and_step_sizes(h, stream)))
      rc = rbt_update(h, stream);
    h->cb0 = 0;
    h->cnb = 0;
    if (rc != RBT_OK) break;
    if (res_host && con_out) {
      rbt::pack_slack_dual_kernel<<<nb * h->n_grid, 64, 0, st>>>(h->d_con + size_t(b0) * h->n_grid * h->S.c_stride, h->S.c_stride,
                                                               h->S.c_slack, 2 * h->S.ncp,
                                                               h->d_sd_stage + size_t(b0) * h->n_grid * 2 * h->S.ncp);
      h->launches += 1;
    }
    RBT_CUDA(h, cudaEventRecord(h->ev[2 * c + 1], st));
    RBT_CUDA(h, cudaStreamWaitEvent(h->s_d2h, h->ev[2 * c + 1], 0));
    if (sol_out) stage_xfer(h, RBT_BUF_SOL, false, nullptr, sol_out, b0, nb, h->s_d2h, true, &rc);
    if (con_out) stage_xfer(h, res_host ? RBT_XFER_SD : RBT_BUF_CON, false, nullptr, con_out, b0, nb, h->s_d2h, true, &rc);
    if (steps_out) stage_xfer(h, RBT_BUF_STEPS, false, nullptr, steps_out, b0, nb, h->s_d2h, true, &rc);
  }
  h->cb0 = 0;
  h->cnb = 0;
  if (rc != RBT_OK) {
    if (h->err.empty() || rc == RBT_ERR_CUDA) h->err = std::string("rbt_iteration_host: ") + cudaGetErrorString(cudaGetLastError());
    return rc;
  }
  RBT_CUDA(h, cudaEventRecord(ev_exit, h->s_d2h));       // `stream` (what the caller synchronizes) covers the downloads too
  RBT_CUDA(h, cudaStreamWaitEvent(st, ev_exit, 0));
  return RBT_OK;
}

int rbt_iteration_host(rbt_handle* h, const double* lin_host, const double* con_host, const double* sol_host,
                       const double* dx0_host, double* sol_out, double* con_out, double* steps_out, void* stream) {
  if (!lin_host) return RBT_ERR_ARG;
  return iteration_host_impl(h, nullptr, lin_host, con_host, sol_host, nullptr, dx0_host, sol_out, con_out, steps_out, stream);
}

int rbt_iteration_host_wire(rbt_handle* h, const double* wire_host, const double* lin_host_switching, const double* con_host,
                            const double* sol_host, const double* dx0_host, double* sol_out, double* con_out,
                            double* steps_out, void* stream) {
  if (!wire_host || !con_host || !sol_host) return RBT_ERR_ARG;
  return iteration_host_impl(h, wire_host, lin_host_switching, con_host, sol_host, nullptr, dx0_host, sol_out, con_out, steps_out, stream);
}

int rbt_iteration_host_resident(rbt_handle* h, const double* wire_host, const double* lin_host_switching, const double* res_host,
                                const double* dx0_host, double* sol_out, double* slack_dual_out, double* steps_out, void* stream) {
  if (!wire_host || !res_host) return RBT_ERR_ARG;
  return iteration_host_impl(h, wire_host, lin_host_switching, nullptr, nullptr, res_host, dx0_host, sol_out, slack_dual_out, steps_out,
                             stream);
}

int rbt_set_wire_cost_structure(rbt_handle* h, int cost_structure) {
  if (!h || (cost_structure & ~(RBT_COST_ROBOTOC | RBT_WIRE_DEVICE_ID)) != 0) return RBT_ERR_ARG;
  if (h->cost_structure != cost_structure) h->wire_dirty = true;
  h->cost_structure = cost_structure;
  return RBT_OK;
}

int rbt_wire_doubles(const rbt_stage_dims* sdims, const rbt_stage_ctrl* ctrl, int n_grid, int cost_structure) {
  if (!sdims || !ctrl || n_grid <= 0) return -1;
  rbt_stage_layout S;
  rbt_make_stage_layout(sdims, &S);
  std::vector<rbt_wire_layout> W;
  return int(make_wire_layouts(S, ctrl, n_grid, cost_structure, W));
}

int rbt_wire_layout_get(const rbt_stage_dims* sdims, const rbt_stage_ctrl* ctrl, int n_grid, int cost_structure, int i,
                        rbt_wire_layout* out) {
  if (!sdims || !ctrl || !out || i < 0 || i >= n_grid) return RBT_ERR_ARG;
  rbt_stage_layout S;
  rbt_make_stage_layout(sdims, &S);
  std::vector<rbt_wire_layout> W;
  make_wire_layouts(S, ctrl, n_grid, cost_structure, W);
  *out = W[i];
  return RBT_OK;
}

int rbt_pack_wire(const rbt_stage_dims* sdims, const rbt_stage_ctrl* ctrl, int n_grid, int cost_structure, const double* lin_host,
                  double* wire_host, long long n_ocps) {
  if (!sdims || !ctrl || n_grid <= 0 || !lin_host || !wire_host || n_ocps < 0) return RBT_ERR_ARG;
  rbt_stage_layout S;
  rbt_make_stage_layout(sdims, &S);
  std::vector<rbt_wire_layout> W;
  const long long w_ocp = make_wire_layouts(S, ctrl, n_grid, cost_structure, W);
  for (long long b = 0; b < n_ocps; ++b)
    for (int i = 0; i < n_grid; ++i)
      rbt_pack_wire_record(&W[i], lin_host + (b * n_grid + i) * S.l_stride, wire_host + b * w_ocp + W[i].ocp_off);
  return RBT_OK;
}

int rbt_riccati_solve_host(rbt_handle* h, const double* kkt_host, const double* dx0_host, double* ric_host,
                           double* dir_host, void* stream) {
  if (!h || !kkt_host || !dx0_host) return RBT_ERR_ARG;
  int rc;
  if ((rc = rbt_upload(h, RBT_BUF_KKT, kkt_host, stream))) return rc;
  if ((rc = rbt_upload(h, RBT_BUF_DX0, dx0_host, stream))) return rc;
  if ((rc = rbt_riccati_backward(h, 0, stream))) return rc;
  if ((rc = rbt_riccati_forward(h, stream))) return rc;
  if (ric_host && (rc = rbt_download(h, RBT_BUF_RIC, ric_host, stream))) return rc;
  if (dir_host && (rc = rbt_download(h, RBT_BUF_DIR, dir_host, stream))) return rc;
  return RBT_OK;
}

// ---- multi-GPU: the Newton step of every OCP on every rank ----------------------------------------------------------------
namespace {
// NCCL is reached through dlsym so that the library neither links against a particular libnccl nor fails to load without
// one: the communicator belongs to the host application, and it is the host's NCCL that must execute the collective.
typedef int (*nccl_allgather_fn)(const void*, void*, size_t, int, void*, cudaStream_t);
nccl_allgather_fn find_nccl_allgather() {
  static nccl_allgather_fn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* sym = dlsym(RTLD_DEFAULT, "ncclAllGather");  // the NCCL the host process already uses
    if (!sym) {
      void* lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
      if (lib) sym = dlsym(lib, "ncclAllGather");
    }
    fn = reinterpret_cast<nccl_allgather_fn>(sym);
  }
  return fn;
}

// direction records (stride d_stride) -> packed step records (the used prefix dx | du | dlmd,dgmm | dxi | dts,dts_next)
__global__ void pack_step_kernel(const double* __restrict__ dir, double* __restrict__ out, int d_stride, int step, long long n_rec) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n_rec * step) return;
  const long long rec = e / step;
  const int k = int(e % step);
  out[e] = dir[rec * d_stride + k];
}
}  // namespace

int rbt_step_doubles(rbt_handle* h) { return h ? h->L.d_dts + 2 : -1; }

int rbt_pack_step(rbt_handle* h, double* packed_dev, void* stream) {
  if (!h || !packed_dev) return RBT_ERR_ARG;
  if (h->n_grid == 0) return RBT_ERR_STATE;
  RBT_CUDA(h, cudaSetDevice(h->device));
  const int step = h->L.d_dts + 2;
  const long long n_rec = (long long)h->batch * h->n_grid;
  pack_step_kernel<<<unsigned((n_rec * step + 255) / 256), 256, 0, (cudaStream_t)stream>>>(h->d_dir, packed_dev, h->L.d_stride, step, n_rec);
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

int rbt_allgather_step(rbt_handle* h, void* nccl_comm, double* all_dev, void* stream) {
  if (!h || !nccl_comm || !all_dev) return RBT_ERR_ARG;
  if (h->n_grid == 0) return RBT_ERR_STATE;
  nccl_allgather_fn allgather = find_nccl_allgather();
  if (!allgather) {
    h->err = "[rbt_allgather_step] no NCCL in this process (ncclAllGather not found, libnccl.so.2 not loadable)";
    return RBT_ERR_STATE;
  }
  RBT_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  const int step = h->L.d_dts + 2;
  const long long n_rec = (long long)h->batch * h->n_grid;
  if (!h->d_step_pack) RBT_CUDA(h, cudaMalloc(&h->d_step_pack, size_t(h->batch) * h->n_grid_max * step * 8));
  if (int prc = rbt_pack_step(h, h->d_step_pack, stream)) return prc;
  const int rc = allgather(h->d_step_pack, all_dev, size_t(n_rec) * step, /*ncclFloat64*/ 8, nccl_comm, st);
  if (rc != 0) {
    h->err = "[rbt_allgather_step] ncclAllGather failed with ncclResult_t " + std::to_string(rc);
    return RBT_ERR_CUDA;
  }
  return RBT_OK;
}

int rbt_sync(rbt_handle* h, void* stream) {
  if (!h) return RBT_ERR_ARG;
  RBT_CUDA(h, cudaSetDevice(h->device));
  RBT_CUDA(h, cudaStreamSynchronize((cudaStream_t)stream));
  return RBT_OK;
}

const char* rbt_last_error(rbt_handle* h) { return h ? h->err.c_str() : "null handle"; }

// bring-up only (not part of the public header): copy the timeline stamps of the last backward launch
extern "C" int rbt_debug_timeline(rbt_handle* h, long long* host, int n) {
  if (!h || !h->d_timeline) return RBT_ERR_STATE;
  return cudaMemcpy(host, h->d_timeline, size_t(n) * sizeof(long long), cudaMemcpyDeviceToHost) == cudaSuccess ? RBT_OK : RBT_ERR_CUDA;
}
long long rbt_launch_count(rbt_handle* h) { return h ? h->launches : 0; }

// ---------------------------------------------------------------------------------------------------------------
// unconstrained path
// ---------------------------------------------------------------------------------------------------------------
#define RBT_UINSTANCES(X) X(7)

int rbt_unconstr_create(int nv, int N, double dt, int batch, int device, rbt_uhandle** out) {
  if (!out || nv < 1 || N < 1 || batch < 1 || !(dt > 0)) return RBT_ERR_ARG;
  bool ok = false;
#define X(NV) \
  if (nv == NV) ok = true;
  RBT_UINSTANCES(X)
#undef X
  if (!ok) return RBT_ERR_ARG;
  rbt_uhandle* h = new rbt_uhandle();
  h->nv = nv;
  h->N = N;
  h->dt = dt;
  h->batch = batch;
  h->device = device;
  rbt_make_ulayout(nv, &h->L);
  *out = h;
  RBT_CUDA(h, cudaSetDevice(device));
  const size_t per = size_t(batch) * (N + 1);
  RBT_CUDA(h, cudaMalloc(&h->d_kkt, per * h->L.k_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_ric, per * h->L.r_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_fact, per * h->L.f_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_dir, per * h->L.d_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_dx0, size_t(batch) * h->L.nx * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_info, size_t(batch) * sizeof(int)));
  RBT_CUDA(h, cudaMemset(h->d_ric, 0, per * h->L.r_stride * 8));
  RBT_CUDA(h, cudaMemset(h->d_fact, 0, per * h->L.f_stride * 8));
  RBT_CUDA(h, cudaMemset(h->d_dir, 0, per * h->L.d_stride * 8));
  RBT_CUDA(h, cudaMemset(h->d_info, 0, size_t(batch) * sizeof(int)));
  return RBT_OK;
}

int rbt_unconstr_destroy(rbt_uhandle* h) {
  if (!h) return RBT_ERR_ARG;
  cudaSetDevice(h->device);
  cudaFree(h->d_kkt);
  cudaFree(h->d_ric);
  cudaFree(h->d_fact);
  cudaFree(h->d_dir);
  cudaFree(h->d_dx0);
  cudaFree(h->d_info);
  cudaFree(h->d_lin);
  cudaFree(h->d_con);
  cudaFree(h->d_ex);
  cudaFree(h->d_sol);
  cudaFree(h->d_xd);
  cudaFree(h->d_steps);
  cudaFree(h->d_ones);
  delete h;
  return RBT_OK;
}

static double* ubuf_ptr(rbt_uhandle* h, int which) {
  switch (which) {
    case RBT_BUF_KKT: return h->d_kkt;
    case RBT_BUF_RIC: return h->d_ric;
    case RBT_BUF_FACT: return h->d_fact;
    case RBT_BUF_DIR: return h->d_dir;
    case RBT_BUF_DX0: return h->d_dx0;
    case RBT_BUF_LIN: return h->d_lin;
    case RBT_BUF_CON: return h->d_con;
    case RBT_BUF_EXP: return h->d_ex;
    case RBT_BUF_SOL: return h->d_sol;
    case RBT_BUF_XDIR: return h->d_xd;
    case RBT_BUF_STEPS: return h->d_steps;
    default: return nullptr;
  }
}

long long rbt_unconstr_buf_doubles(rbt_uhandle* h, int which) {
  if (!h) return -1;
  const long long per = (long long)h->batch * (h->N + 1);
  switch (which) {
    case RBT_BUF_KKT: return per * h->L.k_stride;
    case RBT_BUF_RIC: return per * h->L.r_stride;
    case RBT_BUF_FACT: return per * h->L.f_stride;
    case RBT_BUF_DIR: return per * h->L.d_stride;
    case RBT_BUF_DX0: return (long long)h->batch * h->L.nx;
    default: break;
  }
  if (!h->stage_ready) return -1;
  switch (which) {
    case RBT_BUF_LIN: return per * h->S.l_stride;
    case RBT_BUF_CON: return per * h->S.c_stride;
    case RBT_BUF_EXP: return per * h->S.e_stride;
    case RBT_BUF_SOL: return per * h->S.s_stride;
    case RBT_BUF_XDIR: return per * h->S.x_stride;
    case RBT_BUF_STEPS: return (long long)h->batch * 2;
    default: return -1;
  }
}

double* rbt_unconstr_dev_ptr(rbt_uhandle* h, int which) { return h ? ubuf_ptr(h, which) : nullptr; }

int rbt_unconstr_upload(rbt_uhandle* h, int which, const double* host, void* stream) {
  if (!h || !host) return RBT_ERR_ARG;
  if (which != RBT_BUF_KKT && which != RBT_BUF_DX0 && which != RBT_BUF_LIN && which != RBT_BUF_CON && which != RBT_BUF_SOL)
    return RBT_ERR_ARG;
  // a table with n_box = 0 has an empty PDIPM record: its buffer is a null allocation, and copying it is a no-op
  const long long n = rbt_unconstr_buf_doubles(h, which);
  if (n < 0 || (n > 0 && !ubuf_ptr(h, which))) {
    h->err = "rbt_unconstr_upload: stage layer not set up (rbt_unconstr_stage_setup)";
    return RBT_ERR_STATE;
  }
  if (n == 0) return RBT_OK;
  RBT_CUDA(h, cudaSetDevice(h->device));
  RBT_CUDA(h, cudaMemcpyAsync(ubuf_ptr(h, which), host, size_t(n) * 8, cudaMemcpyHostToDevice, (cudaStream_t)stream));
  return RBT_OK;
}

int rbt_unconstr_download(rbt_uhandle* h, int which, double* host, void* stream) {
  if (!h || !host) return RBT_ERR_ARG;
  const long long n = rbt_unconstr_buf_doubles(h, which);
  if (n < 0 || (n > 0 && !ubuf_ptr(h, which))) return RBT_ERR_ARG;
  if (n == 0) return RBT_OK;
  RBT_CUDA(h, cudaSetDevice(h->device));
  RBT_CUDA(h, cudaMemcpyAsync(host, ubuf_ptr(h, which), size_t(n) * 8, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return RBT_OK;
}

int rbt_unconstr_download_info(rbt_uhandle* h, int* host_flags, void* stream) {
  if (!h || !host_flags) return RBT_ERR_ARG;
  RBT_CUDA(h, cudaSetDevice(h->device));
  RBT_CUDA(h, cudaMemcpyAsync(host_flags, h->d_info, size_t(h->batch) * sizeof(int), cudaMemcpyDeviceToHost,
                              (cudaStream_t)stream));
  return RBT_OK;
}

template <int NV>
static rbt::UParams make_uparams(rbt_uhandle* h, int write_fact) {
  rbt::UParams p;
  p.L = h->L;
  p.N = h->N;
  p.batch = h->batch;
  p.dt = h->dt;
  p.kkt = h->d_kkt;
  p.ric = h->d_ric;
  p.fact = write_fact ? h->d_fact : nullptr;
  p.dx0 = h->d_dx0;
  p.dir = h->d_dir;
  p.info = h->d_info;
  return p;
}

int rbt_unconstr_backward(rbt_uhandle* h, int write_fact, void* stream) {
  if (!h) return RBT_ERR_ARG;
  RBT_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
#define X(NV)                                                                                  \
  if (h->nv == NV) {                                                                           \
    if (rbt::UCfg<NV>::KSTRIDE != h->L.k_stride) return RBT_ERR_STATE;                          \
    RBT_CUDA(h, cudaMemsetAsync(h->d_info, 0, size_t(h->batch) * sizeof(int), st));            \
    rbt::unconstr_backward_kernel<NV><<<h->batch, 32, 0, st>>>(make_uparams<NV>(h, write_fact)); \
    RBT_CUDA(h, cudaGetLastError());                                                           \
    h->launches += 1;                                                                          \
    return RBT_OK;                                                                             \
  }
  RBT_UINSTANCES(X)
#undef X
  return RBT_ERR_ARG;
}

int rbt_unconstr_forward(rbt_uhandle* h, void* stream) {
  if (!h) return RBT_ERR_ARG;
  RBT_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
#define X(NV)                                                                         \
  if (h->nv == NV) {                                                                  \
    rbt::unconstr_forward_kernel<NV><<<h->batch, 32, 0, st>>>(make_uparams<NV>(h, 0)); \
    RBT_CUDA(h, cudaGetLastError());                                                  \
    h->launches += 1;                                                                 \
    return RBT_OK;                                                                    \
  }
  RBT_UINSTANCES(X)
#undef X
  return RBT_ERR_ARG;
}

int rbt_unconstr_solve_host(rbt_uhandle* h, const double* kkt_host, const double* dx0_host, double* ric_host,
                            double* dir_host, void* stream) {
  if (!h || !kkt_host || !dx0_host) return RBT_ERR_ARG;
  int rc;
  if ((rc = rbt_unconstr_upload(h, RBT_BUF_KKT, kkt_host, stream))) return rc;
  if ((rc = rbt_unconstr_upload(h, RBT_BUF_DX0, dx0_host, stream))) return rc;
  if ((rc = rbt_unconstr_backward(h, 0, stream))) return rc;
  if ((rc = rbt_unconstr_forward(h, stream))) return rc;
  if (ric_host && (rc = rbt_unconstr_download(h, RBT_BUF_RIC, ric_host, stream))) return rc;
  if (dir_host && (rc = rbt_unconstr_download(h, RBT_BUF_DIR, dir_host, stream))) return rc;
  return RBT_OK;
}

int rbt_unconstr_sync(rbt_uhandle* h, void* stream) {
  if (!h) return RBT_ERR_ARG;
  RBT_CUDA(h, cudaSetDevice(h->device));
  RBT_CUDA(h, cudaStreamSynchronize((cudaStream_t)stream));
  return RBT_OK;
}

// ---- stage layer of the unconstrained path
int rbt_unconstr_stage_layout_get(int nv, int n_box, const char* field) {
  if (nv < 1 || n_box < 0 || !field) return -1;
  rbt_ustage_layout S;
  rbt_make_ustage_layout(nv, n_box, &S);
  return rbt_ustage_layout_field(&S, field);
}

int rbt_unconstr_stage_setup(rbt_uhandle* h, const rbt_constraint_table* table) {
  if (!h || !table) return RBT_ERR_ARG;
  if (table->n_box < 0 || table->n_box > RBT_MAX_BOX_ROWS || table->n_contacts != 0 || !(table->barrier > 0) ||
      !(table->fraction_to_boundary > 0 && table->fraction_to_boundary < 1)) {
    h->err = "rbt_unconstr_stage_setup: invalid constraint table (n_box range, n_contacts must be 0, barrier > 0, 0 < fraction_to_boundary < 1)";
    return RBT_ERR_ARG;
  }
  for (int r = 0; r < table->n_box; ++r) {
    const rbt_box_row& b = table->box[r];
    if (b.var < RBT_VAR_Q || b.var > RBT_VAR_U || b.idx < 0 || b.idx >= h->nv || (b.sign != 1 && b.sign != -1)) {
      h->err = "rbt_unconstr_stage_setup: box row " + std::to_string(r) + " out of range";
      return RBT_ERR_ARG;
    }
  }
  if (h->stage_ready) {
    h->err = "rbt_unconstr_stage_setup: already set up";
    return RBT_ERR_STATE;
  }
  RBT_CUDA(h, cudaSetDevice(h->device));
  rbt_make_ustage_layout(h->nv, table->n_box, &h->S);
  h->table = *table;
  const size_t per = size_t(h->batch) * (h->N + 1);
  RBT_CUDA(h, cudaMalloc(&h->d_lin, per * h->S.l_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_con, per * h->S.c_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_ex, per * h->S.e_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_sol, per * h->S.s_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_xd, per * h->S.x_stride * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_steps, size_t(h->batch) * 2 * 8));
  RBT_CUDA(h, cudaMalloc(&h->d_ones, size_t(h->batch) * 2 * 8));
  RBT_CUDA(h, cudaMemset(h->d_lin, 0, per * h->S.l_stride * 8));
  RBT_CUDA(h, cudaMemset(h->d_con, 0, per * h->S.c_stride * 8));
  RBT_CUDA(h, cudaMemset(h->d_ex, 0, per * h->S.e_stride * 8));
  RBT_CUDA(h, cudaMemset(h->d_sol, 0, per * h->S.s_stride * 8));
  RBT_CUDA(h, cudaMemset(h->d_xd, 0, per * h->S.x_stride * 8));
  std::vector<double> ones(size_t(h->batch) * 2, 1.0);
  RBT_CUDA(h, cudaMemcpy(h->d_ones, ones.data(), ones.size() * 8, cudaMemcpyHostToDevice));
  RBT_CUDA(h, cudaMemcpy(h->d_steps, ones.data(), ones.size() * 8, cudaMemcpyHostToDevice));
  h->stage_ready = true;
  return RBT_OK;
}

static rbt::UStageParams make_ustage_params(rbt_uhandle* h) {
  rbt::UStageParams p;
  p.K = h->L;
  p.S = h->S;
  p.tab = h->table;
  p.N = h->N;
  p.batch = h->batch;
  p.dt = h->dt;
  p.lin = h->d_lin;
  p.con = h->d_con;
  p.kkt = h->d_kkt;
  p.ex = h->d_ex;
  p.dir = h->d_dir;
  p.xd = h->d_xd;
  p.sol = h->d_sol;
  p.steps = h->d_steps;
  return p;
}

#define RBT_USTAGE_GUARD(h)                                                              \
  if (!h) return RBT_ERR_ARG;                                                            \
  if (!h->stage_ready) {                                                                 \
    h->err = "stage layer not set up: call rbt_unconstr_stage_setup first";              \
    return RBT_ERR_STATE;                                                                \
  }                                                                                      \
  RBT_CUDA(h, cudaSetDevice(h->device));                                                 \
  cudaStream_t st = (cudaStream_t)stream;

int rbt_unconstr_condense(rbt_uhandle* h, void* stream) {
  RBT_USTAGE_GUARD(h)
  const size_t total = size_t(h->batch) * (h->N + 1);
#define X(NV)                                                                                         \
  if (h->nv == NV) {                                                                                  \
    if (rbt::UStageCfg<NV>::LSTRIDE != h->S.l_stride) return RBT_ERR_STATE;                            \
    constexpr int W = rbt::UStageCfg<NV>::WARPS;                                                      \
    rbt::ucondense_kernel<NV><<<unsigned((total + W - 1) / W), 32 * W, 0, st>>>(make_ustage_params(h)); \
    RBT_CUDA(h, cudaGetLastError());                                                                  \
    h->launches += 1;                                                                                 \
    return RBT_OK;                                                                                    \
  }
  RBT_UINSTANCES(X)
#undef X
  return RBT_ERR_ARG;
}

int rbt_unconstr_expand_and_step_sizes(rbt_uhandle* h, void* stream) {
  RBT_USTAGE_GUARD(h)
  const size_t total = size_t(h->batch) * h->N;
  RBT_CUDA(h, cudaMemcpyAsync(h->d_steps, h->d_ones, size_t(h->batch) * 2 * 8, cudaMemcpyDeviceToDevice, st));
#define X(NV)                                                                                 \
  if (h->nv == NV) {                                                                          \
    rbt::uexpand_kernel<NV><<<unsigned((total + 3) / 4), 128, 0, st>>>(make_ustage_params(h)); \
    RBT_CUDA(h, cudaGetLastError());                                                          \
    h->launches += 1;                                                                         \
    return RBT_OK;                                                                            \
  }
  RBT_UINSTANCES(X)
#undef X
  return RBT_ERR_ARG;
}

int rbt_unconstr_update(rbt_uhandle* h, void* stream) {
  RBT_USTAGE_GUARD(h)
  const size_t total = size_t(h->batch) * (h->N + 1);
#define X(NV)                                                                                 \
  if (h->nv == NV) {                                                                          \
    rbt::uupdate_kernel<NV><<<unsigned((total + 3) / 4), 128, 0, st>>>(make_ustage_params(h)); \
    RBT_CUDA(h, cudaGetLastError());                                                          \
    h->launches += 1;                                                                         \
    return RBT_OK;                                                                            \
  }
  RBT_UINSTANCES(X)
#undef X
  return RBT_ERR_ARG;
}

int rbt_unconstr_iteration_host(rbt_uhandle* h, const double* lin_host, const double* con_host, const double* sol_host,
                                const double* dx0_host, double* sol_out, double* con_out, double* steps_out,
                                void* stream) {
  if (!h || !lin_host || !con_host || !sol_host || !dx0_host) return RBT_ERR_ARG;
  int rc;
  if ((rc = rbt_unconstr_upload(h, RBT_BUF_LIN, lin_host, stream))) return rc;
  if ((rc = rbt_unconstr_upload(h, RBT_BUF_CON, con_host, stream))) return rc;
  if ((rc = rbt_unconstr_upload(h, RBT_BUF_SOL, sol_host, stream))) return rc;
  if ((rc = rbt_unconstr_upload(h, RBT_BUF_DX0, dx0_host, stream))) return rc;
  if ((rc = rbt_unconstr_condense(h, stream))) return rc;
  if ((rc = rbt_unconstr_backward(h, 0, stream))) return rc;
  if ((rc = rbt_unconstr_forward(h, stream))) return rc;
  if ((rc = rbt_unconstr_expand_and_step_sizes(h, stream))) return rc;
  if ((rc = rbt_unconstr_update(h, stream))) return rc;
  if (sol_out && (rc = rbt_unconstr_download(h, RBT_BUF_SOL, sol_out, stream))) return rc;
  if (con_out && (rc = rbt_unconstr_download(h, RBT_BUF_CON, con_out, stream))) return rc;
  if (steps_out && (rc = rbt_unconstr_download(h, RBT_BUF_STEPS, steps_out, stream))) return rc;
  return RBT_OK;
}

const char* rbt_unconstr_last_error(rbt_uhandle* h) { return h ? h->err.c_str() : "null handle"; }
long long rbt_unconstr_launch_count(rbt_uhandle* h) { return h ? h->launches : 0; }


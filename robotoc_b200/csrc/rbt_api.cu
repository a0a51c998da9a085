// rbt_api.cu -- C ABI of librobotoc_b200.so (see include/robotoc_b200.h for the reference interfaces replaced).
// Plumbing only: handles, device buffers, stream-ordered copies and kernel launches.  No CPU compute path.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <cstdint>
#include <cstdlib>
#include <string>
#include <utility>
#include <vector>

#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>

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
#include "contact_kernels.cuh"
#include "state_kernels.cuh"

namespace {

#define RBT_CUDA(h, call)                                                                     \
  do {                                                                                        \
    cudaError_t e_ = (call);                                                                  \
    if (e_ != cudaSuccess) {                                                                  \
      (h)->err = std::string(#call) + ": " + cudaGetErrorString(e_);                          \
      return RBT_ERR_CUDA;                                                                    \
    }                                                                                         \
  } while (0)

// The one compiled instance of each path: constrained ANYmal (floating base + 4 point contacts, src/robot/robot.cpp:33-60)
// and unconstrained iiwa14.  rbt_create / rbt_unconstr_create reject every other dimension.
constexpr int CNV = 18, CNU = 12, CNS = 12, CNP = 6;
constexpr int UNV = 7;

// Owns one cudaMalloc allocation, freed with its owner.  ensure(n) grows it to at least n elements (dropping the contents).
template <class T>
class DevBuf {
 public:
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
  DevBuf& operator=(DevBuf&& o) noexcept {
    std::swap(p_, o.p_);
    std::swap(n_, o.n_);
    return *this;
  }
  ~DevBuf() { cudaFree(p_); }
  cudaError_t ensure(size_t n) {
    if (n <= n_) return cudaSuccess;
    cudaFree(p_);
    p_ = nullptr;
    n_ = 0;
    const cudaError_t e = cudaMalloc(&p_, n * sizeof(T));
    if (e != cudaSuccess) p_ = nullptr;
    else n_ = n;
    return e;
  }
  T* get() const { return p_; }

 private:
  T* p_ = nullptr;
  size_t n_ = 0;
};

template <class T>
cudaError_t zeroed(DevBuf<T>& b, size_t n) {
  const cudaError_t e = b.ensure(n);
  return e != cudaSuccess ? e : cudaMemset(b.get(), 0, n * sizeof(T));
}

// Owns a stream or an event.
template <class T, cudaError_t (*Destroy)(T)>
class CudaObj {
 public:
  CudaObj() = default;
  CudaObj(CudaObj&& o) noexcept : v_(std::exchange(o.v_, nullptr)) {}
  CudaObj& operator=(CudaObj&& o) noexcept {
    std::swap(v_, o.v_);
    return *this;
  }
  ~CudaObj() {
    if (v_) Destroy(v_);
  }
  T get() const { return v_; }
  T* out() { return &v_; }  // for the create call

 private:
  T v_ = nullptr;
};
using Stream = CudaObj<cudaStream_t, cudaStreamDestroy>;
using Event = CudaObj<cudaEvent_t, cudaEventDestroy>;

// A buffer the caller may replace with a device allocation of its own (rbt_bind_buffer); the handle keeps its own beside it.
struct Bindable {
  DevBuf<double> own;
  double* bound = nullptr;
  double* get() const { return bound ? bound : own.get(); }
};

// One copy between a device buffer and a host array of the same layout: `rows` rows of `width` doubles, `pitch` doubles
// apart, from offset `off` on both sides.  `host` names the host array (IN_* uploads, OUT_* downloads).
struct Copy {
  double* dev;
  size_t off, width, pitch, rows;
  bool up;
  int host;
};
enum { IN_KKT, IN_WIRE, IN_LIN, IN_CON, IN_SOL, IN_RES, IN_DX0, IN_CPOS, IN_Q0, N_IN };
enum { OUT_SOL, OUT_CON, OUT_STEPS, N_OUT };

// What an RBT_BUF_* id names on a handle.
enum { SC_NONE, SC_GRID, SC_OCP };  // no such double buffer / one record per grid point / one record per OCP
struct BufDesc {
  double* ptr;      // the buffer in use
  long long per;    // doubles per record
  int scope;
  bool stage;       // exists from the stage setup on
  Bindable* bind;   // non-null: rbt_bind_buffer may replace it
  int in;           // the host array rbt_upload reads (IN_*), -1: not uploadable
};

long long buf_doubles(const BufDesc& d, bool stage_ready, int batch, int n_grid) {
  if (d.scope == SC_NONE || (d.stage && !stage_ready)) return -1;
  return d.per * batch * (d.scope == SC_GRID ? n_grid : 1);
}

// A window [b0, b0 + nb) of the batch: the host iteration pipelines its chunks through the launchers, everything else passes
// the whole batch.  rec() is the first record of the window in a buffer of one record per grid point.
struct Win {
  int b0, nb, n_grid;
  size_t rec() const { return size_t(b0) * n_grid; }
};

long long plan_bytes(const std::vector<Copy>& plan, bool up) {
  long long bytes = 0;
  for (const Copy& c : plan)
    if (c.up == up) bytes += (long long)(c.width * 8 * c.rows);
  return bytes;
}

}  // namespace

struct rbt_handle {
  rbt_dims dims;
  rbt_layout L;
  int n_grid_max = 0, n_grid = 0, batch = 0, device = 0;
  double max_dts0 = 0.1;
  DevBuf<rbt_stage_ctrl> d_ctrl;
  std::vector<rbt_stage_ctrl> ctrl;  // host copy
  Bindable d_kkt, d_ric, d_fact, d_dir, d_dx0;
  DevBuf<int> d_info;
  DevBuf<int> d_struct;  // [0]: 1 = every Fxx of the KKT buffer has the mechanical structure (see rbt_set_fxx_structure)
  int fxx_mode = RBT_FXX_AUTO;
  // time-parallel sweeps (riccati_time_parallel.cuh): requested segment count (0 = automatic, 1 = serial) and scratch,
  // allocated on the first segmented sweep; the S-dependent buffers grow with the largest S used
  int tsegs = 0, n_sm = 0;
  DevBuf<double> d_tp_elem, d_tp_scan[2], d_tp_fmap, d_tp_dx;
  DevBuf<int> d_tp_fail;
  const double* tp_seeds = nullptr;  // the scan buffer the last segmented backward sweep read its seeds from
  bool kkt_from_condense = false;  // the KKT records were just written by rbt_condense: structure holds by construction
  // stage layer
  bool stage_ready = false;
  bool keep_info = false;  // condense's Cholesky flags survive the following backward launch
  rbt_stage_dims sdims;
  rbt_stage_layout S;
  rbt_constraint_table table;
  Bindable d_lin, d_con, d_ex, d_sol, d_xd;
  DevBuf<double> d_steps, d_ones;
  DevBuf<double> d_stage_perf, d_perf, d_x0in;  // eval_kernels.cuh
  DevBuf<int> d_tgt;                  // box rows per PDIPM target (stage_kernels.cuh: StageParams::tgt)
  DevBuf<double> d_limits;            // joint limits per box row (rbt_set_joint_limits)
  DevBuf<rbt::RneaModel> d_model;     // robot model of rbt_linearize_inverse_dynamics (rbt_set_robot_model)
  DevBuf<double> d_gains;             // Baumgarte gains per contact (rbt_set_contact_gains)
  DevBuf<double> d_cpos;              // desired contact positions (RBT_BUF_CONTACT_POS), allocated on the first upload
  bool cpos_set = false;              // d_cpos has been uploaded once
  DevBuf<double> d_q0;                // measured configuration per OCP (RBT_BUF_Q0), allocated on the first upload
  bool q0_set = false;                // d_q0 has been uploaded once
  // line search (line_search_kernels.cuh): trial buffers sized on first use, filter state per OCP
  int ls_trials = 0;
  DevBuf<double> d_ls_alphas, d_ls_trial, d_ls_stage_barrier, d_ls_barrier, d_ls_in, d_ls_filt, d_ls_step;
  DevBuf<int> d_ls_nfilt, d_ls_k;
  DevBuf<double> d_step_pack;  // packed Newton step of this rank (rbt_allgather_step), allocated on first use
  long long launches = 0;
  DevBuf<double> d_wire;       // packed host wire records (rbt_iteration_host_wire), allocated on first use
  DevBuf<double> d_res_stage;  // rbt_iteration_host_resident: compact residuals in, compact slack|dual out
  DevBuf<double> d_sd_stage;
  DevBuf<rbt_wire_layout> d_W;  // per grid point (the wire record of a grid point depends on its control word)
  long long w_ocp = 0;          // doubles of one OCP's concatenated wire records
  int cost_structure = RBT_COST_GENERAL;  // what the host's wire records hold (rbt_set_wire_cost_structure)
  bool wire_dirty = true;                 // per-grid-point wire layouts on the device are stale (schedule / cost structure changed)
  bool attr_bwd = false, attr_fwd = false, attr_cond = false, attr_tp = false;  // MaxDynamicSharedMemorySize set on THIS handle's device
  cudaEvent_t ev_condense_mid = nullptr;  // caller-owned event recorded between the two kernels of rbt_condense (timing)
  Stream s_h2d, s_d2h;
  std::vector<Event> ev;
  std::string err;
};

struct rbt_uhandle {
  int nv = 0, N = 0, batch = 0, device = 0;
  double dt = 0;
  rbt_ulayout L;
  DevBuf<double> d_kkt, d_ric, d_fact, d_dir, d_dx0;
  DevBuf<int> d_info;
  // stage layer
  bool stage_ready = false;
  rbt_ustage_layout S;
  rbt_constraint_table table;
  DevBuf<double> d_lin, d_con, d_ex, d_sol, d_xd, d_steps, d_ones;
  long long launches = 0;
  std::string err;
};

static Win full(const rbt_handle* h) { return {0, h->batch, h->n_grid}; }

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
  if (dims->nv != CNV || dims->nu != CNU || dims->ns_max != CNS) return RBT_ERR_ARG;
  rbt_handle* h = new rbt_handle();
  h->dims = *dims;
  rbt_make_layout(dims, &h->L);
  h->n_grid_max = n_grid_max;
  h->batch = batch;
  h->device = device;
  *out = h;
  RBT_CUDA(h, cudaSetDevice(device));
  const size_t per = size_t(batch) * n_grid_max;
  RBT_CUDA(h, h->d_ctrl.ensure(size_t(n_grid_max)));
  RBT_CUDA(h, zeroed(h->d_kkt.own, per * h->L.k_stride));  // condensing skips the switching rows a stage lacks: keep them defined
  RBT_CUDA(h, zeroed(h->d_ric.own, per * h->L.r_stride));
  RBT_CUDA(h, zeroed(h->d_fact.own, per * h->L.f_stride));
  RBT_CUDA(h, zeroed(h->d_dir.own, per * h->L.d_stride));
  RBT_CUDA(h, h->d_dx0.own.ensure(size_t(batch) * h->L.nx));
  RBT_CUDA(h, zeroed(h->d_info, size_t(batch)));
  RBT_CUDA(h, zeroed(h->d_struct, 4));
  RBT_CUDA(h, cudaDeviceGetAttribute(&h->n_sm, cudaDevAttrMultiProcessorCount, device));
  return RBT_OK;
}

// The stage kernels are compiled for nf_max / n_contacts of the constraint table: every grid of the schedule must fit.
static int check_contacts(rbt_handle* h, const rbt_stage_dims& sd, const rbt_stage_ctrl* ctrl, int n_grid) {
  for (int i = 0; i < n_grid; ++i)
    if (ctrl[i].nf > sd.nf_max || ctrl[i].contact_mask >= (1 << sd.n_contacts)) {
      h->err = "[rbt_set_schedule] invalid argument: grid " + std::to_string(i) + " has more contacts than the stage layer was set up for";
      return RBT_ERR_ARG;
    }
  return RBT_OK;
}

int rbt_destroy(rbt_handle* h) {
  if (!h) return RBT_ERR_ARG;
  cudaSetDevice(h->device);
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
  if (h->stage_ready && check_contacts(h, h->sdims, ctrl, n_grid) != RBT_OK) return RBT_ERR_ARG;
  RBT_CUDA(h, cudaSetDevice(h->device));
  RBT_CUDA(h, cudaMemcpy(h->d_ctrl.get(), ctrl, sizeof(rbt_stage_ctrl) * n_grid, cudaMemcpyHostToDevice));
  // stage-conditional outputs (M, STO terms, policies) must not leak from a previous schedule
  RBT_CUDA(h, cudaMemset(h->d_ric.get(), 0, size_t(h->batch) * n_grid * h->L.r_stride * 8));
  RBT_CUDA(h, cudaMemset(h->d_dir.get(), 0, size_t(h->batch) * n_grid * h->L.d_stride * 8));
  h->n_grid = n_grid;
  h->max_dts0 = max_dts0;
  h->ctrl.assign(ctrl, ctrl + n_grid);
  h->wire_dirty = true;
  return RBT_OK;
}

static BufDesc buf(rbt_handle* h, int which) {
  const rbt_layout& L = h->L;
  const rbt_stage_layout& S = h->S;
  const BufDesc t[] = {
      /* KKT   */ {h->d_kkt.get(), L.k_stride, SC_GRID, false, &h->d_kkt, IN_KKT},
      /* RIC   */ {h->d_ric.get(), L.r_stride, SC_GRID, false, &h->d_ric, -1},
      /* FACT  */ {h->d_fact.get(), L.f_stride, SC_GRID, false, &h->d_fact, -1},
      /* DIR   */ {h->d_dir.get(), L.d_stride, SC_GRID, false, &h->d_dir, -1},
      /* DX0   */ {h->d_dx0.get(), L.nx, SC_OCP, false, &h->d_dx0, IN_DX0},
      /* INFO  */ {nullptr, 0, SC_NONE, false, nullptr, -1},
      /* LIN   */ {h->d_lin.get(), S.l_stride, SC_GRID, true, &h->d_lin, IN_LIN},
      /* CON   */ {h->d_con.get(), S.c_stride, SC_GRID, true, &h->d_con, IN_CON},
      /* EXP   */ {h->d_ex.get(), S.e_stride, SC_GRID, true, &h->d_ex, -1},
      /* SOL   */ {h->d_sol.get(), S.s_stride, SC_GRID, true, &h->d_sol, IN_SOL},
      /* XDIR  */ {h->d_xd.get(), S.x_stride, SC_GRID, true, &h->d_xd, -1},
      /* STEPS */ {h->d_steps.get(), 2, SC_OCP, true, nullptr, -1},
      /* PERF  */ {h->d_perf.get(), 8, SC_OCP, true, nullptr, -1},
      /* CPOS  */ {h->d_cpos.get(), 3 * S.ncon, SC_GRID, true, nullptr, IN_CPOS},
      /* Q0    */ {h->d_q0.get(), S.nq, SC_OCP, true, nullptr, IN_Q0},
  };
  return which >= 0 && which < int(sizeof(t) / sizeof(t[0])) ? t[which] : BufDesc{nullptr, 0, SC_NONE, false, nullptr, -1};
}

long long rbt_buf_doubles(rbt_handle* h, int which) {
  return h ? buf_doubles(buf(h, which), h->stage_ready, h->batch, h->n_grid) : -1;
}

double* rbt_dev_ptr(rbt_handle* h, int which) { return h ? buf(h, which).ptr : nullptr; }

int rbt_bind_buffer(rbt_handle* h, int which, double* dev) {
  if (!h) return RBT_ERR_ARG;
  const BufDesc d = buf(h, which);
  if (!d.bind || (d.stage && !h->stage_ready)) return RBT_ERR_ARG;
  if ((reinterpret_cast<uintptr_t>(dev) & 15u) != 0) {
    h->err = "[rbt_bind_buffer] invalid argument: device buffer must be 16-byte aligned";
    return RBT_ERR_ARG;
  }
  d.bind->bound = dev;
  return RBT_OK;
}

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
  if (!h->wire_dirty && h->d_W.get()) return RBT_OK;
  std::vector<rbt_wire_layout> W;
  h->w_ocp = make_wire_layouts(h->S, h->ctrl.data(), h->n_grid, h->cost_structure, W);
  RBT_CUDA(h, h->d_W.ensure(size_t(h->n_grid_max)));
  RBT_CUDA(h, cudaMemcpy(h->d_W.get(), W.data(), size_t(h->n_grid) * sizeof(rbt_wire_layout), cudaMemcpyHostToDevice));
  h->wire_dirty = false;
  return RBT_OK;
}

// ---- host <-> device transfer plans -------------------------------------------------------------------------------------
// KKT upload: one strided copy of the core section [Fxx|Fvu|Fx|lx|lu|Qxx|Qxu|Quu] of every record (record padding and unused
// switching/STO sections never cross PCIe), plus one strided copy per stage that carries extras.
static std::vector<Copy> kkt_plan(const rbt_handle* h) {
  const rbt_layout& L = h->L;
  int n_extra = 0;
  for (const auto& c : h->ctrl) n_extra += (c.ns > 0 || c.sto) ? 1 : 0;
  const bool wide = n_extra * 2 > h->n_grid;  // most stages carry extras (STO horizons): copy core+extras in one go
  double* kkt = h->d_kkt.get();
  std::vector<Copy> v{{kkt, 0, size_t(wide ? L.k_core_size + L.k_extra_size : L.k_core_size), size_t(L.k_stride),
                       size_t(h->batch) * h->n_grid, true, IN_KKT}};
  if (!wide)
    for (int i = 0; i < h->n_grid; ++i)
      if (h->ctrl[i].ns > 0 || h->ctrl[i].sto)
        v.push_back({kkt, size_t(i) * L.k_stride + L.k_Phix, size_t(L.k_extra_size), size_t(L.k_stride) * h->n_grid,
                     size_t(h->batch), true, IN_KKT});
  return v;
}

// The copies of one host iteration of the stage layer over the batch window w, uploads first, in issue order.  Only what the
// kernels read / what persists crosses PCIe: record padding never does, the switching-constraint section of the linearization
// record only for the stages that carry one, of the PDIPM record slack | dual | residual go up and slack | dual come back.
enum { MODE_DENSE, MODE_WIRE, MODE_RESIDENT };  // rbt_iteration_host, _wire, _resident
static std::vector<Copy> iteration_plan(const rbt_handle* h, int mode, long long w_ocp, Win w) {
  const rbt_stage_layout& S = h->S;
  const size_t rows = size_t(w.nb) * h->n_grid, g0 = w.rec();
  std::vector<Copy> v;
  auto add = [&](double* dev, size_t off, size_t width, size_t pitch, size_t nrows, bool up, int host) {
    v.push_back({dev, off, width, pitch, nrows, up, host});
  };
  double *lin = h->d_lin.get(), *con = h->d_con.get(), *sol = h->d_sol.get();
  if (mode == MODE_DENSE) {
    const size_t tail = size_t(S.l_dgdf) + ((15 * S.ncon + 1) & ~1) - S.l_ha;
    add(lin, g0 * S.l_stride, S.l_Phix, S.l_stride, rows, true, IN_LIN);          // M .. se3
    add(lin, g0 * S.l_stride + S.l_ha, tail, S.l_stride, rows, true, IN_LIN);    // ha .. dgdf
  } else {
    add(h->d_wire.get(), size_t(w.b0) * w_ocp, w_ocp, w_ocp, w.nb, true, IN_WIRE);  // packed wire records: contiguous
  }
  for (int i = 0; i < h->n_grid; ++i)  // Phix, Phia, p, Phit of the stages with a switching constraint
    if (h->ctrl[i].ns > 0 && h->ctrl[i].type != RBT_IMPACT)
      add(lin, (g0 + i) * S.l_stride + S.l_Phix, S.l_ha - S.l_Phix, size_t(S.l_stride) * h->n_grid, w.nb, true, IN_LIN);
  if (mode == MODE_RESIDENT) {  // compact PDIPM residuals [batch][n_grid][ncp] (unpack_wire_kernel scatters them into c_res)
    add(h->d_res_stage.get(), g0 * S.ncp, S.ncp, S.ncp, rows, true, IN_RES);
  } else {
    add(con, g0 * S.c_stride + S.c_slack, 3 * size_t(S.ncp), S.c_stride, rows, true, IN_CON);
    // whole records incl. the few padding doubles: ONE contiguous DMA instead of a strided 2-D copy of 1.4 KB rows (the copy
    // engine spends as long per row as on ~4 KB of payload)
    add(sol, g0 * S.s_stride, S.s_stride, S.s_stride, rows, true, IN_SOL);
  }
  add(h->d_dx0.get(), size_t(w.b0) * h->L.nx, h->L.nx, h->L.nx, w.nb, true, IN_DX0);
  add(sol, g0 * S.s_stride, S.s_stride, S.s_stride, rows, false, OUT_SOL);
  if (mode == MODE_RESIDENT)  // compact slack | dual [batch][n_grid][2 ncp] (packed by pack_slack_dual_kernel): contiguous
    add(h->d_sd_stage.get(), g0 * 2 * S.ncp, 2 * size_t(S.ncp), 2 * size_t(S.ncp), rows, false, OUT_CON);
  else
    add(con, g0 * S.c_stride + S.c_slack, 2 * size_t(S.ncp), S.c_stride, rows, false, OUT_CON);
  add(h->d_steps.get(), 2 * size_t(w.b0), 2, 2, w.nb, false, OUT_STEPS);
  return v;
}

// The copies of rbt_upload into buffer `in` (IN_*), over the whole batch.
static std::vector<Copy> upload_plan(const rbt_handle* h, int in) {
  if (in == IN_KKT) return kkt_plan(h);
  if (in == IN_CPOS) {  // contiguous [batch][n_grid][n_contacts][3]
    const size_t n = size_t(h->batch) * h->n_grid * 3 * h->S.ncon;
    return {{h->d_cpos.get(), 0, n, n, 1, true, IN_CPOS}};
  }
  if (in == IN_Q0) {  // contiguous [batch][nq]
    const size_t n = size_t(h->batch) * h->S.nq;
    return {{h->d_q0.get(), 0, n, n, 1, true, IN_Q0}};
  }
  std::vector<Copy> v;
  for (const Copy& c : iteration_plan(h, MODE_DENSE, 0, full(h)))
    if (c.up && c.host == in) v.push_back(c);
  return v;
}

// Issues the copies of `plan` in one direction; a copy whose host array is null is skipped.  A contiguous copy is one
// linear DMA.
static int issue(rbt_handle* h, const std::vector<Copy>& plan, bool up, const double* const* in, double* const* out,
                 cudaStream_t st, const char* who) {
  for (const Copy& c : plan) {
    if (c.up != up || !(up ? in[c.host] : out[c.host])) continue;
    const size_t width = c.width * 8, pitch = c.pitch * 8;
    double* dev = c.dev + c.off;
    cudaError_t e;
    if (up) {
      const double* src = in[c.host] + c.off;
      e = pitch == width ? cudaMemcpyAsync(dev, src, width * c.rows, cudaMemcpyHostToDevice, st)
                         : cudaMemcpy2DAsync(dev, pitch, src, pitch, width, c.rows, cudaMemcpyHostToDevice, st);
    } else {
      double* dst = out[c.host] + c.off;
      e = pitch == width ? cudaMemcpyAsync(dst, dev, width * c.rows, cudaMemcpyDeviceToHost, st)
                         : cudaMemcpy2DAsync(dst, pitch, dev, pitch, width, c.rows, cudaMemcpyDeviceToHost, st);
    }
    if (e != cudaSuccess) {
      h->err = std::string(who) + ": " + cudaGetErrorString(e);
      return RBT_ERR_CUDA;
    }
  }
  return RBT_OK;
}

long long rbt_upload_bytes(rbt_handle* h, int which) {
  if (!h || h->n_grid == 0) return -1;
  const BufDesc d = buf(h, which);
  if (d.in < 0 || (d.stage && !h->stage_ready)) return -1;
  return plan_bytes(upload_plan(h, d.in), true);
}

int rbt_upload(rbt_handle* h, int which, const double* host, void* stream) {
  if (!h || !host) return RBT_ERR_ARG;
  const BufDesc d = buf(h, which);
  if (d.in < 0) return RBT_ERR_ARG;
  if (d.stage && !h->stage_ready) return RBT_ERR_STATE;
  if (h->n_grid == 0) return RBT_ERR_STATE;
  RBT_CUDA(h, cudaSetDevice(h->device));
  if (which == RBT_BUF_KKT) h->kkt_from_condense = false;
  if (which == RBT_BUF_CONTACT_POS) {
    RBT_CUDA(h, h->d_cpos.ensure(size_t(h->batch) * h->n_grid_max * 3 * h->S.ncon));
    h->cpos_set = true;
  }
  if (which == RBT_BUF_Q0) {
    RBT_CUDA(h, h->d_q0.ensure(size_t(h->batch) * h->S.nq));
    h->q0_set = true;
  }
  const double* in[N_IN] = {};
  in[d.in] = host;
  return issue(h, upload_plan(h, d.in), true, in, nullptr, (cudaStream_t)stream, "rbt_upload");
}

int rbt_download(rbt_handle* h, int which, double* host, void* stream) {
  if (!h || !host) return RBT_ERR_ARG;
  const BufDesc d = buf(h, which);
  if ((which == RBT_BUF_CONTACT_POS || which == RBT_BUF_Q0) && h->stage_ready && !d.ptr) {
    h->err = std::string("[rbt_download] ") + (which == RBT_BUF_Q0 ? "RBT_BUF_Q0" : "RBT_BUF_CONTACT_POS") +
             " has not been uploaded yet";
    return RBT_ERR_STATE;
  }
  if (!d.ptr) return RBT_ERR_ARG;
  if (h->n_grid == 0) return RBT_ERR_STATE;
  RBT_CUDA(h, cudaSetDevice(h->device));
  RBT_CUDA(h, cudaMemcpyAsync(host, d.ptr, size_t(buf_doubles(d, h->stage_ready, h->batch, h->n_grid)) * 8,
                              cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return RBT_OK;
}

int rbt_download_info(rbt_handle* h, int* host_flags, void* stream) {
  if (!h || !host_flags) return RBT_ERR_ARG;
  RBT_CUDA(h, cudaSetDevice(h->device));
  RBT_CUDA(h, cudaMemcpyAsync(host_flags, h->d_info.get(), size_t(h->batch) * sizeof(int), cudaMemcpyDeviceToHost,
                              (cudaStream_t)stream));
  return RBT_OK;
}

int rbt_check_info(rbt_handle* h, int* first_bad, void* stream) {
  if (!h) return RBT_ERR_ARG;
  RBT_CUDA(h, cudaSetDevice(h->device));
  std::vector<int> flags(size_t(h->batch), 0);
  RBT_CUDA(h, cudaMemcpyAsync(flags.data(), h->d_info.get(), flags.size() * sizeof(int), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
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

constexpr size_t TP_ESZ = rbt::TpElem<2 * CNV>::SIZE;

static int tp_ensure(rbt_handle* h, int S) {
  if (h->L.nx != 2 * CNV) {
    h->err = "internal: time-parallel element size";
    return RBT_ERR_STATE;
  }
  const size_t nx = h->L.nx, B = h->batch;
  RBT_CUDA(h, h->d_tp_elem.ensure(B * h->n_grid_max * TP_ESZ));
  if (!h->d_tp_fail.get()) RBT_CUDA(h, zeroed(h->d_tp_fail, B));
  for (DevBuf<double>& scan : h->d_tp_scan) RBT_CUDA(h, scan.ensure(B * (S + 1) * TP_ESZ));
  RBT_CUDA(h, h->d_tp_fmap.ensure(B * S * (nx * nx + nx)));
  RBT_CUDA(h, h->d_tp_dx.ensure(B * S * nx));
  return RBT_OK;
}

static rbt::TpParams tp_params(rbt_handle* h, int S, Win w) {
  rbt::TpParams q{};
  const size_t nx = h->L.nx;
  q.L = h->L;
  q.ctrl = h->d_ctrl.get();
  q.n_grid = h->n_grid;
  q.batch = w.nb;
  q.segs = S;
  q.kkt = h->d_kkt.get() + w.rec() * h->L.k_stride;
  q.ric = h->d_ric.get() + w.rec() * h->L.r_stride;
  q.elem = h->d_tp_elem.get() + w.rec() * TP_ESZ;
  q.fmap = h->d_tp_fmap.get() + size_t(w.b0) * S * (nx * nx + nx);
  q.dxseed = h->d_tp_dx.get() + size_t(w.b0) * S * nx;
  q.dx0 = h->d_dx0.get() + size_t(w.b0) * nx;
  q.fail = h->d_tp_fail.get() + w.b0;
  return q;
}

// Elements, in-segment reduction and suffix scan: returns (in h->tp_seeds) the scan buffer whose entry j + 1 is (P, s) at hi_j.
static int tp_backward_boundaries(rbt_handle* h, int S, Win w, cudaStream_t st) {
  constexpr int NX = 2 * CNV;
  using CC = rbt::TpCombCfg<NX>;
  if (!h->attr_tp) {
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::tp_combine_kernel<NX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CC::SMEM_BYTES));
    h->attr_tp = true;
  }
  const int nb = w.nb, N = h->n_grid - 1;
  rbt::TpParams q = tp_params(h, S, w);
  RBT_CUDA(h, cudaMemsetAsync(q.fail, 0, size_t(nb) * sizeof(int), st));
  rbt::tp_element_kernel<CNV, CNU, CNS><<<nb * h->n_grid, rbt::TpElemCfg<CNV, CNU, CNS>::NT, 0, st>>>(q);
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
    q.scan_in = h->d_tp_scan[cur ^ 1].get() + size_t(w.b0) * (S + 1) * TP_ESZ;
    q.scan_out = h->d_tp_scan[cur].get() + size_t(w.b0) * (S + 1) * TP_ESZ;
    rbt::tp_combine_kernel<NX><<<nb * (S + 1), CC::NT, CC::SMEM_BYTES, st>>>(q);
    h->launches += 1;
    q.gather = 0;
    cur ^= 1;
  }
  h->tp_seeds = h->d_tp_scan[cur ^ 1].get();
  RBT_CUDA(h, cudaGetLastError());
  return RBT_OK;
}

static int backward(rbt_handle* h, int write_fact, Win w, cudaStream_t st) {
  using C = rbt::BwdCfg<CNV, CNU, CNS, CNP>;
  if (C::STAGE != h->L.k_stage_size || C::EXTRA != h->L.k_extra_size) {
    h->err = "internal: shared-memory staging size does not match rbt_layout";
    return RBT_ERR_STATE;
  }
  const int S = tp_segments(h);
  auto kern_s = S > 1 ? rbt::riccati_backward_kernel<CNV, CNU, CNS, CNP, true, true>   // Fqq = I, Fqv = dt I outside the floating-base blocks
                      : rbt::riccati_backward_kernel<CNV, CNU, CNS, CNP, true>;
  auto kern_g = S > 1 ? rbt::riccati_backward_kernel<CNV, CNU, CNS, CNP, false, true>  // any Fxx
                      : rbt::riccati_backward_kernel<CNV, CNU, CNS, CNP, false>;
  if (!h->attr_bwd) {  // the attribute is per device: tracked per handle (a handle lives on one device)
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::riccati_backward_kernel<CNV, CNU, CNS, CNP, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::riccati_backward_kernel<CNV, CNU, CNS, CNP, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::riccati_backward_kernel<CNV, CNU, CNS, CNP, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::riccati_backward_kernel<CNV, CNU, CNS, CNP, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    h->attr_bwd = true;
  }
  rbt::BwdParams p{};  // CTA de-phasing and the timeline stamps stay off
  p.L = h->L;
  p.ctrl = h->d_ctrl.get();
  p.n_grid = h->n_grid;
  p.batch = w.nb;
  p.max_dts0 = h->max_dts0;
  p.kkt = h->d_kkt.get() + w.rec() * h->L.k_stride;
  p.ric = h->d_ric.get() + w.rec() * h->L.r_stride;
  p.fact = write_fact ? h->d_fact.get() + w.rec() * h->L.f_stride : nullptr;
  p.info = h->d_info.get() + w.b0;
  p.segs = S;
  const int grid = w.nb * S;
  if (S > 1) {
    int rc = tp_ensure(h, S);
    if (!rc) rc = tp_backward_boundaries(h, S, w, st);
    if (rc) return rc;
    p.seeds = h->tp_seeds + size_t(w.b0) * (S + 1) * TP_ESZ;
    p.tp_fail = h->d_tp_fail.get() + w.b0;
  }
  if (!h->keep_info) RBT_CUDA(h, cudaMemsetAsync(p.info, 0, size_t(w.nb) * sizeof(int), st));
  h->keep_info = false;
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
    RBT_CUDA(h, cudaMemsetAsync(h->d_struct.get(), 0, 2 * sizeof(int), st));
    rbt::check_fxx_structure_kernel<CNV, CNP><<<(w.nb * (h->n_grid - 1) + 7) / 8, 256, 0, st>>>(p, h->d_struct.get());
    p.struct_flag = h->d_struct.get();
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

static int forward(rbt_handle* h, Win w, cudaStream_t st) {
  using C = rbt::FwdCfg<CNV, CNU, CNS>;
  using TF = rbt::TpFwdCfg<CNV, CNU>;
  const int S = tp_segments(h);
  auto kern = S > 1 ? rbt::riccati_forward_kernel<CNV, CNU, CNS, true> : rbt::riccati_forward_kernel<CNV, CNU, CNS>;
  if (!h->attr_fwd) {
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::riccati_forward_kernel<CNV, CNU, CNS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::riccati_forward_kernel<CNV, CNU, CNS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    RBT_CUDA(h, cudaFuncSetAttribute(rbt::tp_fwd_compose_kernel<CNV, CNU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TF::SMEM_BYTES));
    h->attr_fwd = true;
  }
  rbt::FwdParams p;
  p.L = h->L;
  p.ctrl = h->d_ctrl.get();
  p.n_grid = h->n_grid;
  p.batch = w.nb;
  p.kkt = h->d_kkt.get() + w.rec() * h->L.k_stride;
  p.ric = h->d_ric.get() + w.rec() * h->L.r_stride;
  p.dx0 = h->d_dx0.get() + size_t(w.b0) * h->L.nx;
  p.dir = h->d_dir.get() + w.rec() * h->L.d_stride;
  p.segs = S;
  p.dxseed = nullptr;
  p.tp_fail = nullptr;
  if (S > 1) {
    // the backward sweep of this handle ran segmented too (same rule, same handle): its failure flags are current
    if (int rc = tp_ensure(h, S)) return rc;
    rbt::TpParams q = tp_params(h, S, w);
    rbt::tp_fwd_compose_kernel<CNV, CNU><<<w.nb * (S - 1), TF::NT, TF::SMEM_BYTES, st>>>(q);
    rbt::tp_fwd_boundary_kernel<2 * CNV><<<w.nb, 64, 0, st>>>(q);
    h->launches += 2;
    p.dxseed = q.dxseed;
    p.tp_fail = q.fail;
  }
  kern<<<w.nb * S, C::NTHREADS, C::SMEM_BYTES, st>>>(p);
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
  return backward(h, write_fact, full(h), (cudaStream_t)stream);
}

int rbt_riccati_forward(rbt_handle* h, void* stream) {
  if (!h) return RBT_ERR_ARG;
  if (h->n_grid == 0) {
    h->err = "[rbt_riccati_forward] no schedule set";
    return RBT_ERR_STATE;
  }
  RBT_CUDA(h, cudaSetDevice(h->device));
  return forward(h, full(h), (cudaStream_t)stream);
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
  if (3 * sd->nv + sd->nu > RBT_MAX_TARGETS) {
    h->err = "[rbt_stage_setup] invalid argument: too many limit targets";
    return RBT_ERR_ARG;
  }
  // box rows acting on each target entry (var, idx), in ascending row order (deterministic accumulation on the device):
  // entry = (row + 1) * sign, 0 = none.  Device memory, not kernel parameters: the lanes of a warp look up different targets,
  // and a divergent constant-bank access is serialised.  It is followed by the level of every box row (2 = position,
  // 1 = velocity, 0 = acceleration / torque): a row acts on a grid point iff level + ineq_gate <= 2 (ConstraintsData::setTimeStage)
  int tgt[RBT_MAX_TARGETS * 4 + RBT_MAX_BOX_ROWS] = {};
  for (int r = 0; r < table->n_box; ++r) {
    const rbt_box_row& b = table->box[r];
    int* t = tgt + 4 * ((b.var == RBT_VAR_U) ? 3 * sd->nv + b.idx : b.var * sd->nv + b.idx);
    int q = 0;
    while (q < 4 && t[q] != 0) ++q;
    if (q == 4) {
      h->err = "[rbt_stage_setup] invalid argument: more than 4 box rows on one variable";
      return RBT_ERR_ARG;
    }
    t[q] = (r + 1) * (b.sign < 0 ? -1 : 1);
    tgt[RBT_MAX_TARGETS * 4 + r] = b.var == RBT_VAR_Q ? 2 : (b.var == RBT_VAR_V ? 1 : 0);
  }
  if (h->stage_ready) {  // a caller-bound stage buffer is sized for the records of the first table
    h->err = "[rbt_stage_setup] already set up on this handle (create a new handle for another constraint table)";
    return RBT_ERR_STATE;
  }
  if (h->n_grid > 0 && check_contacts(h, *sd, h->ctrl.data(), h->n_grid) != RBT_OK) return RBT_ERR_ARG;
  rbt_stage_layout S;
  rbt_make_stage_layout(sd, &S);
  {  // condense_kernel lands [l_D, l_Phix) and [l_ha, l_dgdq) of the record in place: the static mirror must match
    using C = rbt::CondCfg<CNV, CNU, CNS>;
    using MC = rbt::MjtjCfg<CNV, CNU>;
    const int gsz = (S.l_dgdf - S.l_dgdq) + ((15 * S.ncon + 1) & ~1);
    const int q0 = S.l_Quu - C::IN1A;  // record offset that maps onto the second in-place mirror
    const bool ok = S.l_Qxx - S.l_D == C::IN1A && S.l_Phix - S.l_Quu == C::IN1B && S.l_IDC - S.l_D == C::i_IDC &&
                    S.l_Qaa - S.l_D == C::i_Qaa && S.l_Qff - S.l_D == C::i_Qff && S.l_Qqf - S.l_D == C::i_Qqf &&
                    S.l_lx - q0 == C::i_lx && S.l_la - q0 == C::i_la && S.l_lf - q0 == C::i_lf && S.l_lu - q0 == C::i_lu &&
                    S.l_Fx - q0 == C::i_Fx && S.l_lup - q0 == C::i_lup && S.l_se3 - q0 == C::i_se3 && S.l_dgdq - S.l_ha == C::IN2 &&
                    S.l_hf - S.l_ha == C::j_hf && S.l_hx - S.l_ha == C::j_hx && S.l_hu - S.l_ha == C::j_hu &&
                    S.l_fx - S.l_ha == C::j_fx && S.l_sc - S.l_ha == C::j_sc &&
                    5 * S.ncp + gsz <= C::NVF * C::NX &&  // PDIPM staging fits in the R buffer
                    S.l_J - S.l_M == MC::o_J && S.l_D - S.l_M == MC::MJ;
    if (!ok) {
      h->err = "[rbt_stage_setup] invalid argument: stage layout not supported by the compiled condensing kernel";
      return RBT_ERR_ARG;
    }
  }
  if (S.ncp > 160 || S.l_stride - S.l_dgdq > 512) {  // shared-memory staging areas of expand_kernel
    h->err = "[rbt_stage_setup] invalid argument: more than 160 inequality rows or more than 4 friction cones";
    return RBT_ERR_ARG;
  }
  // everything is allocated before anything is committed: a failed setup leaves the handle as it was
  RBT_CUDA(h, cudaSetDevice(h->device));
  const size_t per = size_t(h->batch) * h->n_grid_max, B = h->batch;
  DevBuf<double> lin, con, ex, sol, xd, steps, ones, stage_perf, perf, x0in;
  DevBuf<int> d_tgt;
  RBT_CUDA(h, zeroed(lin, per * S.l_stride));  // uploads skip record padding: keep it defined
  RBT_CUDA(h, zeroed(con, per * S.c_stride));
  RBT_CUDA(h, zeroed(ex, per * S.e_stride));
  RBT_CUDA(h, zeroed(sol, per * S.s_stride));
  RBT_CUDA(h, zeroed(xd, per * S.x_stride));
  RBT_CUDA(h, steps.ensure(B * 2));
  RBT_CUDA(h, ones.ensure(B * 2));
  RBT_CUDA(h, stage_perf.ensure(per * 4));
  RBT_CUDA(h, zeroed(perf, B * 8));
  RBT_CUDA(h, x0in.ensure(B * 2 * h->dims.nv));
  RBT_CUDA(h, d_tgt.ensure(sizeof(tgt) / sizeof(int)));
  RBT_CUDA(h, cudaMemcpy(d_tgt.get(), tgt, sizeof(tgt), cudaMemcpyHostToDevice));
  const std::vector<double> one(B * 2, 1.0);
  RBT_CUDA(h, cudaMemcpy(ones.get(), one.data(), one.size() * 8, cudaMemcpyHostToDevice));
  RBT_CUDA(h, cudaMemcpy(steps.get(), one.data(), one.size() * 8, cudaMemcpyHostToDevice));
  h->sdims = *sd;
  h->table = *table;
  h->S = S;
  h->d_lin.own = std::move(lin);
  h->d_con.own = std::move(con);
  h->d_ex.own = std::move(ex);
  h->d_sol.own = std::move(sol);
  h->d_xd.own = std::move(xd);
  h->d_steps = std::move(steps);
  h->d_ones = std::move(ones);
  h->d_stage_perf = std::move(stage_perf);
  h->d_perf = std::move(perf);
  h->d_x0in = std::move(x0in);
  h->d_tgt = std::move(d_tgt);
  h->stage_ready = true;
  return RBT_OK;
}

static rbt::StageParams make_stage_params(rbt_handle* h, Win w) {
  rbt::StageParams p;
  const rbt_stage_layout& S = h->S;
  const size_t g0 = w.rec();
  p.K = h->L;
  p.S = S;
  p.tab = h->table;
  p.ctrl = h->d_ctrl.get();
  p.n_grid = h->n_grid;
  p.batch = w.nb;
  p.lin = h->d_lin.get() + g0 * S.l_stride;
  p.con = h->d_con.get() + g0 * S.c_stride;
  p.kkt = h->d_kkt.get() + g0 * h->L.k_stride;
  p.ex = h->d_ex.get() + g0 * S.e_stride;
  p.dir = h->d_dir.get() + g0 * h->L.d_stride;
  p.xd = h->d_xd.get() + g0 * S.x_stride;
  p.sol = h->d_sol.get() + g0 * S.s_stride;
  p.steps = h->d_steps.get() + 2 * size_t(w.b0);
  p.info = h->d_info.get() + w.b0;
  p.tgt = reinterpret_cast<const int4*>(h->d_tgt.get());
  p.row_level = h->d_tgt.get() + RBT_MAX_TARGETS * 4;
  return p;
}

#define RBT_STAGE_CHECK(h, what)                                  \
  if (!(h)) return RBT_ERR_ARG;                                   \
  if (!(h)->stage_ready || (h)->n_grid == 0) {                    \
    (h)->err = "[" what "] stage layer not set up / no schedule"; \
    return RBT_ERR_STATE;                                         \
  }                                                               \
  RBT_CUDA(h, cudaSetDevice((h)->device));

static int condense(rbt_handle* h, Win w, cudaStream_t st) {
  using C = rbt::CondCfg<CNV, CNU, CNS>;
  auto kern = rbt::condense_kernel<CNV, CNU, CNS>;
  if (!h->attr_cond) {
    RBT_CUDA(h, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM_BYTES));
    h->attr_cond = true;
  }
  RBT_CUDA(h, cudaMemsetAsync(h->d_info.get() + w.b0, 0, size_t(w.nb) * sizeof(int), st));
  rbt::mjtjinv_kernel<CNV, CNU><<<(w.nb * h->n_grid + 1) / 2, 64, 0, st>>>(make_stage_params(h, w));  // K1: Z = [[M,J^T],[J,0]]^-1
  RBT_CUDA(h, cudaGetLastError());
  if (h->ev_condense_mid) RBT_CUDA(h, cudaEventRecord(h->ev_condense_mid, st));
  kern<<<w.nb * h->n_grid, C::NTHREADS, C::SMEM_BYTES, st>>>(make_stage_params(h, w));          // K2: condensing (DMMA)
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 2;
  h->keep_info = true;
  h->kkt_from_condense = true;
  return RBT_OK;
}

int rbt_condense(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_condense");
  return condense(h, full(h), (cudaStream_t)stream);
}

int rbt_set_condense_event(rbt_handle* h, void* cuda_event) {
  if (!h) return RBT_ERR_ARG;
  h->ev_condense_mid = (cudaEvent_t)cuda_event;
  return RBT_OK;
}

static int expand(rbt_handle* h, Win w, cudaStream_t st) {
  RBT_CUDA(h, cudaMemcpyAsync(h->d_steps.get() + 2 * size_t(w.b0), h->d_ones.get(), size_t(w.nb) * 2 * 8, cudaMemcpyDeviceToDevice, st));
  rbt::expand_kernel<CNV, CNU, CNS><<<w.nb * h->n_grid, rbt::XTHR, 0, st>>>(make_stage_params(h, w));
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

int rbt_expand_and_step_sizes(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_expand_and_step_sizes");
  return expand(h, full(h), (cudaStream_t)stream);
}

static int update(rbt_handle* h, Win w, cudaStream_t st) {
  rbt::update_kernel<CNV, CNU, CNS><<<w.nb * h->n_grid, rbt::XTHR, 0, st>>>(make_stage_params(h, w));
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

int rbt_update(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_update");
  return update(h, full(h), (cudaStream_t)stream);
}

static rbt::EvalParams make_eval_params(rbt_handle* h, Win w) {
  rbt::EvalParams q;
  q.sp = make_stage_params(h, w);
  q.stage_perf = h->d_stage_perf.get() + w.rec() * 4;
  q.perf = h->d_perf.get() + size_t(w.b0) * 8;
  q.x0in = h->d_x0in.get() + size_t(w.b0) * 2 * h->dims.nv;
  q.dx0 = h->d_dx0.get() + size_t(w.b0) * h->L.nx;
  return q;
}

int rbt_eval_kkt(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_eval_kkt");
  cudaStream_t st = (cudaStream_t)stream;
  const rbt::EvalParams q = make_eval_params(h, full(h));
  rbt::perf_index_kernel<<<(h->batch * h->n_grid + 3) / 4, 128, 0, st>>>(q);
  rbt::perf_reduce_kernel<<<(h->batch + 127) / 128, 128, 0, st>>>(q);
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 2;
  return RBT_OK;
}

int rbt_set_slack_and_dual_positive(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_set_slack_and_dual_positive");
  const rbt::EvalParams q = make_eval_params(h, full(h));
  const long long total = (long long)h->batch * h->n_grid * h->S.ncp;
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
  RBT_CUDA(h, h->d_limits.ensure(RBT_MAX_BOX_ROWS));
  RBT_CUDA(h, cudaMemcpy(h->d_limits.get(), bound_host, sizeof(double) * h->table.n_box, cudaMemcpyHostToDevice));
  return RBT_OK;
}

int rbt_linearize_joint_limits(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_linearize_joint_limits");
  if (!h->d_limits.get()) {
    h->err = "[rbt_linearize_joint_limits] call rbt_set_joint_limits first";
    return RBT_ERR_STATE;
  }
  const rbt::EvalParams q = make_eval_params(h, full(h));
  const long long total = (long long)h->batch * h->n_grid * (3 * h->S.nv + h->S.nu);
  rbt::linearize_joint_limits_kernel<<<unsigned((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(q, h->d_limits.get());
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
  RBT_CUDA(h, h->d_model.ensure(1));
  RBT_CUDA(h, cudaMemcpy(h->d_model.get(), &d, sizeof(rbt::RneaModel), cudaMemcpyHostToDevice));
  return RBT_OK;
}

static int inverse_dynamics(rbt_handle* h, Win w, cudaStream_t st) {
  rbt::linearize_inverse_dynamics_kernel<CNV><<<w.nb * h->n_grid, rbt::RneaCfg<CNV>::NTHR, 0, st>>>(make_stage_params(h, w),
                                                                                                 h->d_model.get());
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

int rbt_linearize_inverse_dynamics(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_linearize_inverse_dynamics");
  if (!h->d_model.get()) {
    h->err = "[rbt_linearize_inverse_dynamics] call rbt_set_robot_model first";
    return RBT_ERR_STATE;
  }
  return inverse_dynamics(h, full(h), (cudaStream_t)stream);
}

int rbt_set_contact_gains(rbt_handle* h, const double* gains_host) {
  if (!h || !gains_host) return RBT_ERR_ARG;
  if (!h->stage_ready) {
    h->err = "[rbt_set_contact_gains] stage layer not set up";
    return RBT_ERR_STATE;
  }
  for (int e = 0; e < 2 * h->S.ncon; ++e)
    if (!(gains_host[e] >= 0.0 && gains_host[e] < HUGE_VAL)) {
      h->err = "[rbt_set_contact_gains] invalid argument: contact " + std::to_string(e / 2) +
               (e % 2 ? ": velocity" : ": position") + " gain must be finite and non-negative";
      return RBT_ERR_ARG;
    }
  RBT_CUDA(h, cudaSetDevice(h->device));
  RBT_CUDA(h, h->d_gains.ensure(2 * RBT_MAX_CONTACTS));
  RBT_CUDA(h, cudaMemcpy(h->d_gains.get(), gains_host, sizeof(double) * 2 * h->S.ncon, cudaMemcpyHostToDevice));
  return RBT_OK;
}

// what rbt_linearize_contact_kinematics needs besides the stage layer: the model, the gains and the desired positions
static const char* contact_kinematics_missing(const rbt_handle* h) {
  if (!h->d_model.get()) return "call rbt_set_robot_model first";
  if (!h->d_gains.get()) return "call rbt_set_contact_gains first";
  if (!h->cpos_set) return "upload RBT_BUF_CONTACT_POS first";
  return nullptr;
}

static int contact_kinematics(rbt_handle* h, Win w, cudaStream_t st) {
  rbt::linearize_contact_kinematics_kernel<CNV><<<w.nb * h->n_grid, rbt::ContactCfg<CNV>::NTHR, 0, st>>>(
      make_stage_params(h, w), h->d_model.get(), h->d_gains.get(), h->d_cpos.get() + w.rec() * 3 * h->S.ncon);
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

int rbt_linearize_contact_kinematics(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_linearize_contact_kinematics");
  if (const char* why = contact_kinematics_missing(h)) {
    h->err = std::string("[rbt_linearize_contact_kinematics] ") + why;
    return RBT_ERR_STATE;
  }
  return contact_kinematics(h, full(h), (cudaStream_t)stream);
}

static int state_equation(rbt_handle* h, Win w, cudaStream_t st) {
  constexpr int NW = rbt::StateCfg::NW;
  const unsigned n = unsigned((size_t(w.nb) * h->n_grid + NW - 1) / NW);
  rbt::linearize_state_equation_kernel<CNV><<<n, 32 * NW, 0, st>>>(make_stage_params(h, w), h->d_q0.get() + size_t(w.b0) * h->S.nq,
                                                                   ctrl_has_sto(h->ctrl.data(), h->n_grid));
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

int rbt_linearize_state_equation(rbt_handle* h, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_linearize_state_equation");
  if (!h->q0_set) {
    h->err = "[rbt_linearize_state_equation] upload RBT_BUF_Q0 first";
    return RBT_ERR_STATE;
  }
  return state_equation(h, full(h), (cudaStream_t)stream);
}

int rbt_initial_state_direction(rbt_handle* h, const double* dq0_v0_host, void* stream) {
  RBT_STAGE_CHECK(h, "rbt_initial_state_direction");
  if (!dq0_v0_host) return RBT_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  RBT_CUDA(h, cudaMemcpyAsync(h->d_x0in.get(), dq0_v0_host, size_t(h->batch) * 2 * h->dims.nv * 8, cudaMemcpyHostToDevice, st));
  const rbt::EvalParams q = make_eval_params(h, full(h));
  const int total = h->batch * h->L.nx;
  rbt::initial_state_direction_kernel<<<(total + 127) / 128, 128, 0, st>>>(q);
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

// ---- line search: trial step sizes as an extra batch axis -------------------------------------------------------------------
enum { RBT_LS_FILTER_CAP = 16 };

static int ls_ensure(rbt_handle* h, int n_trials) {
  if (n_trials <= h->ls_trials) return RBT_OK;
  const size_t kb = size_t(n_trials) * h->batch, B = h->batch;
  RBT_CUDA(h, h->d_ls_alphas.ensure(kb));
  RBT_CUDA(h, h->d_ls_barrier.ensure(kb));
  RBT_CUDA(h, h->d_ls_stage_barrier.ensure(kb * h->n_grid_max));
  RBT_CUDA(h, h->d_ls_trial.ensure(kb * h->n_grid_max * rbt::T_STRIDE));
  RBT_CUDA(h, h->d_ls_in.ensure(2 * kb + 2 * B));  // cost | viol of the trials, cost0 | viol0
  if (!h->d_ls_nfilt.get()) {
    RBT_CUDA(h, h->d_ls_filt.ensure(B * 2 * RBT_LS_FILTER_CAP));
    RBT_CUDA(h, h->d_ls_step.ensure(B));
    RBT_CUDA(h, h->d_ls_k.ensure(B));
    RBT_CUDA(h, zeroed(h->d_ls_nfilt, B));
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
  q.sp = make_stage_params(h, full(h));
  q.n_trials = n_trials;
  q.rate = step_size_reduction_rate;
  q.alphas = h->d_ls_alphas.get();
  q.trial = h->d_ls_trial.get();
  q.stage_barrier = h->d_ls_stage_barrier.get();
  q.barrier = h->d_ls_barrier.get();
  const long long warps = (long long)n_trials * h->batch * h->n_grid;
  rbt::trial_solution_kernel<<<unsigned((warps + 3) / 4), 128, 0, st>>>(q);
  rbt::trial_reduce_kernel<<<(n_trials * h->batch + 127) / 128, 128, 0, st>>>(q);
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 2;
  const size_t kb = size_t(n_trials) * h->batch;
  if (alphas_host) RBT_CUDA(h, cudaMemcpyAsync(alphas_host, h->d_ls_alphas.get(), kb * 8, cudaMemcpyDeviceToHost, st));
  if (barrier_host) RBT_CUDA(h, cudaMemcpyAsync(barrier_host, h->d_ls_barrier.get(), kb * 8, cudaMemcpyDeviceToHost, st));
  if (trial_host) RBT_CUDA(h, cudaMemcpyAsync(trial_host, h->d_ls_trial.get(), kb * h->n_grid * rbt::T_STRIDE * 8, cudaMemcpyDeviceToHost, st));
  return RBT_OK;
}

double* rbt_line_search_trial_dev(rbt_handle* h) { return h ? h->d_ls_trial.get() : nullptr; }

int rbt_line_search_clear_history(rbt_handle* h, void* stream) {
  if (!h) return RBT_ERR_ARG;
  if (h->d_ls_nfilt.get()) RBT_CUDA(h, cudaMemsetAsync(h->d_ls_nfilt.get(), 0, size_t(h->batch) * sizeof(int), (cudaStream_t)stream));
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
  double* d_cost = h->d_ls_in.get();
  double* d_viol = h->d_ls_in.get() + size_t(h->ls_trials) * h->batch;
  double* d_c0 = h->d_ls_in.get() + 2 * size_t(h->ls_trials) * h->batch;
  double* d_v0 = d_c0 + h->batch;
  RBT_CUDA(h, cudaMemcpyAsync(d_cost, cost_host, kb * 8, cudaMemcpyHostToDevice, st));
  RBT_CUDA(h, cudaMemcpyAsync(d_viol, violation_host, kb * 8, cudaMemcpyHostToDevice, st));
  RBT_CUDA(h, cudaMemcpyAsync(d_c0, cost0_host, size_t(h->batch) * 8, cudaMemcpyHostToDevice, st));
  RBT_CUDA(h, cudaMemcpyAsync(d_v0, violation0_host, size_t(h->batch) * 8, cudaMemcpyHostToDevice, st));
  rbt::FilterParams q;
  q.batch = h->batch; q.n_trials = n_trials; q.cap = RBT_LS_FILTER_CAP;
  q.rate = step_size_reduction_rate; q.min_step = min_step_size;
  q.cost_rate = filter_cost_reduction_rate; q.viol_rate = filter_constraint_violation_reduction_rate;
  q.steps = h->d_steps.get(); q.cost0 = d_c0; q.viol0 = d_v0; q.cost = d_cost; q.barrier = h->d_ls_barrier.get(); q.viol = d_viol;
  q.filt = h->d_ls_filt.get(); q.nfilt = h->d_ls_nfilt.get(); q.out_step = h->d_ls_step.get(); q.out_k = h->d_ls_k.get();
  rbt::line_search_filter_kernel<<<(h->batch + 127) / 128, 128, 0, st>>>(q);
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  if (step_host) RBT_CUDA(h, cudaMemcpyAsync(step_host, h->d_ls_step.get(), size_t(h->batch) * 8, cudaMemcpyDeviceToHost, st));
  if (accepted_trial_host) RBT_CUDA(h, cudaMemcpyAsync(accepted_trial_host, h->d_ls_k.get(), size_t(h->batch) * sizeof(int), cudaMemcpyDeviceToHost, st));
  return RBT_OK;
}

int rbt_iteration_host_bytes(rbt_handle* h, int wire, long long* h2d, long long* d2h) {
  if (!h || !h->stage_ready || h->n_grid == 0) return RBT_ERR_STATE;
  const int mode = wire == 2 ? MODE_RESIDENT : (wire ? MODE_WIRE : MODE_DENSE);
  std::vector<rbt_wire_layout> W;
  const long long w_ocp = make_wire_layouts(h->S, h->ctrl.data(), h->n_grid, h->cost_structure, W);
  const std::vector<Copy> plan = iteration_plan(h, mode, w_ocp, full(h));
  if (h2d) *h2d = plan_bytes(plan, true);
  if (d2h) *d2h = plan_bytes(plan, false);
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
    if ((h->cost_structure & RBT_WIRE_DEVICE_ID) && !h->d_model.get()) {
      h->err = "[rbt_iteration_host_wire] the wire records leave the inverse dynamics to the device: call rbt_set_robot_model first";
      return RBT_ERR_STATE;
    }
    if (h->cost_structure & RBT_WIRE_DEVICE_CONTACT) {
      if (const char* why = contact_kinematics_missing(h)) {
        h->err = std::string("[rbt_iteration_host_wire] the wire records leave the contact rows to the device: ") + why;
        return RBT_ERR_STATE;
      }
    }
    if ((h->cost_structure & RBT_WIRE_DEVICE_STATE) && !h->q0_set) {
      h->err = "[rbt_iteration_host_wire] the wire records leave the state equation to the device: upload RBT_BUF_Q0 first";
      return RBT_ERR_STATE;
    }
    if (sw && !lin_host) {
      h->err = "[rbt_iteration_host_wire] invalid argument: the schedule has switching-constraint stages, their sections come from lin_host_switching";
      return RBT_ERR_ARG;
    }
    if (!h->d_wire.get()) {  // sized for the largest possible record at every grid point
      rbt_wire_layout wmax;
      rbt_stage_ctrl cmax = {};
      cmax.type = RBT_INTERMEDIATE; cmax.nf = h->S.nfm; cmax.contact_mask = (1 << h->S.ncon) - 1;
      rbt_make_wire_layout(&h->S, &cmax, 1, RBT_COST_GENERAL, &wmax);
      RBT_CUDA(h, h->d_wire.ensure(size_t(h->batch) * h->n_grid_max * wmax.w_doubles));
    }
    if (res_host) {
      RBT_CUDA(h, h->d_res_stage.ensure(size_t(h->batch) * h->n_grid_max * h->S.ncp));
      RBT_CUDA(h, h->d_sd_stage.ensure(size_t(h->batch) * h->n_grid_max * 2 * h->S.ncp));
    }
  }
  const int mode = res_host ? MODE_RESIDENT : (wire_host ? MODE_WIRE : MODE_DENSE);
  const double* in[N_IN] = {};
  in[IN_WIRE] = wire_host; in[IN_LIN] = lin_host; in[IN_CON] = con_host; in[IN_SOL] = sol_host; in[IN_RES] = res_host;
  in[IN_DX0] = dx0_host;
  double* out[N_OUT] = {sol_out, con_out, steps_out};
  cudaStream_t st = (cudaStream_t)stream;
  // chunks of the batch: the upload of chunk c+1, the kernels of chunk c and the download of chunk c-1 overlap
  int n_chunks = h->batch >= 512 ? 8 : (h->batch >= 128 ? 4 : 1);
  if (const char* e = getenv("RBT_E2E_CHUNKS")) n_chunks = std::max(1, std::min(atoi(e), h->batch));
  for (Stream* s : {&h->s_h2d, &h->s_d2h})
    if (!s->get()) RBT_CUDA(h, cudaStreamCreateWithFlags(s->out(), cudaStreamNonBlocking));
  while ((int)h->ev.size() < 2 * n_chunks + 2) {
    Event e;
    RBT_CUDA(h, cudaEventCreateWithFlags(e.out(), cudaEventDisableTiming));
    h->ev.push_back(std::move(e));
  }
  cudaStream_t s_h2d = h->s_h2d.get(), s_d2h = h->s_d2h.get();
  cudaEvent_t ev_entry = h->ev[2 * n_chunks].get(), ev_exit = h->ev[2 * n_chunks + 1].get();
  RBT_CUDA(h, cudaEventRecord(ev_entry, st));            // device buffers may still be read by earlier work on `stream`
  RBT_CUDA(h, cudaStreamWaitEvent(s_h2d, ev_entry, 0));
  RBT_CUDA(h, cudaStreamWaitEvent(s_d2h, ev_entry, 0));
  const rbt_stage_layout& S = h->S;
  for (int c = 0; c < n_chunks; ++c) {
    const int b0 = int((long long)h->batch * c / n_chunks), b1 = int((long long)h->batch * (c + 1) / n_chunks);
    if (b1 <= b0) continue;
    const Win w{b0, b1 - b0, h->n_grid};
    const std::vector<Copy> plan = iteration_plan(h, mode, h->w_ocp, w);
    int rc = issue(h, plan, true, in, out, s_h2d, "rbt_iteration_host");
    if (rc) return rc;
    RBT_CUDA(h, cudaEventRecord(h->ev[2 * c].get(), s_h2d));
    RBT_CUDA(h, cudaStreamWaitEvent(st, h->ev[2 * c].get(), 0));
    if (wire_host) {  // expand the packed records of this chunk into the linearization records
      rbt::WireParams wp;
      wp.W = h->d_W.get();
      wp.n_grid = h->n_grid;
      wp.ocp_stride = h->w_ocp;
      wp.l_stride = S.l_stride;
      wp.wire = h->d_wire.get() + size_t(b0) * h->w_ocp;
      wp.lin = h->d_lin.get() + w.rec() * S.l_stride;
      wp.res = res_host ? h->d_res_stage.get() + w.rec() * S.ncp : nullptr;
      wp.con = h->d_con.get() + w.rec() * S.c_stride;
      wp.c_stride = S.c_stride; wp.c_res = S.c_res; wp.ncp = S.ncp;
      rbt::unpack_wire_kernel<<<w.nb * h->n_grid, 128, 0, st>>>(wp);
      h->launches += 1;
      if ((h->cost_structure & RBT_WIRE_DEVICE_ID) && (rc = inverse_dynamics(h, w, st))) return rc;
      if ((h->cost_structure & RBT_WIRE_DEVICE_CONTACT) && (rc = contact_kinematics(h, w, st))) return rc;
      if ((h->cost_structure & RBT_WIRE_DEVICE_STATE) && (rc = state_equation(h, w, st))) return rc;
    }
    if ((rc = condense(h, w, st)) || (rc = backward(h, 0, w, st)) || (rc = forward(h, w, st)) || (rc = expand(h, w, st)) ||
        (rc = update(h, w, st)))
      return rc;
    if (res_host && con_out) {
      rbt::pack_slack_dual_kernel<<<w.nb * h->n_grid, 64, 0, st>>>(h->d_con.get() + w.rec() * S.c_stride, S.c_stride, S.c_slack,
                                                                   2 * S.ncp, h->d_sd_stage.get() + w.rec() * 2 * S.ncp);
      h->launches += 1;
    }
    RBT_CUDA(h, cudaEventRecord(h->ev[2 * c + 1].get(), st));
    RBT_CUDA(h, cudaStreamWaitEvent(s_d2h, h->ev[2 * c + 1].get(), 0));
    if ((rc = issue(h, plan, false, in, out, s_d2h, "rbt_iteration_host"))) return rc;
  }
  RBT_CUDA(h, cudaEventRecord(ev_exit, s_d2h));       // `stream` (what the caller synchronizes) covers the downloads too
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
  if (!h || (cost_structure & ~(RBT_COST_ROBOTOC | RBT_WIRE_DEVICE_ID | RBT_WIRE_DEVICE_CONTACT | RBT_WIRE_DEVICE_STATE)) != 0)
    return RBT_ERR_ARG;
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
  pack_step_kernel<<<unsigned((n_rec * step + 255) / 256), 256, 0, (cudaStream_t)stream>>>(h->d_dir.get(), packed_dev, h->L.d_stride, step, n_rec);
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
  RBT_CUDA(h, h->d_step_pack.ensure(size_t(h->batch) * h->n_grid_max * step));
  if (int prc = rbt_pack_step(h, h->d_step_pack.get(), stream)) return prc;
  const int rc = allgather(h->d_step_pack.get(), all_dev, size_t(n_rec) * step, /*ncclFloat64*/ 8, nccl_comm, st);
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
long long rbt_launch_count(rbt_handle* h) { return h ? h->launches : 0; }

// ---------------------------------------------------------------------------------------------------------------
// unconstrained path
// ---------------------------------------------------------------------------------------------------------------
int rbt_unconstr_create(int nv, int N, double dt, int batch, int device, rbt_uhandle** out) {
  if (!out || nv < 1 || N < 1 || batch < 1 || !(dt > 0)) return RBT_ERR_ARG;
  if (nv != UNV) return RBT_ERR_ARG;
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
  RBT_CUDA(h, h->d_kkt.ensure(per * h->L.k_stride));
  RBT_CUDA(h, zeroed(h->d_ric, per * h->L.r_stride));
  RBT_CUDA(h, zeroed(h->d_fact, per * h->L.f_stride));
  RBT_CUDA(h, zeroed(h->d_dir, per * h->L.d_stride));
  RBT_CUDA(h, h->d_dx0.ensure(size_t(batch) * h->L.nx));
  RBT_CUDA(h, zeroed(h->d_info, size_t(batch)));
  return RBT_OK;
}

int rbt_unconstr_destroy(rbt_uhandle* h) {
  if (!h) return RBT_ERR_ARG;
  cudaSetDevice(h->device);
  delete h;
  return RBT_OK;
}

static BufDesc ubuf(rbt_uhandle* h, int which) {
  const rbt_ulayout& L = h->L;
  const rbt_ustage_layout& S = h->S;
  const BufDesc t[] = {
      /* KKT   */ {h->d_kkt.get(), L.k_stride, SC_GRID, false, nullptr, IN_KKT},
      /* RIC   */ {h->d_ric.get(), L.r_stride, SC_GRID, false, nullptr, -1},
      /* FACT  */ {h->d_fact.get(), L.f_stride, SC_GRID, false, nullptr, -1},
      /* DIR   */ {h->d_dir.get(), L.d_stride, SC_GRID, false, nullptr, -1},
      /* DX0   */ {h->d_dx0.get(), L.nx, SC_OCP, false, nullptr, IN_DX0},
      /* INFO  */ {nullptr, 0, SC_NONE, false, nullptr, -1},
      /* LIN   */ {h->d_lin.get(), S.l_stride, SC_GRID, true, nullptr, IN_LIN},
      /* CON   */ {h->d_con.get(), S.c_stride, SC_GRID, true, nullptr, IN_CON},
      /* EXP   */ {h->d_ex.get(), S.e_stride, SC_GRID, true, nullptr, -1},
      /* SOL   */ {h->d_sol.get(), S.s_stride, SC_GRID, true, nullptr, IN_SOL},
      /* XDIR  */ {h->d_xd.get(), S.x_stride, SC_GRID, true, nullptr, -1},
      /* STEPS */ {h->d_steps.get(), 2, SC_OCP, true, nullptr, -1},
  };
  return which >= 0 && which < int(sizeof(t) / sizeof(t[0])) ? t[which] : BufDesc{nullptr, 0, SC_NONE, false, nullptr, -1};
}

long long rbt_unconstr_buf_doubles(rbt_uhandle* h, int which) {
  return h ? buf_doubles(ubuf(h, which), h->stage_ready, h->batch, h->N + 1) : -1;
}

double* rbt_unconstr_dev_ptr(rbt_uhandle* h, int which) { return h ? ubuf(h, which).ptr : nullptr; }

int rbt_unconstr_upload(rbt_uhandle* h, int which, const double* host, void* stream) {
  if (!h || !host) return RBT_ERR_ARG;
  const BufDesc d = ubuf(h, which);
  if (d.in < 0) return RBT_ERR_ARG;
  // a table with n_box = 0 has an empty PDIPM record: its buffer is a null allocation, and copying it is a no-op
  const long long n = buf_doubles(d, h->stage_ready, h->batch, h->N + 1);
  if (n < 0 || (n > 0 && !d.ptr)) {
    h->err = "rbt_unconstr_upload: stage layer not set up (rbt_unconstr_stage_setup)";
    return RBT_ERR_STATE;
  }
  if (n == 0) return RBT_OK;
  RBT_CUDA(h, cudaSetDevice(h->device));
  RBT_CUDA(h, cudaMemcpyAsync(d.ptr, host, size_t(n) * 8, cudaMemcpyHostToDevice, (cudaStream_t)stream));
  return RBT_OK;
}

int rbt_unconstr_download(rbt_uhandle* h, int which, double* host, void* stream) {
  if (!h || !host) return RBT_ERR_ARG;
  const BufDesc d = ubuf(h, which);
  const long long n = buf_doubles(d, h->stage_ready, h->batch, h->N + 1);
  if (n < 0 || (n > 0 && !d.ptr)) return RBT_ERR_ARG;
  if (n == 0) return RBT_OK;
  RBT_CUDA(h, cudaSetDevice(h->device));
  RBT_CUDA(h, cudaMemcpyAsync(host, d.ptr, size_t(n) * 8, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  return RBT_OK;
}

int rbt_unconstr_download_info(rbt_uhandle* h, int* host_flags, void* stream) {
  if (!h || !host_flags) return RBT_ERR_ARG;
  RBT_CUDA(h, cudaSetDevice(h->device));
  RBT_CUDA(h, cudaMemcpyAsync(host_flags, h->d_info.get(), size_t(h->batch) * sizeof(int), cudaMemcpyDeviceToHost,
                              (cudaStream_t)stream));
  return RBT_OK;
}

static rbt::UParams make_uparams(rbt_uhandle* h, int write_fact) {
  rbt::UParams p;
  p.L = h->L;
  p.N = h->N;
  p.batch = h->batch;
  p.dt = h->dt;
  p.kkt = h->d_kkt.get();
  p.ric = h->d_ric.get();
  p.fact = write_fact ? h->d_fact.get() : nullptr;
  p.dx0 = h->d_dx0.get();
  p.dir = h->d_dir.get();
  p.info = h->d_info.get();
  return p;
}

int rbt_unconstr_backward(rbt_uhandle* h, int write_fact, void* stream) {
  if (!h) return RBT_ERR_ARG;
  RBT_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t st = (cudaStream_t)stream;
  if (rbt::UCfg<UNV>::KSTRIDE != h->L.k_stride) return RBT_ERR_STATE;
  RBT_CUDA(h, cudaMemsetAsync(h->d_info.get(), 0, size_t(h->batch) * sizeof(int), st));
  rbt::unconstr_backward_kernel<UNV><<<h->batch, 32, 0, st>>>(make_uparams(h, write_fact));
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

int rbt_unconstr_forward(rbt_uhandle* h, void* stream) {
  if (!h) return RBT_ERR_ARG;
  RBT_CUDA(h, cudaSetDevice(h->device));
  rbt::unconstr_forward_kernel<UNV><<<h->batch, 32, 0, (cudaStream_t)stream>>>(make_uparams(h, 0));
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
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
  // everything is allocated before anything is committed: a failed setup leaves the handle as it was
  RBT_CUDA(h, cudaSetDevice(h->device));
  rbt_ustage_layout S;
  rbt_make_ustage_layout(h->nv, table->n_box, &S);
  const size_t per = size_t(h->batch) * (h->N + 1);
  DevBuf<double> lin, con, ex, sol, xd, steps, ones;
  RBT_CUDA(h, zeroed(lin, per * S.l_stride));
  RBT_CUDA(h, zeroed(con, per * S.c_stride));
  RBT_CUDA(h, zeroed(ex, per * S.e_stride));
  RBT_CUDA(h, zeroed(sol, per * S.s_stride));
  RBT_CUDA(h, zeroed(xd, per * S.x_stride));
  RBT_CUDA(h, steps.ensure(size_t(h->batch) * 2));
  RBT_CUDA(h, ones.ensure(size_t(h->batch) * 2));
  const std::vector<double> one(size_t(h->batch) * 2, 1.0);
  RBT_CUDA(h, cudaMemcpy(ones.get(), one.data(), one.size() * 8, cudaMemcpyHostToDevice));
  RBT_CUDA(h, cudaMemcpy(steps.get(), one.data(), one.size() * 8, cudaMemcpyHostToDevice));
  h->S = S;
  h->table = *table;
  h->d_lin = std::move(lin);
  h->d_con = std::move(con);
  h->d_ex = std::move(ex);
  h->d_sol = std::move(sol);
  h->d_xd = std::move(xd);
  h->d_steps = std::move(steps);
  h->d_ones = std::move(ones);
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
  p.lin = h->d_lin.get();
  p.con = h->d_con.get();
  p.kkt = h->d_kkt.get();
  p.ex = h->d_ex.get();
  p.dir = h->d_dir.get();
  p.xd = h->d_xd.get();
  p.sol = h->d_sol.get();
  p.steps = h->d_steps.get();
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
  if (rbt::UStageCfg<UNV>::LSTRIDE != h->S.l_stride) return RBT_ERR_STATE;
  constexpr int W = rbt::UStageCfg<UNV>::WARPS;
  const size_t total = size_t(h->batch) * (h->N + 1);
  rbt::ucondense_kernel<UNV><<<unsigned((total + W - 1) / W), 32 * W, 0, st>>>(make_ustage_params(h));
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

int rbt_unconstr_expand_and_step_sizes(rbt_uhandle* h, void* stream) {
  RBT_USTAGE_GUARD(h)
  const size_t total = size_t(h->batch) * h->N;
  RBT_CUDA(h, cudaMemcpyAsync(h->d_steps.get(), h->d_ones.get(), size_t(h->batch) * 2 * 8, cudaMemcpyDeviceToDevice, st));
  rbt::uexpand_kernel<UNV><<<unsigned((total + 3) / 4), 128, 0, st>>>(make_ustage_params(h));
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
}

int rbt_unconstr_update(rbt_uhandle* h, void* stream) {
  RBT_USTAGE_GUARD(h)
  const size_t total = size_t(h->batch) * (h->N + 1);
  rbt::uupdate_kernel<UNV><<<unsigned((total + 3) / 4), 128, 0, st>>>(make_ustage_params(h));
  RBT_CUDA(h, cudaGetLastError());
  h->launches += 1;
  return RBT_OK;
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

// cs_b200.cu -- host side of libcsb200.so (C ABI in include/cs_b200.h).
// Plain CUDA runtime, no torch.  One handle = one connected component's operator
// resident on one GPU + a panel workspace for the batched PCG.
#include "../../include/cs_b200.h"

#include <cuda_runtime.h>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <string>
#include <type_traits>
#include <vector>

#include "amg_host.hpp"
#include "win_host.hpp"
#include "kernels.cuh"
#include "raster_assembly.cuh"
#include "setup_device.hpp"

using namespace csb;

namespace {

thread_local std::string g_create_error;

// profile kernel classes: 0 ... 6 the SpMM epilogue MODE (kernels.cuh SP_PLAIN ... SP_ADD), then these
constexpr int PROF_CLASSES = 20;   // cs_b200_profile_classes_n: 10 kernel classes x (fp64, fp32)
constexpr int PROF_PJ = 7;         // class of the fused prolongation + post-smoothing sweep
constexpr int PROF_CGF = 8;        // class of the fused CG step
constexpr int PROF_RSW = 9;        // class of the fused residual update + level-0 residual sweep

struct GraphSlot {
  cudaGraphExec_t exec = nullptr;
  int chunk = 0;
  int64_t kernels = 0, spmms = 0;   // launches inside one graph replay
  cudaGraphExec_t loop_exec = nullptr;        // whole PCG loop as a device-side WHILE graph
  int64_t loop_kernels = 0, loop_spmms = 0;   // launches per loop iteration
};

}  // namespace

// one CSR resident on the device, with its row-block partition (type-erased values)
struct DevCsr {
  int* rowptr = nullptr;
  int* colidx = nullptr;
  void* vals = nullptr;
  int* bstart = nullptr;
  int nblocks = 0;
  int nrows = 0;
  int64_t nnz = 0;
  int lpr = 1;  // lanes per row used by k_spmm for this matrix
  // windowed row-block form for the TMA-staged kernel (win_host.hpp); null => plain kernel
  WinMeta* win_meta = nullptr;
  unsigned char* blob = nullptr;   // per-block records [values | 1/diag | local columns | row offsets]
  int has_dinv = 0;
  int64_t win_blocks = 0;
  int win_nblocks = 0;
  // stencil (DIA) form (kernels.cuh k_stencil): 9 diagonals, ld apart, or with dia_half the 5 upper ones
  // (slots 4 ... 8) of a bitwise symmetric operator; null => CSR kernels
  void* dia = nullptr;
  size_t dia_ld = 0;
  int dia_nr = 0;
  int dia_half = 0;
  // ELL-4 copy of a prolongator with <= 4 entries per row (k_stencil_prolong_jacobi); null otherwise
  int* ell_col = nullptr;
  void* ell_val = nullptr;
  size_t ell_ld = 0;
};

// one multigrid level below the finest (the finest level aliases the handle's own CSR)
struct DevLevel {
  int64_t n = 0, n_pad = 0;
  DevCsr A, P, R;          // P: this level <- next coarser ; R = P^T
  void* dinv = nullptr;
  double omega = 2.0 / 3.0;
  void *x = nullptr, *b = nullptr, *t = nullptr, *y = nullptr;   // panels n_pad x ktmax
};

struct cs_b200_handle {
  int device = 0;
  int dtype = CS_B200_F64;
  int64_t n = 0, n_pad = 0, nnz = 0;
  int* d_rowptr = nullptr;
  int* d_colidx = nullptr;
  void* d_vals = nullptr;
  bool owns_matrix = true;
  void* d_vals0 = nullptr;           // pristine values while grounds are applied (cs_b200_set_grounds)
  void* d_fg = nullptr;              // the finite grounds of the last cs_b200_set_grounds, or null
  // cs_b200_plan_advanced's plan until cs_b200_read_advanced_plan: col_comp, set_ptr, set_rows, src_ptr,
  // src_rows (int64), src_vals (fp64), col_of_row (n int32), back to back in one allocation
  void* d_plan = nullptr;
  int64_t plan_ncol = 0, plan_nset = 0, plan_nsrc = 0;
  void* d_dinv = nullptr;
  int* d_bstart = nullptr;
  int nblocks = 0;
  int ktmax = 8;
  void *X = nullptr, *R = nullptr, *P = nullptr, *AP = nullptr, *B = nullptr, *stage = nullptr;
  void* Z = nullptr;                 // AMG: z = M^-1 r
  void* P2 = nullptr;                // fused CG step (k_stencil_cg): p of even iterations; P holds the odd ones
  void* R2 = nullptr;                // fused residual sweep (k_stencil_res_update): r of odd iterations; R the even ones
  DevCsr A0;                         // view of the finest operator (aliases d_rowptr/...)
  std::vector<DevLevel> lv;          // lv[0] = finest (A aliases A0), lv.back() = coarsest
  double* d_pinv = nullptr;          // dense pseudo-inverse of the coarsest operator
  double amg_opc = 0.0;              // operator complexity
  bool amg = false;
  // mixed precision: fp64 CG around an fp32 V-cycle.  lv32 = float copies of every level's
  // operators and panels (the finest included); R32/X32/T32/Z32 = finest-level float panels.
  bool mixed = false;
  std::vector<DevLevel> lv32;
  void *R32 = nullptr, *X32 = nullptr, *T32 = nullptr, *Z32 = nullptr;
  void *d_cum = nullptr, *d_max = nullptr;
  // branch currents (kernels.cuh k_branch_cur), all built on first use: d_bptr[n+1] the exclusive scan of the
  // strictly-lower entry count per row (nb = d_bptr[n] branches), d_cum_branch the cumulative branch vector
  // (nb), d_branch_stage the nb x ktmax download panel
  int* d_bptr = nullptr;
  int64_t nb = 0;
  void* d_cum_branch = nullptr;
  void* d_branch_stage = nullptr;
  PanelCtl* d_ctl = nullptr;
  PanelCtl* h_ctl = nullptr;  // pinned
  double* d_partials = nullptr;
  float* d_flush = nullptr;
  size_t flush_elems = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev2 = nullptr, ev3 = nullptr;
  // solve_rhs host<->device pipeline: panel i+1 uploads and panel i-1 downloads on two copy
  // streams while panel i solves (column-major staging buffers, double-buffered; lazy)
  // cs_b200_solve_sources scratch (grown on demand)
  long long* d_sp_rows = nullptr;
  double* d_sp_vals = nullptr;
  int* d_sp_ptr = nullptr;
  size_t sp_cap = 0;
  long long* d_probe = nullptr;
  void* d_probe_out = nullptr;
  size_t probe_cap = 0;
  cudaStream_t s_in = nullptr, s_out = nullptr;
  void* io_in[2] = {nullptr, nullptr};
  void* io_out[2] = {nullptr, nullptr};
  cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_used[2] = {nullptr, nullptr};
  cudaEvent_t ev_ready[2] = {nullptr, nullptr}, ev_out[2] = {nullptr, nullptr};
  int num_sms = 132;                 // set from the device in common_create
  int grid_spmm = 132, grid_ew = 132;
  cs_b200_opts opts{};
  cs_b200_stats stats{};
  GraphSlot graphs[4];  // KT = 1,2,4,8
  // cs_b200_solve_region_pairs: the panel's Dirichlet sets as 2*KT row segments (kernels.cuh k_seg_set).
  // Region panels mask AP and Z inside the PCG loop, so they get graph slots of their own; those graphs
  // capture d_rg_seg / d_rg_rows and are dropped whenever the buffers are reallocated.
  bool rg_on = false;                // the panel being solved is a region panel
  bool pair_b = false;               // its right-hand side is ctl's pairs rule, B not written (stage_pair_rhs)
  int* d_rg_seg = nullptr;
  int* d_rg_rows = nullptr;
  size_t rg_cap = 0;
  GraphSlot rgraphs[4];
  // optional per-launch SpMM timing (cs_b200_profile_spmm): event pairs harvested at
  // every host poll, so the pool only has to cover one chunk of iterations.
  int profile = 0;
  std::vector<cudaEvent_t> prof_ev;
  size_t prof_used = 0;
  double prof_ms = 0.0;
  double prof_bytes = 0.0;   // algorithmic bytes of the timed launches (DESIGN.md §4 formula)
  int64_t prof_launches = 0;
  // the same per kernel class (PROF_CLASSES): slot = 2 * class + (fp32 ? 1 : 0)
  std::vector<int> prof_slot;           // one entry per event pair in flight
  std::vector<double> prof_pair_bytes;
  double prof_slot_ms[PROF_CLASSES] = {}, prof_slot_bytes[PROF_CLASSES] = {};
  int64_t prof_slot_launches[PROF_CLASSES] = {};
  std::string err;
  size_t esize() const { return dtype == CS_B200_F64 ? 8 : 4; }
};

namespace {

// CS_B200_VERBOSE=1: one stderr line per setup phase (host hierarchy, windows, uploads)
struct Tick {
  bool on = std::getenv("CS_B200_VERBOSE") != nullptr;
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
  void operator()(const char* what) {
    if (!on) return;
    const auto t1 = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[cs_b200 setup] %-28s %8.1f ms\n", what,
                 std::chrono::duration<double, std::milli>(t1 - t0).count());
    t0 = t1;
  }
};

int set_err(cs_b200_handle* h, int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (h) h->err = buf; else g_create_error = buf;
  return code;
}

#define CK(h, call)                                                                      \
  do {                                                                                   \
    cudaError_t _e = (call);                                                             \
    if (_e != cudaSuccess)                                                               \
      return set_err(h, CS_B200_ERR_CUDA, "CUDA error %s at %s:%d (%s)",                 \
                     cudaGetErrorString(_e), __FILE__, __LINE__, #call);                 \
  } while (0)

// Host->device upload ordered on the handle's (non-blocking) stream.  NOT cudaMemcpy:
// for pageable sources that call may return before the DMA of the last staged chunk has
// landed and is only ordered against the legacy default stream -- a kernel on h->stream
// launched right after could read a stale tail.
cudaError_t h2d(cs_b200_handle* h, void* dst, const void* src, size_t bytes) {
  if (bytes == 0) return cudaSuccess;
  cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, h->stream);
  if (e != cudaSuccess) return e;
  return cudaStreamSynchronize(h->stream);   // the source buffers are short-lived host vectors
}

int kt_index(int kt) { return kt == 1 ? 0 : kt == 2 ? 1 : kt == 4 ? 2 : 3; }

// greedy row blocks: <= NNZ_CAP nnz and <= NT rows; an over-long row stands alone.
void build_row_blocks(const std::vector<int>& rowptr, int64_t n, std::vector<int>& bstart,
                      int max_rows = NT) {
  bstart.clear();
  bstart.push_back(0);
  int64_t r = 0;
  while (r < n) {
    int64_t r1 = r + 1;
    const int64_t base = rowptr[r];
    while (r1 < n && (r1 - r) < max_rows && (int64_t)rowptr[r1 + 1] - base <= NNZ_CAP) ++r1;
    bstart.push_back((int)r1);
    r = r1;
  }
}

template <typename T>
int build_windowed(cs_b200_handle* h, DevCsr& d, const int* rowptr, const int* colidx, int64_t ncols_pad,
                   const T* d_dinv = nullptr);

// upload one host CSR (double values) as a device CSR of T with its row blocks
// debugging aid: CS_B200_WIN_MASK bit 0 = finest A, 1 = coarse A, 2 = P, 3 = R (default all)
int win_mask() {
  const char* e = getenv("CS_B200_WIN_MASK");
  return e ? atoi(e) : 15;
}

// sizes, lanes per row of k_spmm and the row-block height of an operator with `nrows` rows: small operators
// (coarse levels) get shorter blocks so that >= 4 CTAs per SM exist -- their kernels are latency-bound chains
// of dependent gathers, not bandwidth-bound
int size_csr(const cs_b200_handle* h, DevCsr& d, int64_t nrows, int64_t nnz) {
  d.nrows = (int)nrows;
  d.nnz = nnz;
  d.lpr = (nrows > 0 && (double)nnz / (double)nrows >= 20.0) ? 4 : 1;
  const int unit = d.lpr == 4 ? 8 : 32;          // rows per pass of k_spmm at KT = 8
  const int max_rows = (int)((nrows + 4 * h->num_sms - 1) / (4 * h->num_sms));
  return std::min(NT, std::max(unit, (max_rows + unit - 1) / unit * unit));
}

template <typename T>
int upload_csr(cs_b200_handle* h, const csb_amg::Csr& m, DevCsr& d, bool windowed, const T* d_dinv = nullptr) {
  const int max_rows = size_csr(h, d, m.nrows, m.nnz());
  std::vector<int> bstart;
  build_row_blocks(m.ptr, m.nrows, bstart, max_rows);
  d.nblocks = (int)bstart.size() - 1;
  std::vector<T> v(m.val.begin(), m.val.end());
  CK(h, cudaMalloc(&d.rowptr, (size_t)(m.nrows + 1) * sizeof(int)));
  CK(h, cudaMalloc(&d.colidx, std::max<size_t>(1, (size_t)d.nnz) * sizeof(int)));
  CK(h, cudaMalloc(&d.vals, std::max<size_t>(1, (size_t)d.nnz) * sizeof(T)));
  CK(h, cudaMalloc(&d.bstart, bstart.size() * sizeof(int)));
  CK(h, h2d(h, d.rowptr, m.ptr.data(), (size_t)(m.nrows + 1) * sizeof(int)));
  CK(h, h2d(h, d.colidx, m.idx.data(), (size_t)d.nnz * sizeof(int)));
  CK(h, h2d(h, d.vals, v.data(), (size_t)d.nnz * sizeof(T)));
  CK(h, h2d(h, d.bstart, bstart.data(), bstart.size() * sizeof(int)));
  if (h->opts.window >= 0 && windowed) {
    const int64_t ncols_pad = (m.ncols + 3) / 4 * 4;
    return build_windowed<T>(h, d, m.ptr.data(), m.idx.data(), ncols_pad, d_dinv);
  }
  return CS_B200_OK;
}

void free_win(DevCsr& d) {
  cudaFree(d.win_meta); cudaFree(d.blob); cudaFree(d.dia); cudaFree(d.ell_col); cudaFree(d.ell_val);
  d.win_meta = nullptr; d.blob = nullptr; d.dia = nullptr; d.ell_col = nullptr; d.ell_val = nullptr;
  d.dia_half = 0;
}

void free_csr(DevCsr& d) {
  cudaFree(d.rowptr); cudaFree(d.colidx); cudaFree(d.vals); cudaFree(d.bstart);
  free_win(d);
  d = DevCsr{};
}

// Build + upload the windowed row-block form of a CSR already resident in `d`.
// rowptr/colidx: host copies; ncols_pad: rows of the input panel (n_pad of the column space).
template <typename T>
int build_windowed(cs_b200_handle* h, DevCsr& d, const int* rowptr, const int* colidx, int64_t ncols_pad,
                   const T* d_dinv) {
  static_assert(sizeof(WinMeta) == sizeof(csb_win::BlockMeta), "meta layout");
  static_assert(W_RB == csb_win::RB && W_WCAP == csb_win::WCAP && W_WCAP_WIDE == csb_win::WCAP_WIDE && W_NNZ == csb_win::NNZ_CAP &&
                W_MAXSEG == csb_win::MAXSEG, "window geometry");
  csb_win::Windowed w = csb_win::build(rowptr, colidx, d.nrows, ncols_pad, (int)sizeof(T),
                                       d.lpr == 4 ? csb_win::WCAP_WIDE : csb_win::WCAP, d_dinv != nullptr);
  d.has_dinv = d_dinv != nullptr ? 1 : 0;
  d.win_blocks = w.windowed_blocks;
  d.win_nblocks = (int)w.meta.size();
  if (w.windowed_blocks * 2 < (int64_t)w.meta.size()) return CS_B200_OK;   // mostly scattered: keep the plain kernel
  const size_t ne = w.lcol.size();
  int* d_perm = nullptr;
  int* d_roff_off = nullptr;
  unsigned short *d_lcol = nullptr, *d_roff = nullptr;
  CK(h, cudaMalloc(&d.win_meta, w.meta.size() * sizeof(WinMeta)));
  CK(h, cudaMalloc(&d.blob, (size_t)w.blob_bytes));
  CK(h, cudaMalloc(&d_lcol, ne * sizeof(unsigned short)));
  CK(h, cudaMalloc(&d_roff, w.roff.size() * sizeof(unsigned short)));
  CK(h, cudaMalloc(&d_roff_off, w.roff_off.size() * sizeof(int)));
  CK(h, cudaMalloc(&d_perm, ne * sizeof(int)));
  CK(h, h2d(h, d.win_meta, w.meta.data(), w.meta.size() * sizeof(WinMeta)));
  CK(h, h2d(h, d_lcol, w.lcol.data(), ne * sizeof(unsigned short)));
  CK(h, h2d(h, d_roff, w.roff.data(), w.roff.size() * sizeof(unsigned short)));
  CK(h, h2d(h, d_roff_off, w.roff_off.data(), w.roff_off.size() * sizeof(int)));
  CK(h, h2d(h, d_perm, w.perm_off.data(), ne * sizeof(int)));
  CK(h, cudaMemsetAsync(d.blob, 0, (size_t)w.blob_bytes, h->stream));
  k_pack_blob<T><<<std::max(1, std::min(d.win_nblocks, h->num_sms * 16)), 128, 0, h->stream>>>(
      d.win_nblocks, d.win_meta, d_perm, d_lcol, d_roff, d_roff_off, (const T*)d.vals, d_dinv, d.blob);
  CK(h, cudaGetLastError());
  CK(h, cudaStreamSynchronize(h->stream));
  cudaFree(d_lcol);
  cudaFree(d_roff);
  cudaFree(d_roff_off);
  cudaFree(d_perm);
  return CS_B200_OK;
}

// cudaMalloc + zero fill on the handle's stream
int alloc_zeroed(cs_b200_handle* h, void** p, size_t bytes) {
  CK(h, cudaMalloc(p, bytes));
  CK(h, cudaMemsetAsync(*p, 0, bytes, h->stream));
  return CS_B200_OK;
}

// Level l of either builder's hierarchy: n rows, smoother weight omega.  Without `own0` level 0 aliases the
// handle's operator and 1/diag, and false is returned: the builder has no A or 1/diag of its own to make.
bool begin_level(cs_b200_handle* h, DevLevel& L, int l, bool own0, int64_t n, double omega) {
  L.n = n;
  L.n_pad = (n + 3) / 4 * 4;
  L.omega = omega;
  if (l > 0 || own0) return true;
  L.A = h->A0;  // alias, not owned
  L.dinv = h->d_dinv;
  return false;
}

// the x / b / t / y panels of a coarse level
template <typename TV>
int level_panels(cs_b200_handle* h, DevLevel& L) {
  const size_t pe = (size_t)L.n_pad * h->ktmax * sizeof(TV);
  void** bufs[] = {&L.x, &L.b, &L.t, &L.y};
  for (void** bp : bufs)
    if (int rc = alloc_zeroed(h, bp, pe)) return rc;
  return CS_B200_OK;
}

// windowed row-block forms are built for level l's operator (mask bit 0 finest, 1 coarse), P (bit 2), R (bit 3)
bool level_windowed(const cs_b200_handle* h, int l, int64_t n) {
  return h->opts.window > 0 || (n >= 20000 && (win_mask() & (l == 0 ? 1 : 2)));
}

// Upload a host hierarchy as device levels of type TV.  `own0`: the finest level gets its own
// device CSR (float copy for the mixed-precision cycle); otherwise it aliases the handle's.
template <typename TV>
int make_levels(cs_b200_handle* h, const csb_amg::Hierarchy& hier, std::vector<DevLevel>& lv, bool own0) {
  const int nl = (int)hier.levels.size();
  lv.resize(nl);
  for (int l = 0; l < nl; ++l) {
    const csb_amg::HostLevel& hl = hier.levels[l];
    DevLevel& L = lv[l];
    if (begin_level(h, L, l, own0, hl.A.nrows, hl.omega)) {
      std::vector<TV> dv(L.n_pad, TV(0));
      for (int64_t i = 0; i < L.n; ++i) dv[i] = (TV)hl.dinv[i];
      CK(h, cudaMalloc(&L.dinv, (size_t)L.n_pad * sizeof(TV)));
      CK(h, h2d(h, L.dinv, dv.data(), (size_t)L.n_pad * sizeof(TV)));
      int rc = upload_csr<TV>(h, hl.A, L.A, level_windowed(h, l, L.n), (const TV*)L.dinv);
      if (!rc && l > 0) rc = level_panels<TV>(h, L);
      if (rc) return rc;
    }
    if (l + 1 < nl) {
      int rc = upload_csr<TV>(h, hl.P, L.P, L.n >= 20000 && (win_mask() & 4));
      if (rc) return rc;
      rc = upload_csr<TV>(h, hl.R, L.R, L.n >= 20000 && (win_mask() & 8));
      if (rc) return rc;
    }
  }
  return CS_B200_OK;
}

template <typename TV>
int make_levels(cs_b200_handle* h, csb_dev::DHierarchy& hier, std::vector<DevLevel>& lv, bool own0);

void wait_pinv(csb_amg::Hierarchy&) {}
void wait_pinv(csb_dev::DHierarchy& hier) { csb_dev::coarse_pinv_wait(hier); }

// What either builder's hierarchy leaves on the handle: its levels resident (make_levels), the fp32 or Z panels,
// the coarse pseudo-inverse.  fp64 handles run the V-cycle in fp32 (opts.mixed: 0 auto = on, -1 off): the
// preconditioner only has to be a good approximate inverse, CG's own vectors stay fp64.
template <typename T, class Hier>
int adopt_hierarchy(cs_b200_handle* h, Hier& hier) {
  const int nl = (int)hier.levels.size();
  h->mixed = nl > 1 && sizeof(T) == 8 && h->opts.mixed >= 0;
  Tick tick;
  if (h->mixed) {
    int rc = make_levels<float>(h, hier, h->lv32, true);
    if (rc) return rc;
    // the fp64 side only needs level 0's omega / dinv (already on the handle)
    h->lv.resize(nl);
    for (int l = 0; l < nl; ++l) { h->lv[l].n = hier.levels[l].A.nrows; h->lv[l].omega = hier.levels[l].omega; }
    h->lv[0].A = h->A0;
    h->lv[0].dinv = h->d_dinv;
    const size_t pe = (size_t)h->n_pad * h->ktmax * sizeof(float);
    void** bufs[] = {&h->R32, &h->X32, &h->T32, &h->Z32};
    for (void** bp : bufs)
      if ((rc = alloc_zeroed(h, bp, pe))) return rc;
  } else {
    int rc = make_levels<T>(h, hier, h->lv, false);
    if (!rc) rc = alloc_zeroed(h, &h->Z, (size_t)h->n_pad * h->ktmax * sizeof(T));
    if (rc) return rc;
  }
  tick("levels");
  wait_pinv(hier);
  tick("coarse pseudo-inverse (wait)");
  const size_t nc = (size_t)hier.levels.back().A.nrows;
  if (hier.coarse_pinv.size() == nc * nc && nc > 0) {
    CK(h, cudaMalloc(&h->d_pinv, nc * nc * sizeof(double)));
    CK(h, h2d(h, h->d_pinv, hier.coarse_pinv.data(), nc * nc * sizeof(double)));
  }
  CK(h, cudaStreamSynchronize(h->stream));
  h->amg = nl > 1;
  return CS_B200_OK;
}

// Smoothed-aggregation hierarchy: built on the host (amg_host.hpp), resident on the device.
template <typename T>
int setup_amg(cs_b200_handle* h, const std::vector<int>& rp, const std::vector<int>& ci, const T* vals_host) {
  csb_amg::Csr a0;
  a0.nrows = a0.ncols = h->n;
  a0.ptr = rp;
  a0.idx = ci;
  a0.val.assign(vals_host, vals_host + h->nnz);
  Tick tick;
  csb_amg::Hierarchy hier = csb_amg::build_hierarchy(std::move(a0));
  tick("host hierarchy");
  h->amg_opc = hier.operator_complexity();
  return adopt_hierarchy<T>(h, hier);
}

// panels, 1/diag, current vectors, control block: what every handle needs whatever built its operators
template <typename T>
int alloc_common(cs_b200_handle* h) {
  const size_t pe = (size_t)h->n_pad * h->ktmax;
  void** bufs[] = {&h->X, &h->R, &h->P, &h->AP, &h->B, &h->stage};
  const char* ve = std::getenv("CS_B200_VERBOSE");
  const bool v2 = ve && std::atoi(ve) >= 2;
  auto t0 = std::chrono::steady_clock::now();
  auto stamp = [&](const char* what) {
    if (!v2) return;
    cudaStreamSynchronize(h->stream);
    const auto t1 = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[cs_b200 setup/stamp]        %-34s %8.2f ms\n", what,
                 std::chrono::duration<double, std::milli>(t1 - t0).count());
    t0 = t1;
  };
  stamp("alloc_common: entry (pending work)");
  for (void** b : bufs) {
    CK(h, cudaMalloc(b, pe * sizeof(T)));
    CK(h, cudaMemsetAsync(*b, 0, pe * sizeof(T), h->stream));
  }
  stamp("alloc_common: 6 panels");
  CK(h, cudaMalloc(&h->d_dinv, (size_t)h->n_pad * sizeof(T)));
  CK(h, cudaMalloc(&h->d_cum, (size_t)h->n_pad * sizeof(T)));
  CK(h, cudaMalloc(&h->d_max, (size_t)h->n_pad * sizeof(T)));
  CK(h, cudaMalloc(&h->d_ctl, sizeof(PanelCtl)));
  CK(h, cudaMemsetAsync(h->d_ctl, 0, sizeof(PanelCtl), h->stream));
  stamp("alloc_common: dinv/cum/max/ctl");
  CK(h, cudaMallocHost(&h->h_ctl, sizeof(PanelCtl)));
  stamp("alloc_common: cudaMallocHost");
  const int maxgrid = h->num_sms * 8;
  CK(h, cudaMalloc(&h->d_partials, (size_t)maxgrid * 2 * MAXKT * sizeof(double)));
  k_dinv<T><<<std::min<int64_t>((h->n_pad + 255) / 256, 4096), 256, 0, h->stream>>>(
      (int)h->n, (int)h->n_pad, h->d_rowptr, h->d_colidx, (const T*)h->d_vals, (T*)h->d_dinv);
  CK(h, cudaGetLastError());
  stamp("alloc_common: k_dinv");
  return CS_B200_OK;
}

// host-side setup of a handle whose CSR is resident: row blocks and windows built from host copies of the
// pattern, the hierarchy by amg_host.hpp
template <typename T>
int finish_setup(cs_b200_handle* h, const std::vector<int>& h_rowptr) {
  std::vector<int> bstart;
  build_row_blocks(h_rowptr, h->n, bstart);
  h->nblocks = (int)bstart.size() - 1;
  CK(h, cudaMalloc(&h->d_bstart, bstart.size() * sizeof(int)));
  CK(h, cudaMemcpyAsync(h->d_bstart, bstart.data(), bstart.size() * sizeof(int),
                        cudaMemcpyHostToDevice, h->stream));
  h->A0 = DevCsr{h->d_rowptr, h->d_colidx, h->d_vals, h->d_bstart, h->nblocks, (int)h->n, h->nnz, 1};
  int rc0 = alloc_common<T>(h);
  if (rc0) return rc0;
  CK(h, cudaStreamSynchronize(h->stream));
  std::vector<int> h_colidx;
  std::vector<T> h_vals;
  const bool want_win = h->opts.window >= 0 && (h->opts.window > 0 || h->n >= 20000) && (win_mask() & 1);
  const bool want_amg = h->opts.precond == CS_B200_PRECOND_AMG;
  if (want_win || want_amg) {
    h_colidx.resize(h->nnz);
    CK(h, cudaMemcpy(h_colidx.data(), h->d_colidx, (size_t)h->nnz * sizeof(int), cudaMemcpyDeviceToHost));
  }
  if (want_amg) {
    h_vals.resize(h->nnz);
    CK(h, cudaMemcpy(h_vals.data(), h->d_vals, (size_t)h->nnz * sizeof(T), cudaMemcpyDeviceToHost));
  }
  Tick tick;
  if (want_win) {
    int rc = build_windowed<T>(h, h->A0, h_rowptr.data(), h_colidx.data(), h->n_pad, (const T*)h->d_dinv);
    if (rc) return rc;
    tick("finest operator: windows");
  }
  if (want_amg) {
    int rc = setup_amg<T>(h, h_rowptr, h_colidx, h_vals.data());
    if (rc) return rc;
  }
  return cs_b200_reset_currents(h);
}

// ---------------------------------------------------------------------------------------------
// device-side setup (setup_device.cu): row blocks, windowed records and the multigrid hierarchy are
// built on the GPU from the resident CSR; only the ordered aggregation seed pass runs on the host
// ---------------------------------------------------------------------------------------------
int rc_dev(cs_b200_handle* h, int rc) {   // csb_dev codes -> cs_b200 status (h->err already set)
  (void)h;
  if (rc == 0) return CS_B200_OK;
  return rc == -5 ? CS_B200_ERR_UNSUPPORTED : CS_B200_ERR_CUDA;
}

// plain-kernel row blocks of a device CSR (the partition build_row_blocks computes on the host)
int device_row_blocks(cs_b200_handle* h, DevCsr& d, int max_rows) {
  int* bs = nullptr;
  int nb = 0;
  int rc = csb_dev::row_blocks(h->stream, d.rowptr, d.nrows, max_rows, NNZ_CAP, &bs, &nb, h->err);
  if (rc) return rc_dev(h, rc);
  d.bstart = bs;
  d.nblocks = nb;
  return CS_B200_OK;
}

template <typename T>
int device_windows(cs_b200_handle* h, DevCsr& d, int64_t ncols_pad, const T* d_dinv) {
  csb_dev::DWin w;
  int rc = csb_dev::build_windowed<T>(h->stream, d.rowptr, d.colidx, (const T*)d.vals, d.nrows, ncols_pad,
                                      d.lpr == 4 ? W_WCAP_WIDE : W_WCAP, d_dinv, w, h->err);
  if (rc) return rc_dev(h, rc);
  d.has_dinv = d_dinv != nullptr ? 1 : 0;
  d.win_blocks = w.windowed_blocks;
  d.win_nblocks = w.nblocks;
  d.win_meta = reinterpret_cast<WinMeta*>(w.meta);
  d.blob = w.blob;
  return CS_B200_OK;
}

// the stencil kernels stage their operands through the shared-memory pipeline (kernels.cuh k_stencil_pipe,
// k_stencil_cg_pipe); CS_B200_NO_STENCIL_PIPE keeps the register-gather kernels for A/B runs
inline bool stencil_pipe() {
  static const bool off = std::getenv("CS_B200_NO_STENCIL_PIPE") != nullptr;
  return !off;
}

// a bitwise symmetric stencil is stored as its 5 upper diagonals (setup_device.hpp halve_dia);
// CS_B200_FULL_STENCIL keeps all 9 for A/B runs, and so does the register-gather path, which reads 9
inline bool full_stencil() {
  static const bool on = std::getenv("CS_B200_FULL_STENCIL") != nullptr;
  return on || !stencil_pipe();
}

// stencil-form levels keep the zero-guess Jacobi sweep implicit: x0 = omega D^-1 b is formed on the fly
// by the residual kernel (SP_RES0) and by the fused upward kernel, never stored (CS_B200_NO_IMPLICIT_X0
// switches back to the stored form for A/B runs)
inline bool implicit_x0(const DevLevel& L) {
  static const bool off = std::getenv("CS_B200_NO_IMPLICIT_X0") != nullptr || std::getenv("CS_B200_NO_FUSED_PROLONG") != nullptr;
  return L.A.dia != nullptr && !off;
}

// The fused residual sweep (kernels.cuh k_stencil_res_update) forms r -= alpha A p, r32 and the level-0 residual
// of the fp32 V-cycle in one pass, in place of k_cg_update_r0 and the level-0 SP_RES0 sweep.  It is written for
// what the bench workload runs: an fp32 cycle (mixed) on a half-form stencil finest level, pipelined kernels,
// implicit x0 (and, checked when R2 is allocated, fp32 level-0 diagonals that are the fp64 ones rounded).
// CS_B200_NO_FUSED_RES keeps the two kernels for A/B runs.
inline bool fused_res_form(const cs_b200_handle* h) {
  static const bool off = std::getenv("CS_B200_NO_FUSED_RES") != nullptr;
  return !off && h->mixed && stencil_pipe() && h->A0.dia && h->A0.dia_half && !h->lv32.empty() &&
         h->lv32[0].A.dia_half && implicit_x0(h->lv32[0]);
}

// the kernels' view of a stencil-form operator
template <typename T>
DiaDev<T> dia_view(const DevCsr& m) {
  return DiaDev<T>{(const T*)m.dia, m.dia_ld, m.nrows, m.dia_nr, m.dia_half};
}

// The register-gather kernels (k_stencil, k_stencil_cg) read all 9 slots.  full_stencil() keeps every
// operator at 9 slots on that path, so a half-form operator reaching them is a broken invariant, and a
// launch would read past the 5 stored runs: stop instead.
[[noreturn]] inline void refuse_half(const char* kernel) {
  std::fprintf(stderr, "cs_b200: %s was handed a half-form (5-slot) stencil; it reads 9 slots\n", kernel);
  std::abort();
}

// stencil (DIA) form of a square operator, if its pattern allows it (opts.stencil: 0 auto, 1, -1 never)
template <typename T>
int device_stencil(cs_b200_handle* h, DevCsr& d) {
  static const bool env_off = std::getenv("CS_B200_NO_STENCIL") != nullptr;
  if (h->opts.stencil < 0 || env_off) return CS_B200_OK;
  if (h->opts.stencil == 0 && d.nrows < 20000) return CS_B200_OK;
  T* dia = nullptr;
  int nr = 0;
  size_t ld = 0;
  int rc = csb_dev::build_dia<T>(h->stream, d.rowptr, d.colidx, (const T*)d.vals, d.nrows, &dia, &nr, &ld, h->err);
  if (rc) return rc_dev(h, rc);
  if (dia && !full_stencil()) {
    rc = csb_dev::halve_dia<T>(h->stream, &dia, d.nrows, nr, ld, &d.dia_half, h->err);
    if (rc) { cudaFree(dia); return rc_dev(h, rc); }
  }
  d.dia = dia;
  d.dia_nr = nr;
  d.dia_ld = ld;
  return CS_B200_OK;
}

// take over a hierarchy operator as a device CSR of TV: the index arrays move (or are duplicated when
// the source is the handle's own matrix), the fp64 values move or are converted
template <typename TV>
int adopt_csr(cs_b200_handle* h, csb_dev::DCsr& src, bool duplicate, DevCsr& d, bool windowed, const TV* d_dinv) {
  const int max_rows = size_csr(h, d, src.nrows, src.nnz);
  const size_t np = (size_t)src.nrows + 1, ne = std::max<size_t>(1, (size_t)src.nnz);
  if (duplicate) {
    CK(h, cudaMalloc(&d.rowptr, np * sizeof(int)));
    CK(h, cudaMalloc(&d.colidx, ne * sizeof(int)));
    CK(h, cudaMemcpyAsync(d.rowptr, src.ptr, np * sizeof(int), cudaMemcpyDeviceToDevice, h->stream));
    CK(h, cudaMemcpyAsync(d.colidx, src.idx, (size_t)src.nnz * sizeof(int), cudaMemcpyDeviceToDevice, h->stream));
  } else {
    d.rowptr = src.ptr; src.ptr = nullptr;
    d.colidx = src.idx; src.idx = nullptr;
  }
  if (sizeof(TV) == 8 && !duplicate) {
    d.vals = src.val; src.val = nullptr;
  } else {
    CK(h, cudaMalloc(&d.vals, ne * sizeof(TV)));
    if (sizeof(TV) == 8) {
      CK(h, cudaMemcpyAsync(d.vals, src.val, (size_t)src.nnz * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
    } else if (csb_dev::convert_values(h->stream, src.val, (float*)d.vals, src.nnz)) {
      return set_err(h, CS_B200_ERR_CUDA, "value conversion launch failed");
    }
    if (!duplicate) {
      CK(h, cudaStreamSynchronize(h->stream));
      cudaFree(src.val); src.val = nullptr;
    }
  }
  int rc = device_row_blocks(h, d, max_rows);
  if (rc) return rc;
  if (src.nrows == src.ncols && d_dinv != nullptr) {   // square level operator: stencil form if it has one
    rc = device_stencil<TV>(h, d);
    if (rc) return rc;
    if (d.dia) return CS_B200_OK;
  }
  if (h->opts.window >= 0 && windowed) {
    const int64_t ncols_pad = (src.ncols + 3) / 4 * 4;
    return device_windows<TV>(h, d, ncols_pad, d_dinv);
  }
  return CS_B200_OK;
}

template <typename TV>
int make_levels(cs_b200_handle* h, csb_dev::DHierarchy& hier, std::vector<DevLevel>& lv, bool own0) {
  const int nl = (int)hier.levels.size();
  lv.resize(nl);
  Tick lt;
  auto mark = [&](int l, const char* what) {
    if (!lt.on) return;
    cudaStreamSynchronize(h->stream);
    char buf[64];
    snprintf(buf, sizeof buf, "  L%d %s", l, what);
    lt(buf);
  };
  for (int l = 0; l < nl; ++l) {
    csb_dev::DLevel& hl = hier.levels[l];
    DevLevel& L = lv[l];
    if (begin_level(h, L, l, own0, hl.A.nrows, hl.omega)) {
      CK(h, cudaMalloc(&L.dinv, (size_t)L.n_pad * sizeof(TV)));
      CK(h, cudaMemsetAsync(L.dinv, 0, (size_t)L.n_pad * sizeof(TV), h->stream));
      if (sizeof(TV) == 8) {
        CK(h, cudaMemcpyAsync(L.dinv, hl.dinv, (size_t)L.n * sizeof(double), cudaMemcpyDeviceToDevice, h->stream));
      } else if (csb_dev::convert_values(h->stream, hl.dinv, (float*)L.dinv, L.n)) {
        return set_err(h, CS_B200_ERR_CUDA, "dinv conversion launch failed");
      }
      int rc = adopt_csr<TV>(h, hl.A, l == 0, L.A, level_windowed(h, l, L.n), (const TV*)L.dinv);
      if (rc) return rc;
      mark(l, "A: copy/convert, blocks, windows");
      if (l > 0 && (rc = level_panels<TV>(h, L))) return rc;
    }
    if (l + 1 < nl) {
      int rc = adopt_csr<TV>(h, hl.P, false, L.P, L.n >= 20000 && (win_mask() & 4), (const TV*)nullptr);
      if (rc) return rc;
      if (L.A.dia) {          // the fused prolongation kernel of this level reads P as ELL-4 when it can
        int* ec = nullptr;
        TV* ev = nullptr;
        size_t eld = 0;
        int rce = csb_dev::build_ell4<TV>(h->stream, L.P.rowptr, L.P.colidx, (const TV*)L.P.vals, L.P.nrows, &ec, &ev, &eld, h->err);
        if (rce) return rc_dev(h, rce);
        L.P.ell_col = ec; L.P.ell_val = ev; L.P.ell_ld = eld;
      }
      mark(l, "P");
      rc = adopt_csr<TV>(h, hl.R, false, L.R, L.n >= 20000 && (win_mask() & 8), (const TV*)nullptr);
      if (rc) return rc;
      mark(l, "R");
    }
  }
  return CS_B200_OK;
}

// Smoothed-aggregation hierarchy built on the device (setup_device.cu).  `job`, the create sequence's level-0
// seed pass, is handed to build_hierarchy, which consumes it.
template <typename T>
int setup_amg_device(cs_b200_handle* h, const csb_dev::HostPattern& hp, csb_dev::SeedJob*& job,
                     const csb_dev::DeviceSeed* dseed) {
  const bool verbose = std::getenv("CS_B200_VERBOSE") != nullptr;
  csb_dev::DCsr a0;
  a0.nrows = a0.ncols = h->n;
  a0.nnz = h->nnz;
  a0.ptr = h->d_rowptr;
  a0.idx = h->d_colidx;
  double* tmp64 = nullptr;
  if (sizeof(T) == 8) {
    a0.val = (double*)h->d_vals;
  } else {   // the hierarchy is built in fp64 whatever the handle computes in
    cudaError_t e = cudaMalloc(&tmp64, std::max<size_t>(1, (size_t)h->nnz) * sizeof(double));
    if (e != cudaSuccess)
      return set_err(h, CS_B200_ERR_CUDA, "CUDA error %s (fp64 copy of the matrix)", cudaGetErrorString(e));
    csb_dev::convert_values(h->stream, (const float*)h->d_vals, tmp64, h->nnz);
    a0.val = tmp64;
  }
  Tick tick;
  csb_dev::DHierarchy hier;
  csb_dev::SeedJob* pre = job;
  job = nullptr;
  int rc = rc_dev(h, csb_dev::build_hierarchy(h->stream, a0, hp, pre, dseed, 12, 200, hier, h->err, verbose));
  if (!rc) {
    tick("device hierarchy");
    h->amg_opc = hier.operator_complexity;
    rc = adopt_hierarchy<T>(h, hier);
  }
  cudaStreamSynchronize(h->stream);
  csb_dev::free_hierarchy(hier);
  cudaFree(tmp64);
  return rc;
}

// 1/diag, the finest operator's stencil / window form, the multigrid hierarchy: everything that depends
// on the matrix VALUES (re-run by cs_b200_set_grounds after the values changed)
template <typename T>
int build_operators(cs_b200_handle* h, const csb_dev::HostPattern& hp, csb_dev::SeedJob*& job,
                    const csb_dev::DeviceSeed* dseed) {
  int rc = CS_B200_OK;
  k_dinv<T><<<std::min<int64_t>((h->n_pad + 255) / 256, 4096), 256, 0, h->stream>>>(
      (int)h->n, (int)h->n_pad, h->d_rowptr, h->d_colidx, (const T*)h->d_vals, (T*)h->d_dinv);
  const bool want_win = h->opts.window >= 0 && (h->opts.window > 0 || h->n >= 20000) && (win_mask() & 1);
  const bool want_amg = h->opts.precond == CS_B200_PRECOND_AMG;
  Tick tick;
  // stencil = 1 asks for the stencil form at any size, also where no windows are wanted
  if (want_win || h->opts.stencil > 0) {
    rc = device_stencil<T>(h, h->A0);
    if (!rc && !h->A0.dia && want_win) rc = device_windows<T>(h, h->A0, h->n_pad, (const T*)h->d_dinv);
    if (rc) return rc;
    tick(h->A0.dia ? "finest operator: stencil form" : "finest operator: windows");
  }
  if (want_amg) {
    rc = setup_amg_device<T>(h, hp, job, dseed);
    if (rc) return rc;
    if (h->amg && h->A0.dia && !h->P2) {   // second p panel of the fused CG step
      const size_t pe = (size_t)h->n_pad * h->ktmax * sizeof(T);
      cudaError_t e = cudaMalloc(&h->P2, pe);
      if (e == cudaSuccess) e = cudaMemsetAsync(h->P2, 0, pe, h->stream);
      if (e != cudaSuccess) return set_err(h, CS_B200_ERR_CUDA, "CUDA error %s (second p panel)", cudaGetErrorString(e));
    }
    if (h->P2 && fused_res_form(h)) {
      // the fused residual sweep rounds the fp64 diagonals to the fp32 level 0's on chip: it runs only where the
      // stored fp32 runs are exactly those roundings.  R2: its second r panel
      int* d_diff = nullptr;
      int diff = 1;
      cudaError_t e = cudaMalloc(&d_diff, sizeof(int));
      if (e == cudaSuccess) e = cudaMemsetAsync(d_diff, 0, sizeof(int), h->stream);
      if (e == cudaSuccess) {
        k_dia_rounds<T, float><<<std::min<int64_t>((5 * h->n + 255) / 256, 4096), 256, 0, h->stream>>>(
            dia_view<T>(h->A0), dia_view<float>(h->lv32[0].A), d_diff);
        e = cudaMemcpyAsync(&diff, d_diff, sizeof(int), cudaMemcpyDeviceToHost, h->stream);
      }
      if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
      cudaFree(d_diff);
      if (e == cudaSuccess && diff == 0 && !h->R2) {
        const size_t pe = (size_t)h->n_pad * h->ktmax * sizeof(T);
        e = cudaMalloc(&h->R2, pe);
        if (e == cudaSuccess) e = cudaMemsetAsync(h->R2, 0, pe, h->stream);
      } else if (diff != 0) {
        cudaFree(h->R2);
        h->R2 = nullptr;
      }
      if (e != cudaSuccess) return set_err(h, CS_B200_ERR_CUDA, "CUDA error %s (second r panel)", cudaGetErrorString(e));
    }
  }
  Tick tick1;
  csb_dev::trim_pool(h->device);
  tick1("scratch pool released");
  return CS_B200_OK;
}

// device-side setup of a handle whose CSR is resident: row blocks, panels, then build_operators
template <typename T>
int finish_setup_device(cs_b200_handle* h, const csb_dev::HostPattern& hp, csb_dev::SeedJob*& job,
                        const csb_dev::DeviceSeed* dseed) {
  h->A0 = DevCsr{h->d_rowptr, h->d_colidx, h->d_vals, nullptr, 0, (int)h->n, h->nnz, 1};
  Tick tick0;
  int rc = device_row_blocks(h, h->A0, NT);
  if (rc) return rc;
  h->d_bstart = h->A0.bstart;
  h->nblocks = h->A0.nblocks;
  rc = alloc_common<T>(h);
  if (rc) return rc;
  if (tick0.on) { cudaStreamSynchronize(h->stream); tick0("row blocks + panels"); }
  rc = build_operators<T>(h, hp, job, dseed);
  if (rc) return rc;
  return cs_b200_reset_currents(h);
}

int common_create(cs_b200_handle* h, const cs_b200_opts* opts) {
  if (opts) h->opts = *opts;
  if (h->opts.panel_width == 0) h->opts.panel_width = 8;
  if (h->opts.check_every <= 0) h->opts.check_every = 16;
  if (h->opts.resid_gate <= 0) h->opts.resid_gate = 1e-4;
  if (h->opts.use_graph == 0) h->opts.use_graph = 1;  // 0 -> default on; pass -1 to disable
  const int pw = h->opts.panel_width;
  if (pw != 1 && pw != 2 && pw != 4 && pw != 8)
    return set_err(h, CS_B200_ERR_ARG, "panel_width must be 1, 2, 4 or 8 (got %d)", pw);
  h->ktmax = pw;
  if (h->opts.precond != CS_B200_PRECOND_JACOBI && h->opts.precond != CS_B200_PRECOND_AMG)
    return set_err(h, CS_B200_ERR_UNSUPPORTED, "unknown preconditioner %d", h->opts.precond);
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return set_err(h, CS_B200_ERR_CUDA,
                   "no CUDA device available (%s): libcsb200 has no CPU fallback",
                   cudaGetErrorString(e));
  if (h->device < 0 || h->device >= ndev)
    return set_err(h, CS_B200_ERR_ARG, "device %d out of range (0..%d)", h->device, ndev - 1);
  CK(h, cudaSetDevice(h->device));
  cudaDeviceProp prop;
  CK(h, cudaGetDeviceProperties(&prop, h->device));
  h->num_sms = prop.multiProcessorCount;
  h->grid_spmm = h->num_sms * 8;
  h->grid_ew = h->num_sms * 4;
  CK(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  CK(h, cudaEventCreate(&h->ev0));
  CK(h, cudaEventCreate(&h->ev1));
  CK(h, cudaEventCreate(&h->ev2));
  CK(h, cudaEventCreate(&h->ev3));
  return CS_B200_OK;
}

// ---------------------------------------------------------------------------
// launch helpers (all on h->stream)
// ---------------------------------------------------------------------------
template <typename T>
CsrDev<T> view(const DevCsr& m) {
  return CsrDev<T>{m.rowptr, m.colidx, (const T*)m.vals, m.bstart, m.nblocks, m.nrows};
}

// The bookkeeping of one kernel launch, around the launch it scopes: the launch counters, and on profiled
// handles an event pair with the launch's class (slot 2 * cls + fp32) and algorithmic bytes (DESIGN.md §4).
// `timed`: a finest-level launch, counted in spmm_launches and profiled.
struct ProfScope {
  cs_b200_handle* h;
  cudaEvent_t e1 = nullptr;
  ProfScope(cs_b200_handle* h_, bool timed, int cls, bool fp32, double bytes) : h(h_) {
    h->stats.kernel_launches++;
    if (!timed) return;
    h->stats.spmm_launches++;
    if (!h->profile) return;
    if (h->prof_used + 2 > h->prof_ev.size())
      for (int i = 0; i < 2; ++i) { cudaEvent_t e; cudaEventCreate(&e); h->prof_ev.push_back(e); }
    const cudaEvent_t e0 = h->prof_ev[h->prof_used++];
    e1 = h->prof_ev[h->prof_used++];
    h->prof_bytes += bytes;
    h->prof_slot.push_back(2 * cls + (fp32 ? 1 : 0));
    h->prof_pair_bytes.push_back(bytes);
    cudaEventRecord(e0, h->stream);
  }
  ProfScope(const ProfScope&) = delete;
  ProfScope& operator=(const ProfScope&) = delete;
  ~ProfScope() { if (e1) cudaEventRecord(e1, h->stream); }
};

// raise Kernel's dynamic shared-memory limit to `bytes` on the handle's device, once per device (the attribute
// lives in the device's context); each kernel instantiation keeps its own flags
template <auto Kernel>
void set_max_smem_once(const cs_b200_handle* h, int bytes) {
  static bool once[64] = {};
  bool& set = once[h->device & 63];
  if (!set) { cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes); set = true; }
}

// grid of the stencil kernels on m (k_stencil, k_stencil_pipe, k_stencil_cg*): its tiles of NT / CGn rows by
// ST_TC raster columns, at most grid_spmm
template <typename T, int KT>
int stencil_grid(const cs_b200_handle* h, const DevCsr& m) {
  constexpr int V16 = 16 / (int)sizeof(T);
  constexpr int CGn = KT / (KT < V16 ? KT : V16);
  const int rpp = NT / CGn;
  const long long ntiles = (long long)((m.dia_nr + rpp - 1) / rpp) *
                           ((((long long)m.nrows + m.dia_nr - 1) / m.dia_nr + ST_TC - 1) / ST_TC);
  return (int)std::max<long long>(1, std::min<long long>(h->grid_spmm, ntiles));
}

// one resident wave of `kernel` (NT threads, smem bytes) over the (strip of rps rows, column) steps of the stencil
// operator m: every CTA's run of steps is as long as possible, which keeps the halo columns a CTA rebuilds at the
// start of each run rare.  Asked per launch, on the handle's device (host-side query; the launches are captured
// into graphs).
template <typename Kernel>
int wave_grid(const cs_b200_handle* h, Kernel kernel, int smem, const DevCsr& m, int rps) {
  int occ = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, NT, smem);
  occ = std::max(1, occ);
  const long long nsteps = (long long)((m.dia_nr + rps - 1) / rps) * (((long long)m.nrows + m.dia_nr - 1) / m.dia_nr);
  return (int)std::max<long long>(1, std::min<long long>(std::min(h->grid_spmm, h->num_sms * occ), nsteps));
}

// grid of the 256-thread copy kernels (k_panel_to_cm, k_cm_to_panel, k_combine, k_fill) over nelem elements
inline int copy_grid(size_t nelem) { return (int)std::min<size_t>(4096, (nelem + 255) / 256); }

template <typename T, int KT, int MODE, bool HALF>
void launch_stencil_pipe(cs_b200_handle* h, const DiaDev<T>& a, const T* X, T* Y, const SpmmEpi<T>& ep, int sg) {
  constexpr int SMEM = StPipe<T, KT, MODE, HALF>::D::BYTES;
  set_max_smem_once<k_stencil_pipe<T, KT, MODE, HALF>>(h, SMEM);
  k_stencil_pipe<T, KT, MODE, HALF><<<sg, NT, SMEM, h->stream>>>(a, X, Y, ep);
}

// k_stencil<T, KT, MODE> on grid sg, through the pipeline unless it is switched off
template <typename T, int KT, int MODE>
void launch_stencil(cs_b200_handle* h, const DiaDev<T>& a, const T* X, T* Y, const SpmmEpi<T>& ep, int sg) {
  if (!stencil_pipe()) {
    if (a.half) refuse_half("k_stencil");
    k_stencil<T, KT, MODE><<<sg, NT, 0, h->stream>>>(a, X, Y, ep);
    return;
  }
  if (a.half) launch_stencil_pipe<T, KT, MODE, true>(h, a, X, Y, ep, sg);
  else launch_stencil_pipe<T, KT, MODE, false>(h, a, X, Y, ep, sg);
}

// the TMA-staged windowed kernel (WIDE: 4 lanes per row) on m's windowed row blocks
template <typename T, int KT, int MODE, bool WIDE>
void launch_spmm_win(cs_b200_handle* h, const DevCsr& m, const T* X, T* Y, const SpmmEpi<T>& ep) {
  constexpr int SMEM = WinSmem2<T, KT, MODE, WIDE>::TOTAL;
  constexpr int SB = WinMap<T, KT, WIDE>::SB;
  const WinCsr<T> w{m.win_meta, m.blob, m.has_dinv, m.rowptr, m.colidx, (const T*)m.vals, m.win_nblocks};
  const int wg = std::max(1, std::min(h->num_sms, (m.win_nblocks + SB - 1) / SB));
  set_max_smem_once<k_spmm_win<T, KT, MODE, WIDE>>(h, SMEM);
  k_spmm_win<T, KT, MODE, WIDE><<<wg, WTT, SMEM, h->stream>>>(w, X, Y, ep);
}

// Y = op(M X) with the fused epilogue MODE (kernels.cuh).  `timed`: counts as a launch of
// the dominant kernel for the per-launch profile (finest-level operator only).
template <typename T, int KT, int MODE>
void launch_spmm_on(cs_b200_handle* h, const DevCsr& m, const T* X, T* Y, const T* B, const T* dinv,
                    double omega, bool timed, bool pair_b = false) {
  const int grid = std::max(1, std::min(h->grid_spmm, m.nblocks));
  // nnz (s_v + 4) + (n + 1) 4 + X once + Y once (+ B for the residual / sweep epilogues,
  // + 1/diag for the sweeps); pair_b (stencil residual gate of a pairs panel): neither B nor Y
  double bytes = (double)m.nnz * (sizeof(T) + 4) + (double)(m.nrows + 1) * 4 +
                 2.0 * (double)m.nrows * KT * sizeof(T);
  if (MODE == SP_RESNORM || MODE == SP_RES || MODE == SP_JACOBI || MODE == SP_JACOBI_DOT)
    bytes += (double)m.nrows * KT * sizeof(T);
  if (MODE == SP_JACOBI || MODE == SP_JACOBI_DOT) bytes += (double)m.nrows * sizeof(T);
  if (pair_b) bytes -= 2.0 * (double)m.nrows * KT * sizeof(T);
  const ProfScope prof(h, timed, MODE, sizeof(T) == 4, bytes);
  const SpmmEpi<T> ep{B, dinv, (T)omega, h->d_ctl, h->d_partials, pair_b ? 1 : 0};
  if (m.dia && MODE != SP_ADD) {
    if constexpr (MODE != SP_ADD) launch_stencil<T, KT, MODE>(h, dia_view<T>(m), X, Y, ep, stencil_grid<T, KT>(h, m));
  } else if (m.win_meta) {
    if (m.lpr == 4) launch_spmm_win<T, KT, MODE, true>(h, m, X, Y, ep);
    else launch_spmm_win<T, KT, MODE, false>(h, m, X, Y, ep);
  } else if (m.lpr == 4 && KT * 4 <= 32) {
    k_spmm<T, KT, MODE, (KT * 4 <= 32 ? 4 : 1)><<<grid, NT, 0, h->stream>>>(view<T>(m), X, Y, ep);
  } else {
    k_spmm<T, KT, MODE, 1><<<grid, NT, 0, h->stream>>>(view<T>(m), X, Y, ep);
  }
}

template <typename T, int KT, int MODE>
void launch_spmm(cs_b200_handle* h, const T* X, T* Y, const T* B) {
  launch_spmm_on<T, KT, MODE>(h, h->A0, X, Y, B, (const T*)h->d_dinv, 0.0, true);
}

// after a stream sync: fold the recorded SpMM event pairs into the profile totals
void harvest_profile(cs_b200_handle* h) {
  for (size_t i = 0; i + 1 < h->prof_used; i += 2) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, h->prof_ev[i], h->prof_ev[i + 1]) == cudaSuccess) {
      h->prof_ms += ms;
      h->prof_launches++;
      if (i / 2 < h->prof_slot.size()) {
        const int sl = h->prof_slot[i / 2];
        h->prof_slot_ms[sl] += ms;
        h->prof_slot_bytes[sl] += h->prof_pair_bytes[i / 2];
        h->prof_slot_launches[sl]++;
      }
    }
  }
  h->prof_used = 0;
  h->prof_slot.clear();
  h->prof_pair_bytes.clear();
}

template <typename T, int KT>
int ew_grid_n(cs_b200_handle* h, int64_t n_pad) {
  const size_t nelem = (size_t)n_pad * KT;
  const size_t per = (size_t)NT * Vec<T>::N;
  return (int)std::max<size_t>(1, std::min<size_t>(h->grid_ew, (nelem + per - 1) / per));
}

// the finest level's
template <typename T, int KT>
int ew_grid(cs_b200_handle* h) { return ew_grid_n<T, KT>(h, h->n_pad); }

// T = B - A (omega D^-1 B) on a stencil-form level
template <typename T, int KT>
void launch_stencil_res0(cs_b200_handle* h, DevLevel& L, const T* B, T* Tout, bool timed) {
  const DevCsr& m = L.A;
  const DiaDev<T> a = dia_view<T>(m);
  const SpmmEpi<T> ep{B, (const T*)L.dinv, (T)L.omega, h->d_ctl, h->d_partials};
  // what it replaces: the residual SpMM on A (X, B read, T written); the zero-guess sweep is folded in
  const double fb = (double)m.nnz * (sizeof(T) + 4) + (double)(m.nrows + 1) * 4 + 3.0 * (double)m.nrows * KT * sizeof(T);
  const ProfScope prof(h, timed, SP_RES, sizeof(T) == 4, fb);
  launch_stencil<T, KT, SP_RES0>(h, a, nullptr, Tout, ep, stencil_grid<T, KT>(h, m));
}

// fused upward step of a stencil-form level (kernels.cuh k_stencil_prolong_jacobi):
//   Yout = (X0 + P Yc) + omega D^-1 (B - A (X0 + P Yc))   [+ dot(B, Yout) on the finest level]
template <typename T, int KT, int MODE>
void launch_prolong_jacobi(cs_b200_handle* h, DevLevel& L, const T* Yc, const T* X0, T* Yout, const T* B, bool timed) {
  const DevCsr& m = L.A;
  const DiaDev<T> a = dia_view<T>(m);
  const CsrP<T> p{L.P.rowptr, L.P.colidx, (const T*)L.P.vals, L.P.ell_col, (const T*)L.P.ell_val, L.P.ell_ld};
  const SpmmEpi<T> ep{B, (const T*)L.dinv, (T)L.omega, h->d_ctl, h->d_partials};
  using S = PjShape<T, KT>;
  constexpr int SMEM = S::SMEM;
  constexpr int MINB = sizeof(T) == 4 ? PJ_MINB_F32 : PJ_MINB_F64;
  static_assert(SMEM <= 48 * 1024, "the strip buffers fit the default dynamic shared memory");
  const int grid = wave_grid(h, k_stencil_prolong_jacobi<T, KT, MODE, MINB>, SMEM, m, S::RPS);
  // the two launches it replaces: SP_ADD on P (nnz_P (s+4) + (n+1) 4 + Yc + X read + X write) and the
  // Jacobi sweep on A (nnz (s+4) + (n+1) 4 + X + Y + B + 1/diag)
  const double fb = (double)m.nnz * (sizeof(T) + 4) + (double)(m.nrows + 1) * 4 + 3.0 * (double)m.nrows * KT * sizeof(T) +
                    (double)m.nrows * sizeof(T) + (double)L.P.nnz * (sizeof(T) + 4) + (double)(m.nrows + 1) * 4 +
                    2.0 * (double)m.nrows * KT * sizeof(T);
  const ProfScope prof(h, timed, PROF_PJ, sizeof(T) == 4, fb);
  k_stencil_prolong_jacobi<T, KT, MODE, MINB><<<grid, NT, SMEM, h->stream>>>(a, p, Yc, X0, Yout, ep);
}

// z = M^-1 r : one V(1,1) cycle, damped Jacobi, on panels of width KT.
//   in : h->R (residual, read-only)      out: h->Z ; rho_new = r.z folded into the last kernel
// Level buffers: b = right-hand side, x = running correction, t = residual scratch,
// y = post-smoothed correction.  Finest level: b = R, x = stage, t = AP, y = Z.
// level0_residual: t of the finest level is already formed (k_stencil_res_update); the cycle starts at the
// restriction.
struct VcBufs { void *b0, *x0, *t0, *y0; };   // finest-level panels of the cycle

template <typename T, int KT>
void launch_vcycle_on(cs_b200_handle* h, std::vector<DevLevel>& lv, const VcBufs& vb, bool level0_presmoothed,
                      bool level0_residual) {
  const int nl = (int)lv.size();
  auto B = [&](int l) { return l == 0 ? (T*)vb.b0 : (T*)lv[l].b; };
  auto X = [&](int l) { return l == 0 ? (T*)vb.x0 : (T*)lv[l].x; };
  auto Tm = [&](int l) { return l == 0 ? (T*)vb.t0 : (T*)lv[l].t; };
  auto Y = [&](int l) { return l == 0 ? (T*)vb.y0 : (T*)lv[l].y; };
  for (int l = 0; l < nl - 1; ++l) {
    DevLevel& L = lv[l];
    const size_t nelem = (size_t)L.n_pad * KT;
    if (implicit_x0(L)) {
      if (!(l == 0 && level0_residual)) launch_stencil_res0<T, KT>(h, L, B(l), Tm(l), l == 0);
    } else {
      if (!(l == 0 && level0_presmoothed)) {
        k_jacobi0<T, KT><<<ew_grid_n<T, KT>(h, L.n_pad), NT, 0, h->stream>>>(
            nelem, B(l), (const T*)L.dinv, (T)L.omega, X(l));
        h->stats.kernel_launches++;
      }
      launch_spmm_on<T, KT, SP_RES>(h, L.A, X(l), Tm(l), B(l), nullptr, 0.0, l == 0);
    }
    launch_spmm_on<T, KT, SP_PLAIN>(h, L.R, Tm(l), B(l + 1), nullptr, nullptr, 0.0, false);
  }
  {
    DevLevel& C = lv[nl - 1];
    if (h->d_pinv) {
      k_coarse_dense<T, KT><<<((int)C.n * KT + NT - 1) / NT, NT, 0, h->stream>>>((int)C.n, h->d_pinv, (const T*)B(nl - 1), Y(nl - 1));
      h->stats.kernel_launches++;
    } else {  // coarsening stalled above the dense limit: 4 damped-Jacobi sweeps (symmetric)
      const int l = nl - 1;
      k_jacobi0<T, KT><<<ew_grid_n<T, KT>(h, C.n_pad), NT, 0, h->stream>>>(
          (size_t)C.n_pad * KT, B(l), (const T*)C.dinv, (T)C.omega, X(l));
      h->stats.kernel_launches++;
      launch_spmm_on<T, KT, SP_JACOBI>(h, C.A, X(l), Y(l), B(l), (const T*)C.dinv, C.omega, false);
      launch_spmm_on<T, KT, SP_JACOBI>(h, C.A, Y(l), X(l), B(l), (const T*)C.dinv, C.omega, false);
      launch_spmm_on<T, KT, SP_JACOBI>(h, C.A, X(l), Y(l), B(l), (const T*)C.dinv, C.omega, false);
    }
  }
  static const bool fuse_off = std::getenv("CS_B200_NO_FUSED_PROLONG") != nullptr;
  for (int l = nl - 2; l >= 0; --l) {
    DevLevel& L = lv[l];
    if (L.A.dia && !fuse_off) {
      // stencil-form level: prolongate + correct + post-smooth in one kernel (x1 stays in shared memory)
      const T* x0 = implicit_x0(L) ? nullptr : X(l);
      if (l == 0) launch_prolong_jacobi<T, KT, SP_JACOBI_DOT>(h, L, Y(l + 1), x0, Y(l), B(l), true);
      else launch_prolong_jacobi<T, KT, SP_JACOBI>(h, L, Y(l + 1), x0, Y(l), B(l), false);
      continue;
    }
    launch_spmm_on<T, KT, SP_ADD>(h, L.P, Y(l + 1), X(l), X(l) /* staged as B */, nullptr, 0.0, false);
    if (l == 0)
      launch_spmm_on<T, KT, SP_JACOBI_DOT>(h, L.A, X(l), Y(l), B(l), (const T*)L.dinv, L.omega, true);
    else
      launch_spmm_on<T, KT, SP_JACOBI>(h, L.A, X(l), Y(l), B(l), (const T*)L.dinv, L.omega, false);
  }
}

// the cycle of this handle: fp32 copies when `mixed`, else the handle's own type
template <typename T, int KT>
void launch_vcycle(cs_b200_handle* h, bool level0_presmoothed, bool level0_residual = false) {
  if (h->mixed) {
    const VcBufs vb{h->R32, h->X32, h->T32, h->Z32};
    launch_vcycle_on<float, KT>(h, h->lv32, vb, level0_presmoothed, level0_residual);
  } else {
    const VcBufs vb{h->R, h->stage, h->AP, h->Z};
    launch_vcycle_on<T, KT>(h, h->lv, vb, level0_presmoothed, level0_residual);
  }
}

// region panels: zero the set rows of a panel (Dirichlet mask), or set the set_b rows to v
template <typename T, int KT>
void launch_seg_set(cs_b200_handle* h, void* panel, int set_b_only, T v) {
  k_seg_set<T, KT><<<2 * KT, NT, 0, h->stream>>>((T*)panel, h->d_rg_seg, h->d_rg_rows, set_b_only, v);
  h->stats.kernel_launches++;
}

// z = mask M^-1 mask r on a region panel (r is zero on the sets already)
template <typename T, int KT>
void mask_z(cs_b200_handle* h) {
  if (!h->rg_on) return;
  if (h->mixed) launch_seg_set<float, KT>(h, h->Z32, 0, 0.0f);
  else launch_seg_set<T, KT>(h, h->Z, 0, T(0));
}

inline GraphSlot& graph_slot(cs_b200_handle* h, int kt) {
  return (h->rg_on ? h->rgraphs : h->graphs)[kt_index(kt)];
}

void drop_graphs(GraphSlot* slots) {
  for (int i = 0; i < 4; ++i) {
    if (slots[i].exec) cudaGraphExecDestroy(slots[i].exec);
    if (slots[i].loop_exec) cudaGraphExecDestroy(slots[i].loop_exec);
    slots[i] = GraphSlot{};
  }
}

// AMG-PCG on a stencil-form finest level runs the fused CG step (kernels.cuh k_stencil_cg) in place of the
// CG SpMM and k_cg_update_xp2; CS_B200_NO_FUSED_CG keeps the unfused pair for A/B runs
inline bool fused_cg(const cs_b200_handle* h) {
  static const bool off = std::getenv("CS_B200_NO_FUSED_CG") != nullptr;
  return h->amg && h->A0.dia && h->P2 && !off;
}

// the iteration runs the fused residual sweep; region panels mask AP between the CG step and the residual
// update, so they keep k_cg_update_r0
inline bool fused_res(const cs_b200_handle* h) {
  return fused_cg(h) && h->R2 && !h->rg_on && fused_res_form(h);
}

// The passes around a fused AMG-PCG panel's loop (pipelined stencil kernels): X and P are not zero-filled (the
// CG step and k_cg_x_tail read the zeros they would hold as zeros), r and r32 come from one pass
// (k_panel_start), and a pairs panel writes no B: its start pass and residual gate take b from ctl, and the gate
// stores no B - A X (nothing reads it after a pairs panel).  CS_B200_NO_FUSED_PANEL_ENDS keeps the fills,
// B, the copy and the conversion for A/B runs.
inline bool panel_ends(const cs_b200_handle* h) {
  static const bool off = std::getenv("CS_B200_NO_FUSED_PANEL_ENDS") != nullptr;
  return !off && fused_cg(h) && stencil_pipe();
}

template <typename T, int KT, typename TV, bool HALF, bool STORE_AP>
void launch_stencil_cg_pipe(cs_b200_handle* h, const DiaDev<T>& a, const TV* Z, int sg) {
  constexpr int SMEM = StPipeCg<T, KT, TV, HALF>::D::BYTES;
  set_max_smem_once<k_stencil_cg_pipe<T, KT, TV, HALF, STORE_AP>>(h, SMEM);
  k_stencil_cg_pipe<T, KT, TV, HALF, STORE_AP><<<sg, NT, SMEM, h->stream>>>(a, Z, (T*)h->P2, (T*)h->P, (T*)h->X,
                                                                            (T*)h->AP, h->d_ctl, h->d_partials);
}

// the z panel the CG update reads: the fp32 cycle's output on mixed handles.  !store_ap (fused_res): A p is not
// stored, the residual sweep forms it again.
template <typename T, int KT, typename TV>
void launch_stencil_cg(cs_b200_handle* h, const TV* Z, bool store_ap) {
  const DevCsr& m = h->A0;
  const DiaDev<T> a = dia_view<T>(m);
  const int sg = stencil_grid<T, KT>(h, m);   // = k_stencil<SP_CG>'s
  // 9 diagonals, Z and p_{it-1} in, AP (store_ap) and p_it out; X in + out and p_{it-2} in on every other step
  const double pe = (double)m.nrows * KT * sizeof(T);
  const double fb = (double)m.nrows * 9 * sizeof(T) + (double)m.nrows * KT * sizeof(TV) + (store_ap ? 3.0 : 2.0) * pe +
                    1.5 * pe;
  const ProfScope prof(h, true, PROF_CGF, sizeof(T) == 4, fb);
  if (stencil_pipe()) {
    if (!store_ap) {   // fused_res: fp64 with an fp32 cycle, half form
      if constexpr (sizeof(T) == 8 && sizeof(TV) == 4) launch_stencil_cg_pipe<T, KT, TV, true, false>(h, a, Z, sg);
    } else if (a.half) launch_stencil_cg_pipe<T, KT, TV, true, true>(h, a, Z, sg);
    else launch_stencil_cg_pipe<T, KT, TV, false, true>(h, a, Z, sg);
  } else {
    if (a.half) refuse_half("k_stencil_cg");
    k_stencil_cg<T, KT, TV><<<sg, NT, 0, h->stream>>>(a, Z, (T*)h->P2, (T*)h->P, (T*)h->X, (T*)h->AP, h->d_ctl,
                                                       h->d_partials);
  }
}

// r -= alpha A p, r32 = (float) r and the level-0 residual T32 of the fp32 cycle (kernels.cuh
// k_stencil_res_update), in place of k_cg_update_r0 and the cycle's level-0 SP_RES0 sweep
template <typename T, int KT>
void launch_res_update(cs_b200_handle* h) {
  const DevCsr& m = h->A0;
  DevLevel& L = h->lv32[0];
  using SH = RuShape<T, float, KT>;
  constexpr int SMEM = SH::D::BYTES;
  set_max_smem_once<k_stencil_res_update<T, float, KT>>(h, SMEM);
  const int grid = wave_grid(h, k_stencil_res_update<T, float, KT>, SMEM, m, SH::RPS);
  // p, r in and r out (T), R32 and T32 out (float), the 5 upper diagonals (T), the float 1/diag
  const double nr = (double)m.nrows;
  const double fb = nr * KT * (3.0 * sizeof(T) + 2.0 * sizeof(float)) + nr * 5 * sizeof(T) + nr * sizeof(float);
  const ProfScope prof(h, true, PROF_RSW, sizeof(T) == 4, fb);
  k_stencil_res_update<T, float, KT><<<grid, NT, SMEM, h->stream>>>(
      dia_view<T>(m), (const float*)L.dinv, (float)L.omega, (const T*)h->P2, (const T*)h->P,
      (T*)h->R, (T*)h->R2, (float*)h->R32, (float*)h->T32, h->d_ctl);
}

// r -= alpha Ap with the finest pre-smoothing folded in, into the cycle's own precision (k_cg_update_r0): the fp32
// r32 and x0 panels of a mixed handle, else x0 in the stage panel; no x0 where it stays implicit
template <typename T, int KT>
void launch_update_r0(cs_b200_handle* h) {
  const size_t nelem = (size_t)h->n_pad * KT;
  const int g = ew_grid<T, KT>(h);
  if (h->mixed)
    k_cg_update_r0<T, KT, float><<<g, NT, 0, h->stream>>>(nelem, (const T*)h->AP, (const T*)h->d_dinv,
                                                          (T)h->lv[0].omega, (T*)h->R,
                                                          implicit_x0(h->lv32[0]) ? nullptr : (float*)h->X32,
                                                          (float*)h->R32, h->d_ctl);
  else
    k_cg_update_r0<T, KT, T><<<g, NT, 0, h->stream>>>(nelem, (const T*)h->AP, (const T*)h->d_dinv, (T)h->lv[0].omega,
                                                      (T*)h->R, implicit_x0(h->lv[0]) ? nullptr : (T*)h->stage, nullptr,
                                                      h->d_ctl);
  h->stats.kernel_launches++;
}

// the deferred x += alpha p with p = z + beta p (k_cg_update_xp2), z the cycle's output: Z32 on mixed handles
template <typename T, int KT>
void launch_update_xp2(cs_b200_handle* h) {
  const size_t nelem = (size_t)h->n_pad * KT;
  const int g = ew_grid<T, KT>(h);
  if (h->mixed)
    k_cg_update_xp2<T, KT, float><<<g, NT, 0, h->stream>>>(nelem, (const float*)h->Z32, (T*)h->X, (T*)h->P, h->d_ctl);
  else
    k_cg_update_xp2<T, KT, T><<<g, NT, 0, h->stream>>>(nelem, (const T*)h->Z, (T*)h->X, (T*)h->P, h->d_ctl);
  h->stats.kernel_launches++;
}

template <typename T, int KT>
void launch_iteration(cs_b200_handle* h) {
  const size_t nelem = (size_t)h->n_pad * KT;
  const int g = ew_grid<T, KT>(h);
  const bool fused = fused_cg(h);
  const bool fres = sizeof(T) == 8 && fused_res(h);   // fused_res: mixed handles, which are fp64 ones
  if (fused) {
    if (h->mixed) launch_stencil_cg<T, KT, float>(h, (const float*)h->Z32, !fres);
    else launch_stencil_cg<T, KT, T>(h, (const T*)h->Z, true);
  } else {
    launch_spmm<T, KT, SP_CG>(h, (const T*)h->P, (T*)h->AP, nullptr);
  }
  // region panel: r stays zero on the sets (p is zero there, so p.Ap needs no mask)
  if (h->rg_on) launch_seg_set<T, KT>(h, h->AP, 0, T(0));
  if (!h->amg) {
    k_cg_update_r<T, KT><<<g, NT, 0, h->stream>>>(nelem, (const T*)h->AP, (const T*)h->d_dinv,
                                                  (T*)h->R, h->d_ctl, h->d_partials);
    k_cg_update_xp<T, KT><<<g, NT, 0, h->stream>>>(nelem, (const T*)h->R, (const T*)h->d_dinv,
                                                   (T*)h->X, (T*)h->P, h->d_ctl);
    h->stats.kernel_launches += 2;
  } else {
    // r -= alpha Ap with the finest pre-smoothing folded in; V-cycle; then the deferred
    // x += alpha p together with p = z + beta p  (9 instead of 11 panel passes), which the fused
    // CG step of the next iteration does instead
    if (fres) {
      if constexpr (sizeof(T) == 8) launch_res_update<T, KT>(h);
    } else {
      launch_update_r0<T, KT>(h);
    }
    launch_vcycle<T, KT>(h, true, fres);
    mask_z<T, KT>(h);
    if (!fused) launch_update_xp2<T, KT>(h);
  }
}

// after the PCG loop: the x updates the fused CG steps left pending
template <typename T, int KT>
void finish_x(cs_b200_handle* h) {
  if (!fused_cg(h)) return;
  k_cg_x_tail<T, KT><<<ew_grid<T, KT>(h), NT, 0, h->stream>>>((size_t)h->n_pad * KT, (const T*)h->P2, (const T*)h->P,
                                                             (T*)h->X, h->d_ctl);
  h->stats.kernel_launches++;
}

template <typename T, int KT>
int run_chunk(cs_b200_handle* h, int chunk) {
  GraphSlot& gs = graph_slot(h, KT);
  if (h->opts.use_graph > 0 && !h->profile) {   // use_graph == 2: host-polled chunks
    if (!gs.exec || gs.chunk != chunk) {
      if (gs.exec) cudaGraphExecDestroy(gs.exec);
      gs.exec = nullptr;
      cudaGraph_t graph;
      const int64_t kl = h->stats.kernel_launches, sl = h->stats.spmm_launches;
      CK(h, cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
      for (int i = 0; i < chunk; ++i) launch_iteration<T, KT>(h);
      CK(h, cudaStreamEndCapture(h->stream, &graph));
      gs.kernels = h->stats.kernel_launches - kl;
      gs.spmms = h->stats.spmm_launches - sl;
      h->stats.kernel_launches = kl;
      h->stats.spmm_launches = sl;
      CK(h, cudaGraphInstantiate(&gs.exec, graph, 0));
      cudaGraphDestroy(graph);
      gs.chunk = chunk;
    }
    CK(h, cudaGraphLaunch(gs.exec, h->stream));
    h->stats.kernel_launches += gs.kernels;
    h->stats.spmm_launches += gs.spmms;
  } else {
    for (int i = 0; i < chunk; ++i) launch_iteration<T, KT>(h);
    CK(h, cudaGetLastError());
  }
  return CS_B200_OK;
}

// The whole PCG loop of a panel as ONE graph launch: a kernel node that evaluates the loop
// condition, then a WHILE conditional node whose body is one captured iteration followed by
// the condition kernel.  The device decides when to stop (cg_after_precond / k_cg_update_r
// clear ctl->nactive; itmax bounds the loop), the host neither polls nor re-launches.
template <typename T, int KT>
int run_loop(cs_b200_handle* h) {
  GraphSlot& gs = graph_slot(h, KT);
  if (!gs.loop_exec) {
    cudaGraph_t graph;
    CK(h, cudaGraphCreate(&graph, 0));
    cudaGraphConditionalHandle cond;
    CK(h, cudaGraphConditionalHandleCreate(&cond, graph, 0, cudaGraphCondAssignDefault));
    cudaGraphNode_t n_pre, n_while;
    PanelCtl* ctl = h->d_ctl;
    void* args[] = {&cond, &ctl};
    cudaKernelNodeParams kp = {};
    kp.func = (void*)k_loop_cond;
    kp.gridDim = dim3(1);
    kp.blockDim = dim3(1);
    kp.kernelParams = args;
    CK(h, cudaGraphAddKernelNode(&n_pre, graph, nullptr, 0, &kp));
    cudaGraphNodeParams cp = {cudaGraphNodeTypeConditional};
    cp.conditional.handle = cond;
    cp.conditional.type = cudaGraphCondTypeWhile;
    cp.conditional.size = 1;
    CK(h, cudaGraphAddNode(&n_while, graph, &n_pre, 1, &cp));
    cudaGraph_t body = cp.conditional.phGraph_out[0];
    const int64_t kl = h->stats.kernel_launches, sl = h->stats.spmm_launches;
    CK(h, cudaStreamBeginCaptureToGraph(h->stream, body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
    launch_iteration<T, KT>(h);
    k_loop_cond<<<1, 1, 0, h->stream>>>(cond, h->d_ctl);
    CK(h, cudaStreamEndCapture(h->stream, nullptr));
    gs.loop_kernels = h->stats.kernel_launches - kl + 1;
    gs.loop_spmms = h->stats.spmm_launches - sl;
    h->stats.kernel_launches = kl;
    h->stats.spmm_launches = sl;
    CK(h, cudaGraphInstantiate(&gs.loop_exec, graph, 0));
    cudaGraphDestroy(graph);
  }
  CK(h, cudaGraphLaunch(gs.loop_exec, h->stream));
  return CS_B200_OK;
}

// Solve A X = B for the panel whose B is already staged (or, h->pair_b, whose b is the pairs rule of ctl) and
// whose ctl (src/dst/weight) has been uploaded.  Leaves X = solution, ctl (host copy) updated (resid, bnorm) and
// AP = B - A X, except on a pair_b panel, where AP is not written (nothing reads it after a pairs panel).
template <typename T, int KT>
int solve_panel(cs_b200_handle* h, double rtol, int64_t itmax) {
  const size_t nelem = (size_t)h->n_pad * KT;
  // Krylov.jl's default is sqrt(eps(T)); for T = Float32 that (3.5e-4) sits ABOVE the
  // reference's own 1e-4 residual gate, so the fp32 path keeps the fp64 value.
  const double atol = h->opts.atol > 0 ? h->opts.atol
                      : h->opts.atol < 0 ? 0.0
                      : std::sqrt(std::numeric_limits<double>::epsilon());
  const int g = ew_grid<T, KT>(h);
  const int imax = (int)std::min<int64_t>(itmax, std::numeric_limits<int>::max() - 1);
  CK(h, cudaEventRecord(h->ev2, h->stream));
  if (!h->amg) {
    k_set_stall<<<1, 1, 0, h->stream>>>(h->d_ctl, 2000);
    k_cg_init<T, KT><<<g, NT, 0, h->stream>>>(nelem, (const T*)h->B, (const T*)h->d_dinv, (T*)h->X,
                                              (T*)h->R, (T*)h->P, h->d_ctl, h->d_partials, rtol, atol,
                                              imax);
    h->stats.kernel_launches++;
  } else {
    // x = 0, p = 0, r = b ; z = M^-1 r (V-cycle; its last kernel sets rho0, tolerances,
    // activity because ctl->init = 1) ; p = z + 0*p  (fused CG step: formed by the first step, which
    // takes p_{-1} = 0 with beta = 0 -- read from the zero-filled P, or under panel_ends staged as zeros with
    // P not filled)
    const bool fused = fused_cg(h);
    if (panel_ends(h)) {
      // x = 0 and p = 0 stay implicit; r (and r32) in one pass, from ctl on a pairs panel
      k_set_ctl<<<1, 1, 0, h->stream>>>(h->d_ctl, rtol, atol, imax, 40);
      k_panel_start<T, KT><<<g, NT, 0, h->stream>>>(nelem, h->pair_b ? nullptr : (const T*)h->B, (T*)h->R,
                                                    h->mixed ? (float*)h->R32 : nullptr, h->d_ctl);
      h->stats.kernel_launches += 2;
    } else {
      CK(h, cudaMemsetAsync(h->X, 0, nelem * sizeof(T), h->stream));
      CK(h, cudaMemsetAsync(h->P, 0, nelem * sizeof(T), h->stream));
      CK(h, cudaMemcpyAsync(h->R, h->B, nelem * sizeof(T), cudaMemcpyDeviceToDevice, h->stream));
      k_set_ctl<<<1, 1, 0, h->stream>>>(h->d_ctl, rtol, atol, imax, 40);
      h->stats.kernel_launches++;
      if (h->mixed) {
        k_convert<T, float><<<g, NT, 0, h->stream>>>(nelem, (const T*)h->R, (float*)h->R32);
        h->stats.kernel_launches++;
      }
    }
    launch_vcycle<T, KT>(h, false);
    mask_z<T, KT>(h);
    if (!fused) launch_update_xp2<T, KT>(h);
  }
  CK(h, cudaGetLastError());
  const int chunk = h->amg ? std::min(h->opts.check_every, 4) : h->opts.check_every;
  const bool device_loop = h->opts.use_graph == 1 && !h->profile;
  if (device_loop) {
    int rc = run_loop<T, KT>(h);
    if (rc) return rc;
  }
  for (;;) {
    CK(h, cudaMemcpyAsync(h->h_ctl, h->d_ctl, sizeof(PanelCtl), cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    if (h->profile) harvest_profile(h);
    if (device_loop) {
      GraphSlot& gs = graph_slot(h, KT);
      h->stats.kernel_launches += 1 + gs.loop_kernels * h->h_ctl->iter;
      h->stats.spmm_launches += gs.loop_spmms * h->h_ctl->iter;
      break;
    }
    if (h->h_ctl->nactive == 0) break;
    int rc = run_chunk<T, KT>(h, chunk);
    if (rc) return rc;
  }
  if (h->amg) finish_x<T, KT>(h);
  // true residual  AP = B - A X  (core.jl:640, 648-651)
  if (h->rg_on) {
    // masked system: the set rows of B - A X hold the flux, not a residual -> zero them, then the norms
    launch_spmm<T, KT, SP_RES>(h, (const T*)h->X, (T*)h->AP, (const T*)h->B);
    launch_seg_set<T, KT>(h, h->AP, 0, T(0));
    k_resnorm<T, KT><<<g, NT, 0, h->stream>>>(nelem, (size_t)h->n * KT, (const T*)h->AP, (const T*)h->B, h->d_ctl, h->d_partials);
    h->stats.kernel_launches++;
  } else {
    // pair_b: b from ctl, AP not written
    launch_spmm_on<T, KT, SP_RESNORM>(h, h->A0, (const T*)h->X, (T*)h->AP, (const T*)h->B, (const T*)h->d_dinv, 0.0,
                                      true, h->pair_b);
  }
  CK(h, cudaGetLastError());
  CK(h, cudaEventRecord(h->ev3, h->stream));
  CK(h, cudaMemcpyAsync(h->h_ctl, h->d_ctl, sizeof(PanelCtl), cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  if (h->profile) harvest_profile(h);
  float ms = 0;
  CK(h, cudaEventElapsedTime(&ms, h->ev2, h->ev3));
  h->stats.kernel_ms += ms;
  return CS_B200_OK;
}

int next_kt(int64_t remaining, int ktmax) {
  int kt = ktmax;
  while (kt > remaining) kt >>= 1;
  return kt < 1 ? 1 : kt;
}

#define DISPATCH_KT(kt, CALL)                    \
  switch (kt) {                                  \
    case 1: { constexpr int KT = 1; CALL; } break; \
    case 2: { constexpr int KT = 2; CALL; } break; \
    case 4: { constexpr int KT = 4; CALL; } break; \
    default: { constexpr int KT = 8; CALL; } break; \
  }

// f(T{}) in the handle's element type T
template <typename F>
decltype(auto) with_type(const cs_b200_handle* h, F&& f) {
  return h->dtype == CS_B200_F64 ? f(double{}) : f(float{});
}

// f(KT) for panel width kt (1, 2, 4, 8), KT a std::integral_constant
template <typename F>
decltype(auto) with_width(int kt, F&& f) {
  DISPATCH_KT(kt, return f(std::integral_constant<int, KT>{}));
}

// f(T{}, KT): with_type, then with_width
template <typename F>
decltype(auto) with_type_width(const cs_b200_handle* h, int kt, F&& f) {
  return with_type(h, [&](auto t) -> decltype(auto) {
    return with_width(kt, [&](auto KT) -> decltype(auto) { return f(t, KT); });
  });
}

// The column driver of the batched solve entries: walks a call's columns in panels, collects every
// column's residual-gate and itmax status, and maps them to the call's return code.
struct ColumnDriver {
  cs_b200_handle* h;
  bool any_fail = false, any_maxit = false;
  std::string msg;   // the first column over the residual gate

  // columns c_begin .. c_end-1 in panels of next_kt width: panel(KT, c0) with KT a std::integral_constant;
  // stops at the first panel that fails
  template <typename Panel>
  int run(int64_t c_begin, int64_t c_end, Panel&& panel) {
    for (int64_t c0 = c_begin; c0 < c_end;) {
      const int kt = next_kt(c_end - c0, h->ktmax);
      if (int rc = with_width(kt, [&](auto KT) { return panel(KT, c0); })) return rc;
      c0 += kt;
    }
    return CS_B200_OK;
  }

  // solve_panel on the staged panel of columns c0 .. c0+KT-1 (under its Dirichlet segments when masked), then
  // gather its status
  template <typename T, int KT>
  int solve(int64_t c0, double rtol, int64_t itmax, int64_t* iters, double* relres, bool masked = false) {
    h->rg_on = masked;
    const int rc = solve_panel<T, KT>(h, rtol, itmax);
    h->rg_on = false;
    h->pair_b = false;
    if (!rc) gather(KT, c0, iters, relres, itmax);
    return rc;
  }

  // the status of the panel whose solve_panel just returned (columns c0 .. c0+kt-1)
  void gather(int kt, int64_t c0, int64_t* iters, double* relres, int64_t itmax) {
    for (int c = 0; c < kt; ++c) {
      const PanelCtl& ct = *h->h_ctl;
      const double bn = ct.bnorm[c];
      const double rr = bn > 0 ? std::sqrt(ct.resid[c] / bn) : 0.0;
      if (iters) iters[c0 + c] = ct.iters[c];
      if (relres) relres[c0 + c] = rr;
      h->stats.iterations += ct.iters[c];
      if (!(rr < h->opts.resid_gate)) {
        if (!any_fail) {
          char buf[256];
          snprintf(buf, sizeof buf,
                   "CUDA PCG solver residual %g exceeds tolerance %g for column %lld (%d iterations)",
                   rr, h->opts.resid_gate, (long long)(c0 + c + 1), ct.iters[c]);
          msg = buf;
        }
        any_fail = true;
      }
      // a column frozen by the stagnation guard above its tolerance is reported like one that ran into
      // itmax: results written, CS_B200_ERR_MAXITER, the true-residual gate decides (core.jl:639-641)
      if ((ct.iters[c] >= itmax || ct.stalled[c]) && std::sqrt(ct.rho[c]) > ct.tol[c]) any_maxit = true;
    }
  }

  // the call's return code: rc of a failed panel, else the residual gate, else the itmax stop
  int verdict(int rc) const {
    if (rc) return rc;
    if (any_fail) return set_err(h, CS_B200_ERR_RESIDUAL, "%s", msg.c_str());
    if (any_maxit) return set_err(h, CS_B200_ERR_MAXITER, "itmax reached (or the recurrence stagnated) before rtol");
    return CS_B200_OK;
  }
};

// the grid of the node-current kernels
template <int KT>
int cur_grid(cs_b200_handle* h) {
  return (int)std::min<int64_t>(h->grid_spmm, (h->n + (NT / KT) - 1) / (NT / KT));
}

// the branch-current maxima of the panel in X (ctl->maxpos / maxneg), the first pass of launch_currents
template <typename T, int KT>
void launch_cur_max(cs_b200_handle* h) {
  const int grid = cur_grid<KT>(h);
  if (h->A0.dia)
    k_cur_max_dia<T, KT><<<grid, NT, 0, h->stream>>>(dia_view<T>(h->A0), (const T*)h->X, h->d_ctl, h->d_partials);
  else
    k_cur_max<T, KT><<<grid, NT, 0, h->stream>>>((int)h->n, h->d_rowptr, h->d_colidx, (const T*)h->d_vals,
                                                 (const T*)h->X, h->d_ctl, h->d_partials);
  h->stats.kernel_launches++;
}

// node currents of the panel in X (src/out.jl:178-290): branch-current maxima, then max(inflow, outflow)
// per node with the 1e-8 zeroing, accumulated into the cumulative / max vectors (src/out.jl:100-107).
// fg: the finite-ground currents of each node join the sums (cs_b200_solve_advanced), or null.
template <typename T, int KT>
void launch_currents(cs_b200_handle* h, bool want_curr, int accumulate, const void* fg = nullptr) {
  const int grid = cur_grid<KT>(h);
  launch_cur_max<T, KT>(h);
  if (h->A0.dia) {
    const DiaDev<T> a = dia_view<T>(h->A0);
    k_cur_acc_dia<T, KT><<<grid, NT, 0, h->stream>>>(a, (const T*)h->X, (const T*)fg, h->d_ctl,
                                                     want_curr ? (T*)h->AP : nullptr,
                                                     (T*)h->d_cum, (T*)h->d_max, accumulate, h->opts.log_transform, KT);
  } else {
    k_cur_acc<T, KT><<<grid, NT, 0, h->stream>>>((int)h->n, h->d_rowptr, h->d_colidx, (const T*)h->d_vals,
                                                 (const T*)h->X, (const T*)fg, h->d_ctl,
                                                 want_curr ? (T*)h->AP : nullptr,
                                                 (T*)h->d_cum, (T*)h->d_max, accumulate, h->opts.log_transform, KT);
  }
  h->stats.kernel_launches++;
}

// ---- panel staging and downloads shared by the column kinds ------------------------------------
struct ColCtl {
  long long src, dst;
  double weight;
};

inline double col_weight(const double* weight, int64_t c) { return weight ? weight[c] : 1.0; }

// the panel's control block: zeroed, column c's src / dst / weight from col(c), uploaded
template <typename Col>
int upload_ctl(cs_b200_handle* h, int kt, Col&& col) {
  PanelCtl* hc = h->h_ctl;
  std::memset(hc, 0, sizeof(PanelCtl));
  for (int c = 0; c < kt; ++c) {
    const ColCtl v = col(c);
    hc->src[c] = v.src;
    hc->dst[c] = v.dst;
    hc->weight[c] = v.weight;
  }
  CK(h, cudaMemcpyAsync(h->d_ctl, hc, sizeof(PanelCtl), cudaMemcpyHostToDevice, h->stream));
  h->stats.h2d_bytes += sizeof(PanelCtl);
  return CS_B200_OK;
}

// host copy of the control block as the kernels after solve_panel left it
int read_ctl(cs_b200_handle* h) {
  CK(h, cudaMemcpyAsync(h->h_ctl, h->d_ctl, sizeof(PanelCtl), cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  h->stats.d2h_bytes += sizeof(PanelCtl);
  return CS_B200_OK;
}

// d_sp_*: the panel's sparse right-hand sides for k_sparse_rhs.  ptr: the kt+1 column offsets into
// rows / vals.  The capacity is recorded only once every buffer of the family is allocated.
int upload_sparse_rhs(cs_b200_handle* h, int kt, const int64_t* ptr, const int64_t* rows, const double* vals) {
  int ent_ptr[MAXKT + 1];
  for (int c = 0; c <= kt; ++c) ent_ptr[c] = (int)(ptr[c] - ptr[0]);
  const size_t nent = (size_t)ent_ptr[kt];
  if (!h->d_sp_ptr || nent > h->sp_cap) {
    cudaFree(h->d_sp_ptr); cudaFree(h->d_sp_rows); cudaFree(h->d_sp_vals);
    h->d_sp_ptr = nullptr; h->d_sp_rows = nullptr; h->d_sp_vals = nullptr;
    h->sp_cap = 0;
    const size_t cap = std::max<size_t>(nent, 1024);
    CK(h, cudaMalloc(&h->d_sp_ptr, (MAXKT + 1) * sizeof(int)));
    CK(h, cudaMalloc(&h->d_sp_rows, cap * sizeof(long long)));
    CK(h, cudaMalloc(&h->d_sp_vals, cap * sizeof(double)));
    h->sp_cap = cap;
  }
  CK(h, h2d(h, h->d_sp_ptr, ent_ptr, (kt + 1) * sizeof(int)));
  CK(h, h2d(h, h->d_sp_rows, rows + ptr[0], nent * sizeof(long long)));
  CK(h, h2d(h, h->d_sp_vals, vals + ptr[0], nent * sizeof(double)));
  h->stats.h2d_bytes += (kt + 1) * sizeof(int) + nent * 16.0;
  return CS_B200_OK;
}

// d_rg_*: the panel's Dirichlet sets as the 2*kt row segments of k_seg_set -- segment 2c the rows of set
// set_a[c], segment 2c+1 those of set_b[c] (empty without set_b, or where the set index is -1).  Growing the buffers drops the region
// graphs, which captured their addresses; the capacity is recorded once both buffers are allocated.
int upload_set_segments(cs_b200_handle* h, int kt, const int64_t* set_ptr, const int64_t* set_rows,
                        const int64_t* set_a, const int64_t* set_b) {
  int seg[2 * MAXKT + 1];
  std::vector<int> rows;
  seg[0] = 0;
  for (int s = 0; s < 2 * kt; ++s) {
    const int64_t* sets = (s & 1) ? set_b : set_a;
    if (sets && sets[s / 2] >= 0)
      for (int64_t e = set_ptr[sets[s / 2]]; e < set_ptr[sets[s / 2] + 1]; ++e) rows.push_back((int)set_rows[e]);
    seg[s + 1] = (int)rows.size();
  }
  if (!h->d_rg_seg || rows.size() > h->rg_cap) {
    CK(h, cudaStreamSynchronize(h->stream));
    drop_graphs(h->rgraphs);
    cudaFree(h->d_rg_seg); cudaFree(h->d_rg_rows);
    h->d_rg_seg = nullptr; h->d_rg_rows = nullptr;
    h->rg_cap = 0;
    const size_t cap = std::max<size_t>(rows.size(), 4096);
    CK(h, cudaMalloc(&h->d_rg_seg, (2 * MAXKT + 1) * sizeof(int)));
    CK(h, cudaMalloc(&h->d_rg_rows, cap * sizeof(int)));
    h->rg_cap = cap;
  }
  CK(h, h2d(h, h->d_rg_seg, seg, (2 * kt + 1) * sizeof(int)));
  CK(h, h2d(h, h->d_rg_rows, rows.data(), rows.size() * sizeof(int)));
  h->stats.h2d_bytes += (2.0 * kt + 1 + rows.size()) * sizeof(int);
  return CS_B200_OK;
}

// d_probe*: the probe rows of cs_b200_solve_sources and room for one panel of their voltages; the
// capacity is recorded once both buffers are allocated
int upload_probe(cs_b200_handle* h, int64_t nprobe, const int64_t* probe) {
  const size_t need = (size_t)nprobe;
  if (need > h->probe_cap) {
    cudaFree(h->d_probe); cudaFree(h->d_probe_out);
    h->d_probe = nullptr; h->d_probe_out = nullptr;
    h->probe_cap = 0;
    CK(h, cudaMalloc(&h->d_probe, need * sizeof(long long)));
    CK(h, cudaMalloc(&h->d_probe_out, need * MAXKT * sizeof(double)));
    h->probe_cap = need;
  }
  CK(h, h2d(h, h->d_probe, probe, need * sizeof(long long)));
  return CS_B200_OK;
}

// the panel's node currents (AP) and voltages (X; less each column's xsrc when volt_shift) into columns
// c0 .. c0+KT-1 of the caller's column-major arrays, through the staging buffer; either may be null.
// Checks the launches queued before it first.
template <typename T, int KT>
int download_outputs(cs_b200_handle* h, int64_t c0, T* curr, T* volt, int volt_shift) {
  CK(h, cudaGetLastError());
  const int tg = copy_grid((size_t)h->n_pad * KT);
  auto download = [&](const void* panel, int shift, T* out) -> int {
    k_panel_to_cm<T, KT><<<tg, 256, 0, h->stream>>>((int)h->n, (size_t)h->n, (const T*)panel, (T*)h->stage,
                                                    h->d_ctl, shift);
    h->stats.kernel_launches++;
    CK(h, cudaMemcpyAsync(out + (size_t)c0 * h->n, h->stage, (size_t)h->n * KT * sizeof(T),
                          cudaMemcpyDeviceToHost, h->stream));
    h->stats.d2h_bytes += (double)h->n * KT * sizeof(T);
    return CS_B200_OK;
  };
  if (curr)
    if (int rc = download(h->AP, 0, curr)) return rc;
  if (volt)
    if (int rc = download(h->X, volt_shift, volt)) return rc;
  return CS_B200_OK;
}

// the node currents of launch_currents (into AP for curr, into the maps when accumulating), then download_outputs
template <typename T, int KT>
int currents_and_outputs(cs_b200_handle* h, int64_t c0, T* curr, T* volt, int accumulate, int volt_shift,
                         const void* fg = nullptr) {
  if (accumulate || curr) launch_currents<T, KT>(h, curr != nullptr, accumulate, fg);
  return download_outputs<T, KT>(h, c0, curr, volt, volt_shift);
}

// ---- the column kinds ------------------------------------------------------------------------
// B of a pairs panel, -1 at src and +1 at dst (k_pair_rhs); under panel_ends B is not written and the panel's
// start pass and residual gate take b from ctl (pair_b, cleared by ColumnDriver::solve)
template <typename T, int KT>
int stage_pair_rhs(cs_b200_handle* h) {
  h->pair_b = panel_ends(h);
  if (h->pair_b) return CS_B200_OK;
  CK(h, cudaMemsetAsync(h->B, 0, (size_t)h->n_pad * KT * sizeof(T), h->stream));
  k_pair_rhs<T, KT><<<1, 32, 0, h->stream>>>((T*)h->B, h->d_ctl);
  h->stats.kernel_launches++;
  return CS_B200_OK;
}

template <typename T, int KT>
int pairs_panel(cs_b200_handle* h, int64_t c0, const int64_t* src, const int64_t* dst,
                const double* weight, double rtol, int64_t itmax, T* R, T* volt, T* curr,
                int accumulate, int64_t* iters, double* relres, ColumnDriver& cols) {
  if (int rc = upload_ctl(h, KT, [&](int c) {
        return ColCtl{src[c0 + c], dst[c0 + c], col_weight(weight, c0 + c)};
      }))
    return rc;
  if (int rc = stage_pair_rhs<T, KT>(h)) return rc;
  if (int rc = cols.solve<T, KT>(c0, rtol, itmax, iters, relres)) return rc;
  k_pair_extract<T, KT><<<1, 32, 0, h->stream>>>((const T*)h->X, h->d_ctl);
  h->stats.kernel_launches++;
  if (int rc = currents_and_outputs<T, KT>(h, c0, curr, volt, accumulate, 1)) return rc;
  if (int rc = read_ctl(h)) return rc;   // xsrc / xdst of k_pair_extract
  for (int c = 0; c < KT; ++c) R[c0 + c] = (T)(h->h_ctl->xdst[c] - h->h_ctl->xsrc[c]);
  return CS_B200_OK;
}

// panel of cs_b200_solve_sources: like pairs_panel, with the right-hand sides scattered from
// the caller's sparse columns and the shifted voltages of the probe rows as the small result
template <typename T, int KT>
int sources_panel(cs_b200_handle* h, int64_t c0, const int64_t* colptr, const int64_t* rows,
                  const double* vals, const int64_t* ref, const double* weight, double rtol,
                  int64_t itmax, int64_t nprobe, T* probe_volt, T* volt, T* curr, int accumulate,
                  int64_t* iters, double* relres, ColumnDriver& cols) {
  if (int rc = upload_ctl(h, KT, [&](int c) { return ColCtl{ref[c0 + c], -1, col_weight(weight, c0 + c)}; }))
    return rc;
  if (int rc = upload_sparse_rhs(h, KT, colptr + c0, rows, vals)) return rc;
  CK(h, cudaMemsetAsync(h->B, 0, (size_t)h->n_pad * KT * sizeof(T), h->stream));
  k_sparse_rhs<T, KT><<<1, 32, 0, h->stream>>>((T*)h->B, h->d_sp_ptr, h->d_sp_rows, h->d_sp_vals);
  h->stats.kernel_launches++;
  if (int rc = cols.solve<T, KT>(c0, rtol, itmax, iters, relres)) return rc;
  k_pair_extract<T, KT><<<1, 32, 0, h->stream>>>((const T*)h->X, h->d_ctl);
  h->stats.kernel_launches++;
  if (nprobe > 0 && probe_volt) {
    k_probe<T, KT><<<(int)std::min<int64_t>(64, (nprobe * KT + 255) / 256), 256, 0, h->stream>>>(
        (const T*)h->X, h->d_ctl, h->d_probe, (int)nprobe, (T*)h->d_probe_out);
    h->stats.kernel_launches++;
    CK(h, cudaMemcpyAsync(probe_volt + (size_t)c0 * nprobe, h->d_probe_out, (size_t)nprobe * KT * sizeof(T),
                          cudaMemcpyDeviceToHost, h->stream));
    h->stats.d2h_bytes += (double)nprobe * KT * sizeof(T);
  }
  if (int rc = currents_and_outputs<T, KT>(h, c0, curr, volt, accumulate, 1)) return rc;
  CK(h, cudaStreamSynchronize(h->stream));
  return CS_B200_OK;
}

// ---- superposition driver (cs_b200_solve_pairs_superposed) ----------------------------------
// panel of point solves  A u_x = e_{nodes[x]} - e_{nodes[0]}  for x = x0 .. x0+KT-1 (1-based among
// the focal nodes); the shifted solutions land in columns x0-1 .. of U (column-major, ld = n_pad)
template <typename T, int KT>
int point_panel(cs_b200_handle* h, int64_t x0, const int64_t* nodes, double rtol, int64_t itmax, T* U,
                int64_t* point_iters, ColumnDriver& cols) {
  const size_t nelem = (size_t)h->n_pad * KT;
  if (int rc = upload_ctl(h, KT, [&](int c) { return ColCtl{nodes[0], nodes[x0 + c], 1.0}; })) return rc;
  if (int rc = stage_pair_rhs<T, KT>(h)) return rc;
  if (int rc = cols.solve<T, KT>(0, rtol, itmax, nullptr, nullptr)) return rc;
  if (point_iters)
    for (int c = 0; c < KT; ++c) point_iters[x0 - 1 + c] = h->h_ctl->iters[c];
  k_pair_extract<T, KT><<<1, 32, 0, h->stream>>>((const T*)h->X, h->d_ctl);
  const int tg = copy_grid(nelem);
  k_panel_to_cm<T, KT><<<tg, 256, 0, h->stream>>>((int)h->n, (size_t)h->n_pad, (const T*)h->X,
                                                  U + (size_t)(x0 - 1) * h->n_pad, h->d_ctl, 1);
  h->stats.kernel_launches += 2;
  CK(h, cudaGetLastError());
  CK(h, cudaStreamSynchronize(h->stream));
  return CS_B200_OK;
}

// panel of pairs c0 .. c0+KT-1 formed from U; same outputs as pairs_panel
template <typename T, int KT>
int combine_panel(cs_b200_handle* h, int64_t c0, const int64_t* nodes, const int64_t* pi, const int64_t* pj,
                  const double* weight, const T* U, int* d_ci, int* d_cj, T* R, T* volt, T* curr,
                  int accumulate, double* relres, int64_t itmax, ColumnDriver& cols) {
  const size_t nelem = (size_t)h->n_pad * KT;
  if (int rc = upload_ctl(h, KT, [&](int c) {
        return ColCtl{nodes[pi[c0 + c]], nodes[pj[c0 + c]], col_weight(weight, c0 + c)};
      }))
    return rc;
  int ci[MAXKT], cj[MAXKT];
  for (int c = 0; c < KT; ++c) {
    ci[c] = (int)pi[c0 + c] - 1;      // point 0 is the reference: its solution is identically 0
    cj[c] = (int)pj[c0 + c] - 1;
  }
  CK(h, h2d(h, d_ci, ci, KT * sizeof(int)));
  CK(h, h2d(h, d_cj, cj, KT * sizeof(int)));
  h->stats.h2d_bytes += 2.0 * KT * sizeof(int);
  const int tg = copy_grid(nelem);
  k_combine<T, KT><<<tg, 256, 0, h->stream>>>((int)h->n, (size_t)h->n_pad, U, d_ci, d_cj, (T*)h->X);
  CK(h, cudaMemsetAsync(h->B, 0, nelem * sizeof(T), h->stream));
  k_pair_rhs<T, KT><<<1, 32, 0, h->stream>>>((T*)h->B, h->d_ctl);
  // the reference's gate on the combined voltage: AP = B - A X, ||AP|| / ||B||  (core.jl:640-641)
  launch_spmm<T, KT, SP_RESNORM>(h, (const T*)h->X, (T*)h->AP, (const T*)h->B);
  h->stats.kernel_launches += 2;
  CK(h, cudaGetLastError());
  if (int rc = read_ctl(h)) return rc;
  cols.gather(KT, c0, nullptr, relres, itmax);
  k_pair_extract<T, KT><<<1, 32, 0, h->stream>>>((const T*)h->X, h->d_ctl);
  h->stats.kernel_launches++;
  if (int rc = currents_and_outputs<T, KT>(h, c0, curr, volt, accumulate, 1)) return rc;
  if (int rc = read_ctl(h)) return rc;
  for (int c = 0; c < KT; ++c) R[c0 + c] = (T)(h->h_ctl->xdst[c] - h->h_ctl->xsrc[c]);
  return CS_B200_OK;
}

int ensure_io_pipeline(cs_b200_handle* h) {
  if (h->s_in) return CS_B200_OK;
  CK(h, cudaStreamCreateWithFlags(&h->s_in, cudaStreamNonBlocking));
  CK(h, cudaStreamCreateWithFlags(&h->s_out, cudaStreamNonBlocking));
  const size_t bytes = (size_t)h->n * h->ktmax * h->esize();
  for (int i = 0; i < 2; ++i) {
    CK(h, cudaMalloc(&h->io_in[i], bytes));
    CK(h, cudaMalloc(&h->io_out[i], bytes));
    CK(h, cudaEventCreateWithFlags(&h->ev_in[i], cudaEventDisableTiming));
    CK(h, cudaEventCreateWithFlags(&h->ev_used[i], cudaEventDisableTiming));
    CK(h, cudaEventCreateWithFlags(&h->ev_ready[i], cudaEventDisableTiming));
    CK(h, cudaEventCreateWithFlags(&h->ev_out[i], cudaEventDisableTiming));
  }
  return CS_B200_OK;
}

// upload of panel `ip` (columns c0 .. c0+kt) into its staging slot, on the upload stream;
// waits until the panel that used the slot two panels ago has been transposed out of it
template <typename T>
int rhs_upload(cs_b200_handle* h, int ip, int64_t c0, int kt, const T* rhs) {
  const int s = ip & 1;
  if (ip >= 2) CK(h, cudaStreamWaitEvent(h->s_in, h->ev_used[s], 0));
  CK(h, cudaMemcpyAsync(h->io_in[s], rhs + (size_t)c0 * h->n, (size_t)h->n * kt * sizeof(T),
                        cudaMemcpyHostToDevice, h->s_in));
  CK(h, cudaEventRecord(h->ev_in[s], h->s_in));
  h->stats.h2d_bytes += (double)h->n * kt * sizeof(T);
  return CS_B200_OK;
}

template <typename T, int KT>
int rhs_panel(cs_b200_handle* h, int ip, int64_t c0, T* lhs, double rtol, int64_t itmax,
              int64_t* iters, double* relres, ColumnDriver& cols) {
  const size_t nelem = (size_t)h->n_pad * KT;
  const int s = ip & 1;
  if (int rc = upload_ctl(h, KT, [](int) { return ColCtl{-1, -1, 0.0}; })) return rc;
  CK(h, cudaMemsetAsync(h->B, 0, nelem * sizeof(T), h->stream));
  const int tg = copy_grid(nelem);
  CK(h, cudaStreamWaitEvent(h->stream, h->ev_in[s], 0));
  k_cm_to_panel<T, KT><<<tg, 256, 0, h->stream>>>((int)h->n, (size_t)h->n, (const T*)h->io_in[s],
                                                  (T*)h->B, KT);
  CK(h, cudaEventRecord(h->ev_used[s], h->stream));
  h->stats.kernel_launches++;
  if (int rc = cols.solve<T, KT>(c0, rtol, itmax, iters, relres)) return rc;
  if (ip >= 2) CK(h, cudaStreamWaitEvent(h->stream, h->ev_out[s], 0));   // slot's last download done
  k_panel_to_cm<T, KT><<<tg, 256, 0, h->stream>>>((int)h->n, (size_t)h->n, (const T*)h->X,
                                                  (T*)h->io_out[s], h->d_ctl, 0);
  h->stats.kernel_launches++;
  CK(h, cudaEventRecord(h->ev_ready[s], h->stream));
  CK(h, cudaStreamWaitEvent(h->s_out, h->ev_ready[s], 0));
  CK(h, cudaMemcpyAsync(lhs + (size_t)c0 * h->n, h->io_out[s], (size_t)h->n * KT * sizeof(T),
                        cudaMemcpyDeviceToHost, h->s_out));
  CK(h, cudaEventRecord(h->ev_out[s], h->s_out));
  h->stats.d2h_bytes += (double)h->n * KT * sizeof(T);
  return CS_B200_OK;
}

// ---- focal-region pairs (cs_b200_solve_region_pairs) ----------------------------------------
// Column c: L w = 0 off the sets, w = 0 on set_a and set_b, right-hand side -L 1_b, so u = w + 1_b
// holds set_a at 0 V and set_b at 1 V.  flux = u.L u ; v = u / flux ; R = 1 / flux.
template <typename T, int KT>
int region_panel(cs_b200_handle* h, int64_t c0, const int64_t* set_ptr, const int64_t* set_rows,
                 const int64_t* set_a, const int64_t* set_b, const double* weight, double rtol,
                 int64_t itmax, T* R, T* volt, T* curr, int accumulate, int64_t* iters, double* relres,
                 ColumnDriver& cols) {
  const size_t nelem = (size_t)h->n_pad * KT;
  const int g = ew_grid<T, KT>(h);
  if (int rc = upload_ctl(h, KT, [&](int c) { return ColCtl{-1, -1, col_weight(weight, c0 + c)}; })) return rc;
  if (int rc = upload_set_segments(h, KT, set_ptr, set_rows, set_a + c0, set_b + c0)) return rc;
  // B = -L 1_b, zero on the sets (and on the pad rows, which the SpMM does not write)
  CK(h, cudaMemsetAsync(h->B, 0, nelem * sizeof(T), h->stream));
  CK(h, cudaMemsetAsync(h->X, 0, nelem * sizeof(T), h->stream));
  launch_seg_set<T, KT>(h, h->X, 1, T(-1));
  launch_spmm<T, KT, SP_PLAIN>(h, (const T*)h->X, (T*)h->B, nullptr);
  launch_seg_set<T, KT>(h, h->B, 0, T(0));
  if (int rc = cols.solve<T, KT>(c0, rtol, itmax, iters, relres, true)) return rc;
  // u = w + 1_b (w is zero on the sets); flux = u.L u, second order in the error of w
  launch_seg_set<T, KT>(h, h->X, 1, T(1));
  launch_spmm<T, KT, SP_PLAIN>(h, (const T*)h->X, (T*)h->AP, nullptr);
  k_flux<T, KT><<<g, NT, 0, h->stream>>>(nelem, (size_t)h->n * KT, (const T*)h->X, (const T*)h->AP, h->d_ctl, h->d_partials);
  h->stats.kernel_launches++;
  CK(h, cudaGetLastError());
  if (int rc = read_ctl(h)) return rc;
  for (int c = 0; c < KT; ++c) {
    const double flux = h->h_ctl->xdst[c];
    if (!(flux > 0.0))
      return set_err(h, CS_B200_ERR_ARG, "region pair %lld: flux into set_b is %g (no conducting path to set_a)",
                     (long long)(c0 + c), flux);
    R[c0 + c] = (T)(1.0 / flux);
  }
  k_scale_flux<T, KT><<<g, NT, 0, h->stream>>>(nelem, (T*)h->X, h->d_ctl);
  h->stats.kernel_launches++;
  if (accumulate || curr) {
    launch_currents<T, KT>(h, true, 0);
    k_seg_current<T, KT><<<2 * KT, NT, 0, h->stream>>>((T*)h->AP, h->d_rg_seg, h->d_rg_rows);
    h->stats.kernel_launches++;
    if (accumulate) {
      const int ag = (int)std::max<int64_t>(1, std::min<int64_t>(h->grid_ew, (h->n + NT - 1) / NT));
      k_cur_accum<T, KT><<<ag, NT, 0, h->stream>>>((int)h->n, (const T*)h->AP, h->d_ctl, (T*)h->d_cum,
                                                   (T*)h->d_max, h->opts.log_transform);
      h->stats.kernel_launches++;
    }
  }
  if (int rc = download_outputs<T, KT>(h, c0, curr, volt, 0)) return rc;
  CK(h, cudaStreamSynchronize(h->stream));
  return CS_B200_OK;
}

// ---- direct-ground columns (cs_b200_solve_grounded, cs_b200_solve_advanced) -------------------
// Column c: the rows of its ground set are Dirichlet rows at 0 V (segment 2c of the region-panel table,
// empty for gset[c] = -1; segment 2c+1, the region panels' set_b, is empty), b = its sparse sources,
// masked; A_c v = b.  No flux or scaling step, and no set fix-up of the currents: every ground row is a
// node of its own.  fg: the handle's finite grounds when their currents join the node currents, or null.
template <typename T, int KT>
int grounded_panel(cs_b200_handle* h, int64_t c0, const int64_t* set_ptr, const int64_t* set_rows,
                   const int64_t* gset, const int64_t* src_ptr, const int64_t* src_rows, const double* src_vals,
                   const double* weight, double rtol, int64_t itmax, T* src_volt, T* volt, T* curr,
                   int accumulate, int64_t* iters, double* relres, ColumnDriver& cols, const void* fg) {
  // k_pair_extract probes the first source row
  if (int rc = upload_ctl(h, KT, [&](int c) {
        return ColCtl{-1, src_rows[src_ptr[c0 + c]], col_weight(weight, c0 + c)};
      }))
    return rc;
  if (int rc = upload_set_segments(h, KT, set_ptr, set_rows, gset + c0, nullptr)) return rc;
  if (int rc = upload_sparse_rhs(h, KT, src_ptr + c0, src_rows, src_vals)) return rc;
  // B = sum of the sources, zero on the ground rows (the entry point rejects a source there) and pad rows
  CK(h, cudaMemsetAsync(h->B, 0, (size_t)h->n_pad * KT * sizeof(T), h->stream));
  k_sparse_rhs<T, KT><<<1, 32, 0, h->stream>>>((T*)h->B, h->d_sp_ptr, h->d_sp_rows, h->d_sp_vals);
  h->stats.kernel_launches++;
  launch_seg_set<T, KT>(h, h->B, 0, T(0));
  if (int rc = cols.solve<T, KT>(c0, rtol, itmax, iters, relres, true)) return rc;
  k_pair_extract<T, KT><<<1, 32, 0, h->stream>>>((const T*)h->X, h->d_ctl);
  h->stats.kernel_launches++;
  if (int rc = currents_and_outputs<T, KT>(h, c0, curr, volt, accumulate, 0, fg)) return rc;
  if (int rc = read_ctl(h)) return rc;
  if (src_volt)
    for (int c = 0; c < KT; ++c) src_volt[c0 + c] = (T)h->h_ctl->xdst[c];
  return CS_B200_OK;
}

// ---- branch currents (cs_b200_branch_index, cs_b200_solve_pairs_branch, cs_b200_solve_advanced_network) --
// device scratch of one call, freed on every return path
struct DevScratch {
  void* p = nullptr;
  DevScratch() = default;
  DevScratch(const DevScratch&) = delete;
  DevScratch& operator=(const DevScratch&) = delete;
  ~DevScratch() { cudaFree(p); }
};

// d_bptr and nb, on first use (the CSR's pattern never changes after create); a row whose columns do not
// ascend is CS_B200_ERR_ARG
int ensure_branch_index(cs_b200_handle* h) {
  if (h->d_bptr) return CS_B200_OK;
  const int n = (int)h->n;
  const int g = (int)std::min<int64_t>((h->n + 255) / 256, (int64_t)h->num_sms * 32);
  DevScratch bptr, cnt, bad, tmp;
  CK(h, cudaMalloc(&bptr.p, ((size_t)n + 1) * sizeof(int)));
  CK(h, cudaMalloc(&cnt.p, std::max(1, n) * sizeof(int)));
  CK(h, cudaMalloc(&bad.p, sizeof(int)));
  const int none = INT32_MAX;
  CK(h, h2d(h, bad.p, &none, sizeof(int)));
  k_branch_count<<<g, 256, 0, h->stream>>>(n, h->d_rowptr, h->d_colidx, (int*)cnt.p, (int*)bad.p);
  size_t tb = 0;
  CK(h, cub::DeviceScan::InclusiveSum(nullptr, tb, (const int*)cnt.p, (int*)bptr.p + 1, n, h->stream));
  CK(h, cudaMalloc(&tmp.p, std::max<size_t>(tb, 1)));
  CK(h, cub::DeviceScan::InclusiveSum(tmp.p, tb, (const int*)cnt.p, (int*)bptr.p + 1, n, h->stream));
  CK(h, cudaMemsetAsync(bptr.p, 0, sizeof(int), h->stream));
  CK(h, cudaGetLastError());
  int bad_row = none, nb = 0;
  CK(h, cudaMemcpyAsync(&bad_row, bad.p, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaMemcpyAsync(&nb, (int*)bptr.p + n, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  h->stats.kernel_launches += 3;
  if (bad_row != none)
    return set_err(h, CS_B200_ERR_ARG, "row %d: column indices do not ascend (branch currents need sorted rows)",
                   bad_row);
  h->d_bptr = (int*)bptr.p;
  bptr.p = nullptr;
  h->nb = nb;
  return CS_B200_OK;
}

// d_cum_branch, zeroed, on first use
int ensure_cum_branch(cs_b200_handle* h) {
  if (h->d_cum_branch) return CS_B200_OK;
  const size_t bytes = (size_t)std::max<int64_t>(h->nb, 1) * h->esize();
  CK(h, cudaMalloc(&h->d_cum_branch, bytes));
  CK(h, cudaMemsetAsync(h->d_cum_branch, 0, bytes, h->stream));
  return CS_B200_OK;
}

// the branch pass of the panel in X, after k_cur_max left its maxima in ctl: the branch currents into
// columns c0 .. c0+KT-1 of the caller's column-major nb x k `branch` (or null), and with `accumulate`
// weighted by ctl->weight into d_cum_branch.  Needs ensure_branch_index.
template <typename T, int KT>
int branch_pass(cs_b200_handle* h, int64_t c0, T* branch, int accumulate, int ncols) {
  if ((!branch && !accumulate) || h->nb == 0) return CS_B200_OK;
  if (branch && !h->d_branch_stage) CK(h, cudaMalloc(&h->d_branch_stage, (size_t)h->nb * h->ktmax * sizeof(T)));
  if (accumulate)
    if (int rc = ensure_cum_branch(h)) return rc;
  const int grid = (int)std::min<int64_t>((int64_t)h->num_sms * 16, (h->n + NT - 1) / NT);
  k_branch_cur<T, KT><<<grid, NT, 0, h->stream>>>((int)h->n, h->d_rowptr, h->d_colidx, (const T*)h->d_vals,
                                                  h->d_bptr, (const T*)h->X, h->d_ctl,
                                                  branch ? (T*)h->d_branch_stage : nullptr, (size_t)h->nb,
                                                  accumulate ? (T*)h->d_cum_branch : nullptr, ncols);
  h->stats.kernel_launches++;
  CK(h, cudaGetLastError());
  if (branch) {
    CK(h, cudaMemcpyAsync(branch + (size_t)c0 * h->nb, h->d_branch_stage, (size_t)h->nb * KT * sizeof(T),
                          cudaMemcpyDeviceToHost, h->stream));
    h->stats.d2h_bytes += (double)h->nb * KT * sizeof(T);
  }
  CK(h, cudaStreamSynchronize(h->stream));
  return CS_B200_OK;
}

// cs_b200_solve_advanced_network: every column on grounded_panel, each column's voltages added into vsum
// on the rows it owns, then one node-current and branch pass over vsum as a KT = 1 panel
template <typename T>
int advanced_network_t(cs_b200_handle* h, const int64_t* set_ptr, const int64_t* set_rows, int64_t k,
                       const int64_t* gset, const int64_t* src_ptr, const int64_t* src_rows, const double* src_vals,
                       const int64_t* owner, double rtol, int64_t itmax, T* volt, T* curr, T* branch,
                       int64_t* iters, double* relres, ColumnDriver& cols) {
  if (branch)
    if (int rc = ensure_branch_index(h)) return rc;
  const size_t np = (size_t)h->n_pad;
  DevScratch vsum, own;
  CK(h, cudaMalloc(&vsum.p, np * sizeof(T)));
  CK(h, cudaMalloc(&own.p, (size_t)h->n * sizeof(long long)));
  CK(h, cudaMemsetAsync(vsum.p, 0, np * sizeof(T), h->stream));
  CK(h, h2d(h, own.p, owner, (size_t)h->n * sizeof(long long)));
  const int g = (int)std::min<int64_t>((h->n + 255) / 256, (int64_t)h->num_sms * 32);
  const int rc = cols.run(0, k, [&](auto kt, int64_t c0) -> int {
    if (int rc = grounded_panel<T, kt>(h, c0, set_ptr, set_rows, gset, src_ptr, src_rows, src_vals, nullptr, rtol,
                                       itmax, (T*)nullptr, (T*)nullptr, (T*)nullptr, 0, iters, relres, cols, h->d_fg))
      return rc;
    k_owner_sum<T, kt><<<g, 256, 0, h->stream>>>((int)h->n, (const T*)h->X, (const long long*)own.p, c0,
                                                 (T*)vsum.p);
    h->stats.kernel_launches++;
    return CS_B200_OK;
  });
  if (rc) return rc;
  // the whole graph's voltages as one column: one 1e-8 cut over the graph for node and branch currents
  CK(h, cudaMemcpyAsync(h->X, vsum.p, np * sizeof(T), cudaMemcpyDeviceToDevice, h->stream));
  if (int rc = upload_ctl(h, 1, [](int) { return ColCtl{-1, -1, 1.0}; })) return rc;
  if (curr)
    launch_currents<T, 1>(h, true, 0, h->d_fg);
  else if (branch)
    launch_cur_max<T, 1>(h);
  if (int rc = download_outputs<T, 1>(h, 0, curr, volt, 0)) return rc;
  if (int rc = branch_pass<T, 1>(h, 0, branch, 0, 1)) return rc;
  CK(h, cudaStreamSynchronize(h->stream));
  return CS_B200_OK;
}

template <typename T>
int solve_pairs_superposed_t(cs_b200_handle* h, int64_t np, const int64_t* nodes, int64_t k,
                             const int64_t* pi, const int64_t* pj, const double* weight, double rtol,
                             int64_t itmax, T* R, T* volt, T* curr, int accumulate,
                             int64_t* point_iters, double* relres, ColumnDriver& cols) {
  T* U = nullptr;
  int *d_ci = nullptr, *d_cj = nullptr;
  const size_t ubytes = (size_t)h->n_pad * (size_t)(np - 1) * sizeof(T);
  auto cleanup = [&]() { cudaFree(U); cudaFree(d_ci); cudaFree(d_cj); };
  cudaError_t e = cudaMalloc(&U, ubytes);
  if (e == cudaSuccess) e = cudaMalloc(&d_ci, MAXKT * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&d_cj, MAXKT * sizeof(int));
  if (e == cudaSuccess) e = cudaMemsetAsync(U, 0, ubytes, h->stream);
  if (e != cudaSuccess) {
    cleanup();
    return set_err(h, CS_B200_ERR_CUDA, "CUDA error %s allocating %zu bytes for the point solutions",
                   cudaGetErrorString(e), ubytes);
  }
  int rc = cols.run(1, np, [&](auto kt, int64_t x0) {
    return point_panel<T, kt>(h, x0, nodes, rtol, itmax, U, point_iters, cols);
  });
  if (!rc)
    rc = cols.run(0, k, [&](auto kt, int64_t c0) {
      return combine_panel<T, kt>(h, c0, nodes, pi, pj, weight, U, d_ci, d_cj, R, volt, curr, accumulate, relres,
                                  itmax, cols);
    });
  cudaStreamSynchronize(h->stream);
  cleanup();
  return rc;
}

template <typename T>
int solve_rhs_t(cs_b200_handle* h, int64_t k, const T* rhs, T* lhs, double rtol, int64_t itmax,
                int64_t* iters, double* relres, ColumnDriver& cols) {
  int rc = ensure_io_pipeline(h);
  if (rc) return rc;
  // the upload stream must not overtake work of an earlier call that still reads the slots
  CK(h, cudaEventRecord(h->ev_used[0], h->stream));
  CK(h, cudaStreamWaitEvent(h->s_in, h->ev_used[0], 0));
  int ip = 0;
  rc = rhs_upload<T>(h, 0, 0, next_kt(k, h->ktmax), rhs);
  if (!rc)
    rc = cols.run(0, k, [&](auto kt, int64_t c0) {
      const int64_t c1 = c0 + kt;
      if (c1 < k)   // next panel's upload overlaps this panel's solve
        if (int urc = rhs_upload<T>(h, ip + 1, c1, next_kt(k - c1, h->ktmax), rhs)) return urc;
      return rhs_panel<T, kt>(h, ip++, c0, lhs, rtol, itmax, iters, relres, cols);
    });
  // drain both copy streams whatever happened: the caller owns rhs/lhs again on return
  cudaStreamSynchronize(h->s_in);
  cudaStreamSynchronize(h->s_out);
  cudaStreamSynchronize(h->stream);
  return rc;
}

void begin_call(cs_b200_handle* h) {
  cudaSetDevice(h->device);
  h->err.clear();
  const double setup = h->stats.setup_ms;
  h->stats = cs_b200_stats{};
  h->stats.setup_ms = setup;
  cudaEventRecord(h->ev0, h->stream);
}
void end_call(cs_b200_handle* h) {
  cudaEventRecord(h->ev1, h->stream);
  cudaEventSynchronize(h->ev1);
  float ms = 0;
  cudaEventElapsedTime(&ms, h->ev0, h->ev1);
  h->stats.solve_ms = ms;
}

// a batched solve entry's call: solve(T{}, cols) in the handle's element type T, then the verdict of the
// column driver, between begin_call and end_call
template <typename Solve>
int solve_call(cs_b200_handle* h, Solve&& solve) {
  if (!h) return set_err(h, CS_B200_ERR_ARG, "null handle");
  begin_call(h);
  ColumnDriver cols{h};
  const int rc = cols.verdict(with_type(h, [&](auto t) { return solve(t, cols); }));
  end_call(h);
  return rc;
}

int ensure_flush(cs_b200_handle* h) {
  if (h->d_flush) return 0;
  h->flush_elems = (size_t)64 << 20;  // 256 MB of floats > 50 MB L2
  CK(h, cudaMalloc(&h->d_flush, h->flush_elems * sizeof(float)));
  CK(h, cudaMemsetAsync(h->d_flush, 0, h->flush_elems * sizeof(float), h->stream));
  return 0;
}

}  // namespace

// the text cs_b200_last_error(NULL) returns, for handle-less entry points in other translation units
int set_handleless_error(int code, const char* msg) {
  g_create_error = msg;
  return code;
}

// ---------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------
namespace {
template <typename T>
int assemble_raster(cs_b200_handle* h, int64_t nrows, int64_t ncols, const T* g_host, int four, int avg_res) {
  const int64_t ncell = nrows * ncols;
  T* d_g = nullptr;
  int *d_valid = nullptr, *d_nodeid = nullptr, *d_rowcnt = nullptr;
  auto cleanup = [&]() { cudaFree(d_g); cudaFree(d_valid); cudaFree(d_nodeid); cudaFree(d_rowcnt); };
#define CKR(call)                                                                          \
  do {                                                                                     \
    cudaError_t _e = (call);                                                               \
    if (_e != cudaSuccess) {                                                               \
      cleanup();                                                                           \
      return set_err(h, CS_B200_ERR_CUDA, "CUDA error %s at %s:%d (%s)",                   \
                     cudaGetErrorString(_e), __FILE__, __LINE__, #call);                   \
    }                                                                                      \
  } while (0)
  CKR(cudaMalloc(&d_g, (size_t)ncell * sizeof(T)));
  CKR(cudaMalloc(&d_valid, (size_t)ncell * sizeof(int)));
  CKR(cudaMalloc(&d_nodeid, (size_t)ncell * sizeof(int)));
  CKR(h2d(h, d_g, g_host, (size_t)ncell * sizeof(T)));
  const int grid = (int)std::min<int64_t>((ncell + 255) / 256, (int64_t)h->num_sms * 32);
  ras::k_valid<T><<<grid, 256, 0, h->stream>>>(ncell, d_g, d_valid);
  CKR(cudaGetLastError());
  CKR(ras::exclusive_scan(d_valid, d_nodeid, ncell, h->stream));
  int last_id = 0, last_valid = 0;
  CKR(cudaMemcpy(&last_id, d_nodeid + (ncell - 1), sizeof(int), cudaMemcpyDeviceToHost));
  CKR(cudaMemcpy(&last_valid, d_valid + (ncell - 1), sizeof(int), cudaMemcpyDeviceToHost));
  const int64_t n = (int64_t)last_id + last_valid;
  if (n <= 0) { cleanup(); return set_err(h, CS_B200_ERR_ARG, "raster has no cell with conductance > 0"); }
  CKR(cudaMalloc(&d_rowcnt, (size_t)(n + 1) * sizeof(int)));
  CKR(cudaMemsetAsync(d_rowcnt, 0, (size_t)(n + 1) * sizeof(int), h->stream));
  ras::k_count<<<grid, 256, 0, h->stream>>>((int)nrows, (int)ncols, four, d_valid, d_nodeid, d_rowcnt);
  CKR(cudaGetLastError());
  CKR(cudaMalloc(&h->d_rowptr, (size_t)(n + 1) * sizeof(int)));
  CKR(ras::exclusive_scan(d_rowcnt, h->d_rowptr, n + 1, h->stream));
  int nnz = 0;
  CKR(cudaMemcpy(&nnz, h->d_rowptr + n, sizeof(int), cudaMemcpyDeviceToHost));
  if (nnz <= 0) { cleanup(); return set_err(h, CS_B200_ERR_ARG, "assembled matrix is empty"); }
  CKR(cudaMalloc(&h->d_colidx, (size_t)nnz * sizeof(int)));
  CKR(cudaMalloc(&h->d_vals, (size_t)nnz * sizeof(T)));
  ras::k_fill<T><<<grid, 256, 0, h->stream>>>((int)nrows, (int)ncols, four, avg_res, d_g, d_valid, d_nodeid,
                                              h->d_rowptr, h->d_colidx, (T*)h->d_vals);
  CKR(cudaGetLastError());
  CKR(cudaStreamSynchronize(h->stream));
#undef CKR
  cleanup();
  h->n = n;
  h->nnz = nnz;
  return CS_B200_OK;
}

// A caller's host CSR onto the handle (h->n rows, h->nnz entries of the handle's dtype): the index arrays go up
// as they are and are narrowed to int32 0-based on the device, whatever their width and base.  With no rowptr
// the arrays are only allocated (the ranks that receive the matrix by broadcast).
int upload_host_csr(cs_b200_handle* h, const void* rowptr, const void* colidx, const void* vals, int index_bits,
                    int index_base) {
  const int64_t n = h->n, nnz = h->nnz;
  CK(h, cudaMalloc(&h->d_rowptr, (size_t)(n + 1) * sizeof(int)));
  CK(h, cudaMalloc(&h->d_colidx, std::max<size_t>(1, (size_t)nnz) * sizeof(int)));
  CK(h, cudaMalloc(&h->d_vals, std::max<size_t>(1, (size_t)nnz) * h->esize()));
  if (!rowptr) return CS_B200_OK;
  if (index_bits == 32 && index_base == 0) {
    CK(h, cudaMemcpyAsync(h->d_rowptr, rowptr, (size_t)(n + 1) * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CK(h, cudaMemcpyAsync(h->d_colidx, colidx, (size_t)nnz * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  } else {
    const size_t ib = index_bits / 8;
    void* raw = nullptr;
    CK(h, cudaMalloc(&raw, std::max<size_t>((size_t)(n + 1), (size_t)nnz) * ib));
    cudaError_t e = cudaMemcpyAsync(raw, rowptr, (size_t)(n + 1) * ib, cudaMemcpyHostToDevice, h->stream);
    if (e == cudaSuccess) e = (cudaError_t)csb_dev::narrow_indices(h->stream, raw, index_bits, index_base, n + 1, h->d_rowptr);
    if (e == cudaSuccess) e = cudaMemcpyAsync(raw, colidx, (size_t)nnz * ib, cudaMemcpyHostToDevice, h->stream);
    if (e == cudaSuccess) e = (cudaError_t)csb_dev::narrow_indices(h->stream, raw, index_bits, index_base, nnz, h->d_colidx);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    cudaFree(raw);
    CK(h, e);
  }
  CK(h, cudaMemcpyAsync(h->d_vals, vals, (size_t)nnz * h->esize(), cudaMemcpyHostToDevice, h->stream));
  return CS_B200_OK;
}

// Level-0 aggregation seeds for the device builder, wanted under device setup with AMG and n > 200.  `job` runs
// the seed pass on a helper thread from the caller's host pattern; `dev` holds seeds an operator source left
// on the device instead (n + 1 ints, the last the aggregate count).
struct Seeds {
  bool wanted = false;
  csb_dev::SeedJob* job = nullptr;   // the create sequence's: a source may wait on it, never free it
  int* d_seed = nullptr;             // freed by the create sequence
  csb_dev::DeviceSeed dev;
};

// The one create sequence behind every cs_b200_create* entry: a handle of n rows and nnz entries (0, 0 when the
// source assembles the operator), the seed pass started before the operator arrives so that it hides behind the
// upload, the operator from `source(h, seeds)` (it leaves d_rowptr / d_colidx / d_vals, n, nnz and owns_matrix
// on the handle), then one of the two builders (opts.setup: 1 host, else device).  A failure's text goes to
// cs_b200_last_error(NULL) and, if given, to *err_copy; the handle is destroyed.
template <class Source>
int create_handle(int64_t n, int64_t nnz, int dtype, int device, const cs_b200_opts* opts,
                  const csb_dev::HostPattern& hp, std::string* err_copy, cs_b200_handle** out, Source&& source) {
  cs_b200_handle* h = new cs_b200_handle();
  h->n = n; h->nnz = nnz; h->dtype = dtype; h->device = device;
  Seeds seeds;
  auto finish = [&](int rc) {
    csb_dev::seed_discard(seeds.job);
    cudaFree(seeds.d_seed);
    if (rc == CS_B200_OK) {
      cudaEventRecord(h->ev1, h->stream);
      cudaEventSynchronize(h->ev1);
      float ms = 0;
      cudaEventElapsedTime(&ms, h->ev0, h->ev1);
      h->stats.setup_ms = ms;
      *out = h;
      return rc;
    }
    g_create_error = h->err;
    if (err_copy) *err_copy = h->err;
    cs_b200_destroy(h);
    return rc;
  };
  int rc = common_create(h, opts);
  if (rc) return finish(rc);
  cudaEventRecord(h->ev0, h->stream);
  const bool device_setup = h->opts.setup != 1;
  seeds.wanted = device_setup && h->opts.precond == CS_B200_PRECOND_AMG && n > 200;
  if (seeds.wanted && hp.rowptr) seeds.job = csb_dev::seed_start(n, hp);
  Tick up_tick;
  rc = source(h, seeds);
  if (rc) return finish(rc);
  if (up_tick.on) { cudaStreamSynchronize(h->stream); up_tick("operator on the device"); }
  h->n_pad = (h->n + 3) / 4 * 4;
  const bool f64 = dtype == CS_B200_F64;
  if (device_setup) {
    const csb_dev::DeviceSeed* dseed = seeds.d_seed ? &seeds.dev : nullptr;
    return finish(f64 ? finish_setup_device<double>(h, hp, seeds.job, dseed)
                      : finish_setup_device<float>(h, hp, seeds.job, dseed));
  }
  std::vector<int> rp((size_t)h->n + 1);
  cudaError_t e = cudaMemcpyAsync(rp.data(), h->d_rowptr, rp.size() * sizeof(int), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  if (e != cudaSuccess) return finish(set_err(h, CS_B200_ERR_CUDA, "CUDA error %s reading rowptr", cudaGetErrorString(e)));
  return finish(f64 ? finish_setup<double>(h, rp) : finish_setup<float>(h, rp));
}

}  // namespace

namespace {
template <typename T>
__global__ void k_apply_grounds(int n, const int* __restrict__ rowptr, const int* __restrict__ colidx,
                                T* __restrict__ vals, const T* __restrict__ g, const unsigned char* __restrict__ mask) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const bool mi = mask && mask[i];
    for (int j = rowptr[i]; j < rowptr[i + 1]; ++j) {
      const int c = colidx[j];
      if (mi) vals[j] = c == i ? T(1) : T(0);
      else if (mask && mask[c]) vals[j] = T(0);
      else if (c == i && g) vals[j] += g[i];
    }
  }
}
}  // namespace

// everything derived from the operator's VALUES: captured graphs (they hold level pointers), the
// finest operator's stencil / window records, the multigrid levels.  The CSR, the plain row blocks
// and the panels stay.
static void teardown_operators(cs_b200_handle* h) {
  if (h->stream) cudaStreamSynchronize(h->stream);
  drop_graphs(h->graphs);
  drop_graphs(h->rgraphs);
  free_win(h->A0);
  h->A0.has_dinv = 0; h->A0.win_blocks = 0; h->A0.win_nblocks = 0; h->A0.dia_nr = 0; h->A0.dia_ld = 0;
  for (size_t l = 0; l < h->lv.size(); ++l) {
    DevLevel& L = h->lv[l];
    if (l > 0) {
      free_csr(L.A);
      cudaFree(L.dinv); cudaFree(L.x); cudaFree(L.b); cudaFree(L.t); cudaFree(L.y);
    }
    free_csr(L.P);
    free_csr(L.R);
  }
  for (size_t l = 0; l < h->lv32.size(); ++l) {
    DevLevel& L = h->lv32[l];
    free_csr(L.A);
    cudaFree(L.dinv); cudaFree(L.x); cudaFree(L.b); cudaFree(L.t); cudaFree(L.y);
    free_csr(L.P);
    free_csr(L.R);
  }
  h->lv.clear();
  h->lv32.clear();
  cudaFree(h->R32); cudaFree(h->X32); cudaFree(h->T32); cudaFree(h->Z32);
  h->R32 = h->X32 = h->T32 = h->Z32 = nullptr;
  cudaFree(h->Z); h->Z = nullptr;
  cudaFree(h->d_pinv); h->d_pinv = nullptr;
  h->amg = false;
  h->mixed = false;
}

// Z = M^-1 R with the cycle solve_panel launches for its first z (k_set_ctl first, so the last kernel
// runs cg_after_precond's init branch and leaves |r.z| in ctl->rho0).  r, z: host column-major n x KT.
template <typename T, int KT>
int apply_precond_t(cs_b200_handle* h, const void* r, void* z, double* rz) {
  const size_t bytes = (size_t)h->n * KT * sizeof(T);
  const size_t nelem = (size_t)h->n_pad * KT;
  const int tg = copy_grid(nelem);
  const int g = ew_grid<T, KT>(h);
  CK(h, cudaMemcpyAsync(h->stage, r, bytes, cudaMemcpyHostToDevice, h->stream));
  CK(h, cudaMemsetAsync(h->R, 0, nelem * sizeof(T), h->stream));
  k_cm_to_panel<T, KT><<<tg, 256, 0, h->stream>>>((int)h->n, (size_t)h->n, (const T*)h->stage, (T*)h->R, KT);
  k_set_ctl<<<1, 1, 0, h->stream>>>(h->d_ctl, 0.0, 0.0, 1, 40);
  if (h->mixed) k_convert<T, float><<<g, NT, 0, h->stream>>>(nelem, (const T*)h->R, (float*)h->R32);
  launch_vcycle<T, KT>(h, false);   // the fp64 cycle uses h->stage as its finest x: staging is done by now
  if (h->mixed) k_convert<float, T><<<g, NT, 0, h->stream>>>(nelem, (const float*)h->Z32, (T*)h->X);
  k_panel_to_cm<T, KT><<<tg, 256, 0, h->stream>>>((int)h->n, (size_t)h->n, (const T*)(h->mixed ? h->X : h->Z),
                                                  (T*)h->stage, h->d_ctl, 0);
  CK(h, cudaGetLastError());
  CK(h, cudaMemcpyAsync(z, h->stage, bytes, cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaMemcpyAsync(h->h_ctl, h->d_ctl, sizeof(PanelCtl), cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  if (rz)
    for (int c = 0; c < KT; ++c) rz[c] = h->h_ctl->rho0[c];
  return CS_B200_OK;
}


// cs_b200_plan_advanced's stream-ordered scratch, released (after the stream) on every return
struct PoolScratch {
  cudaStream_t s;
  std::vector<void*> p;
  explicit PoolScratch(cudaStream_t s_) : s(s_) {}
  template <typename X>
  cudaError_t get(X** out, size_t count) {
    void* q = nullptr;
    cudaError_t e = cudaMallocAsync(&q, std::max<size_t>(count * sizeof(X), 1), s);
    if (e == cudaSuccess) p.push_back(q);
    *out = (X*)q;
    return e;
  }
  ~PoolScratch() { for (void* q : p) cudaFreeAsync(q, s); cudaStreamSynchronize(s); }
};

static int nbits_for(unsigned v) { int b = 1; while (b < 32 && (v >> b)) ++b; return b; }

// the plan's arrays inside d_plan (see cs_b200_handle)
struct PlanView {
  long long *col_comp, *set_ptr, *set_rows, *src_ptr, *src_rows;
  double* src_vals;
  int* col_of_row;
  size_t bytes;
  PlanView(void* base, int64_t ncol, int64_t nset, int64_t nsrc, int64_t n) {
    long long* q = (long long*)base;
    col_comp = q; q += ncol;
    set_ptr = q; q += ncol + 1;
    set_rows = q; q += nset;
    src_ptr = q; q += ncol + 1;
    src_rows = q; q += nsrc;
    src_vals = (double*)q; q += nsrc;
    col_of_row = (int*)q;
    bytes = (size_t)((char*)(col_of_row + n) - (char*)base);
  }
};

extern "C" {

int cs_b200_version(void) { return 1008; }

const char* cs_b200_last_error(const cs_b200_handle* h) {
  return h ? h->err.c_str() : g_create_error.c_str();
}

int cs_b200_create(int64_t n, int64_t nnz, const void* rowptr, const void* colidx,
                   const void* vals, int index_bits, int index_base, int dtype, int device,
                   const cs_b200_opts* opts, cs_b200_handle** out) {
  if (!out) return set_err(nullptr, CS_B200_ERR_ARG, "out is NULL");
  *out = nullptr;
  if (n <= 0 || nnz < 0 || !rowptr || (nnz > 0 && (!colidx || !vals)))
    return set_err(nullptr, CS_B200_ERR_ARG, "bad matrix arguments (n=%lld nnz=%lld)",
                   (long long)n, (long long)nnz);
  if ((index_bits != 32 && index_bits != 64) || (index_base != 0 && index_base != 1) ||
      (dtype != CS_B200_F32 && dtype != CS_B200_F64))
    return set_err(nullptr, CS_B200_ERR_ARG, "bad index_bits/index_base/dtype");
  if (nnz >= (int64_t)1 << 31 || n >= (int64_t)1 << 31)
    return set_err(nullptr, CS_B200_ERR_UNSUPPORTED,
                   "n and nnz must be < 2^31 (device indices are int32)");
  // the raw values, before any narrowing: the seed pass and the device read rowptr[0 .. n] as the bounds of colidx
  const int64_t first = index_bits == 64 ? ((const int64_t*)rowptr)[0] : (int64_t)((const int32_t*)rowptr)[0];
  const int64_t last = index_bits == 64 ? ((const int64_t*)rowptr)[n] : (int64_t)((const int32_t*)rowptr)[n];
  if (first - index_base != 0 || last - index_base != nnz)
    return set_err(nullptr, CS_B200_ERR_ARG, "rowptr does not span [0, nnz] (got %lld..%lld)",
                   (long long)(first - index_base), (long long)(last - index_base));
  const csb_dev::HostPattern hp{rowptr, colidx, index_bits, index_base};
  return create_handle(n, nnz, dtype, device, opts, hp, nullptr, out, [&](cs_b200_handle* h, Seeds&) -> int {
    return upload_host_csr(h, rowptr, colidx, vals, index_bits, index_base);
  });
}

int cs_b200_create_from_device(int64_t n, int64_t nnz, const int32_t* d_rowptr,
                               const int32_t* d_colidx, const void* d_vals, int dtype, int device,
                               const cs_b200_opts* opts, cs_b200_handle** out) {
  if (!out) return set_err(nullptr, CS_B200_ERR_ARG, "out is NULL");
  *out = nullptr;
  if (n <= 0 || nnz <= 0 || !d_rowptr || !d_colidx || !d_vals ||
      (dtype != CS_B200_F32 && dtype != CS_B200_F64) || nnz >= (int64_t)1 << 31)
    return set_err(nullptr, CS_B200_ERR_ARG, "bad arguments");
  return create_handle(n, nnz, dtype, device, opts, {}, nullptr, out, [&](cs_b200_handle* h, Seeds&) -> int {
    h->owns_matrix = false;
    h->d_rowptr = const_cast<int*>(d_rowptr);
    h->d_colidx = const_cast<int*>(d_colidx);
    h->d_vals = const_cast<void*>(d_vals);
    return CS_B200_OK;
  });
}

int cs_b200_create_from_raster(int64_t nrows, int64_t ncols, const void* g, int dtype,
                               int four_neighbors, int avg_res, int device,
                               const cs_b200_opts* opts, cs_b200_handle** out,
                               int64_t* n_out, int64_t* nnz_out) {
  if (!out) return set_err(nullptr, CS_B200_ERR_ARG, "out is NULL");
  *out = nullptr;
  if (nrows <= 0 || ncols <= 0 || !g || (dtype != CS_B200_F32 && dtype != CS_B200_F64) ||
      nrows > (int64_t)1 << 30 || ncols > (int64_t)1 << 30)
    return set_err(nullptr, CS_B200_ERR_ARG, "bad arguments");
  if (nrows * ncols * 9 >= (int64_t)1 << 31)
    return set_err(nullptr, CS_B200_ERR_UNSUPPORTED, "raster too large: 9 * cells must be < 2^31 (device indices are int32)");
  return create_handle(0, 0, dtype, device, opts, {}, nullptr, out, [&](cs_b200_handle* h, Seeds&) -> int {
    const int four = four_neighbors ? 1 : 0, avg = avg_res ? 1 : 0;
    const int rc = dtype == CS_B200_F64 ? assemble_raster<double>(h, nrows, ncols, (const double*)g, four, avg)
                                        : assemble_raster<float>(h, nrows, ncols, (const float*)g, four, avg);
    if (rc) return rc;
    if (n_out) *n_out = h->n;
    if (nnz_out) *nnz_out = h->nnz;
    return CS_B200_OK;
  });
}

int cs_b200_create_from_raster_poly(int64_t nrows, int64_t ncols, const void* g, const int32_t* polymap,
                                    int dtype, int four_neighbors, int avg_res, int device,
                                    const cs_b200_opts* opts, cs_b200_handle** out, int64_t* n_out,
                                    int64_t* nnz_out, int32_t* nodemap_out) {
  if (!out) return set_err(nullptr, CS_B200_ERR_ARG, "out is NULL");
  *out = nullptr;
  if (nrows <= 0 || ncols <= 0 || !g || (dtype != CS_B200_F32 && dtype != CS_B200_F64) ||
      nrows > (int64_t)1 << 30 || ncols > (int64_t)1 << 30)
    return set_err(nullptr, CS_B200_ERR_ARG, "bad arguments");
  if (nrows * ncols * 17 >= (int64_t)1 << 31)
    return set_err(nullptr, CS_B200_ERR_UNSUPPORTED, "raster too large: 17 * cells must be < 2^31 (device indices are int32)");
  const int64_t ncell = nrows * ncols;
  int max_poly = 0;
  if (polymap) {
    for (int64_t i = 0; i < ncell; ++i) {
      if (polymap[i] < 0) return set_err(nullptr, CS_B200_ERR_ARG, "polygon ids must be >= 0 (cell %lld holds %d)", (long long)i, polymap[i]);
      max_poly = std::max(max_poly, (int)polymap[i]);
    }
    if (max_poly > (1 << 27)) return set_err(nullptr, CS_B200_ERR_UNSUPPORTED, "polygon ids above 2^27 are not supported");
  }
  return create_handle(0, 0, dtype, device, opts, {}, nullptr, out, [&](cs_b200_handle* h, Seeds&) -> int {
    double* d_g = nullptr;
    int* d_poly = nullptr;
    int* d_node = nullptr;
    void* d_raw = nullptr;
    csb_dev::DCsr L;
    auto cleanup = [&](int rc) { cudaFree(d_g); cudaFree(d_poly); cudaFree(d_node); cudaFree(d_raw); return rc; };
    cudaError_t e = cudaMalloc(&d_g, (size_t)ncell * sizeof(double));
    if (e == cudaSuccess && dtype == CS_B200_F64) e = h2d(h, d_g, g, (size_t)ncell * sizeof(double));
    if (e == cudaSuccess && dtype == CS_B200_F32) {
      e = cudaMalloc(&d_raw, (size_t)ncell * sizeof(float));
      if (e == cudaSuccess) e = h2d(h, d_raw, g, (size_t)ncell * sizeof(float));
      if (e == cudaSuccess) e = (cudaError_t)csb_dev::convert_values(h->stream, (const float*)d_raw, d_g, ncell);
    }
    if (e == cudaSuccess && polymap) {
      e = cudaMalloc(&d_poly, (size_t)ncell * sizeof(int));
      if (e == cudaSuccess) e = h2d(h, d_poly, polymap, (size_t)ncell * sizeof(int));
    }
    if (e != cudaSuccess) return cleanup(set_err(h, CS_B200_ERR_CUDA, "CUDA error %s (raster upload)", cudaGetErrorString(e)));
    int rc = csb_dev::assemble_raster_polygons(h->stream, nrows, ncols, d_g, d_poly, max_poly, four_neighbors ? 1 : 0,
                                               avg_res ? 1 : 0, L, &d_node, h->err);
    if (rc) return cleanup(rc == -1 ? CS_B200_ERR_ARG : rc_dev(h, rc));
    h->n = L.nrows;
    h->nnz = L.nnz;
    h->d_rowptr = L.ptr;
    h->d_colidx = L.idx;
    if (dtype == CS_B200_F64) {
      h->d_vals = L.val;
    } else {
      e = cudaMalloc(&h->d_vals, std::max<size_t>(1, (size_t)L.nnz) * sizeof(float));
      if (e == cudaSuccess) e = (cudaError_t)csb_dev::convert_values(h->stream, L.val, (float*)h->d_vals, L.nnz);
      if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
      cudaFree(L.val);
      if (e != cudaSuccess) return cleanup(set_err(h, CS_B200_ERR_CUDA, "CUDA error %s (value conversion)", cudaGetErrorString(e)));
    }
    if (nodemap_out) {
      e = cudaMemcpyAsync(nodemap_out, d_node, (size_t)ncell * sizeof(int), cudaMemcpyDeviceToHost, h->stream);
      if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
      if (e != cudaSuccess) return cleanup(set_err(h, CS_B200_ERR_CUDA, "CUDA error %s (node map download)", cudaGetErrorString(e)));
    }
    if (n_out) *n_out = h->n;
    if (nnz_out) *nnz_out = h->nnz;
    return cleanup(CS_B200_OK);
  });
}

int cs_b200_get_csr(cs_b200_handle* h, int32_t* rowptr, int32_t* colidx, void* vals) {
  if (!h) return CS_B200_ERR_ARG;
  cudaSetDevice(h->device);
  CK(h, cudaStreamSynchronize(h->stream));
  if (rowptr) CK(h, cudaMemcpy(rowptr, h->d_rowptr, (size_t)(h->n + 1) * sizeof(int), cudaMemcpyDeviceToHost));
  if (colidx) CK(h, cudaMemcpy(colidx, h->d_colidx, (size_t)h->nnz * sizeof(int), cudaMemcpyDeviceToHost));
  if (vals) CK(h, cudaMemcpy(vals, h->d_vals, (size_t)h->nnz * h->esize(), cudaMemcpyDeviceToHost));
  return CS_B200_OK;
}

static const DevCsr* pick_level(cs_b200_handle* h, int level, int which, bool* is_f32, double* omega,
                                int64_t* ncols) {
  if (!h || level < 0 || which < 0 || which > 2) return nullptr;
  std::vector<DevLevel>& lv = h->mixed ? h->lv32 : h->lv;
  if (lv.empty() && level == 0 && which == 0) {   // no hierarchy (Jacobi): the handle's own operator
    *is_f32 = h->dtype == CS_B200_F32;
    *omega = 0.0;
    *ncols = h->n;
    return &h->A0;
  }
  if (level >= (int)lv.size()) return nullptr;
  if (which > 0 && level + 1 >= (int)lv.size()) return nullptr;
  *is_f32 = h->mixed || h->dtype == CS_B200_F32;
  *omega = lv[level].omega;
  const DevCsr* m = which == 0 ? &lv[level].A : which == 1 ? &lv[level].P : &lv[level].R;
  *ncols = which == 0 ? lv[level].n : which == 1 ? lv[level + 1].n : lv[level].n;
  if (which == 2) *ncols = lv[level].n;
  return m;
}

int cs_b200_level_info(cs_b200_handle* h, int level, int which, int64_t* nrows, int64_t* ncols,
                       int64_t* nnz, double* omega, int* windowed) {
  bool f32 = false;
  double om = 0.0;
  int64_t nc = 0;
  const DevCsr* m = pick_level(h, level, which, &f32, &om, &nc);
  if (!m) return CS_B200_ERR_ARG;
  if (nrows) *nrows = m->nrows;
  if (ncols) *ncols = nc;
  if (nnz) *nnz = m->nnz;
  if (omega) *omega = om;
  if (windowed) *windowed = m->dia ? 2 : (m->win_meta ? 1 : 0);   // 2 = stencil (DIA) form
  return CS_B200_OK;
}

int cs_b200_level_stencil(cs_b200_handle* h, int level, int* slots) {
  bool f32 = false;
  double om = 0.0;
  int64_t nc = 0;
  const DevCsr* m = pick_level(h, level, 0, &f32, &om, &nc);
  if (!m || !slots) return CS_B200_ERR_ARG;
  *slots = !m->dia ? 0 : m->dia_half ? 5 : 9;
  return CS_B200_OK;
}

int cs_b200_level_csr(cs_b200_handle* h, int level, int which, int32_t* rowptr, int32_t* colidx,
                      double* vals) {
  bool f32 = false;
  double om = 0.0;
  int64_t nc = 0;
  const DevCsr* m = pick_level(h, level, which, &f32, &om, &nc);
  if (!m) return CS_B200_ERR_ARG;
  cudaSetDevice(h->device);
  CK(h, cudaStreamSynchronize(h->stream));
  if (rowptr) CK(h, cudaMemcpy(rowptr, m->rowptr, (size_t)(m->nrows + 1) * sizeof(int), cudaMemcpyDeviceToHost));
  if (colidx) CK(h, cudaMemcpy(colidx, m->colidx, (size_t)m->nnz * sizeof(int), cudaMemcpyDeviceToHost));
  if (vals) {
    if (f32) {
      std::vector<float> tmp((size_t)m->nnz);
      CK(h, cudaMemcpy(tmp.data(), m->vals, (size_t)m->nnz * sizeof(float), cudaMemcpyDeviceToHost));
      for (int64_t i = 0; i < m->nnz; ++i) vals[i] = (double)tmp[i];
    } else {
      CK(h, cudaMemcpy(vals, m->vals, (size_t)m->nnz * sizeof(double), cudaMemcpyDeviceToHost));
    }
  }
  return CS_B200_OK;
}

// Whether the handle can take cs_b200_set_grounds (error text set when not).
static int grounds_supported(cs_b200_handle* h) {
  if (h->opts.setup == 1)
    return set_err(h, CS_B200_ERR_UNSUPPORTED, "cs_b200_set_grounds needs the device-side setup (opts.setup != 1)");
  if (!h->owns_matrix)
    return set_err(h, CS_B200_ERR_UNSUPPORTED, "cs_b200_set_grounds: the handle borrows its matrix (create_from_device)");
  return CS_B200_OK;
}

// cs_b200_set_grounds once its arguments are on the device: the pristine values restored, d_g (n values of the
// handle's type, or null) added to the diagonal and kept as the handle's finite grounds, the rows of d_m (n
// bytes, or null) tied to ground, then 1/diag, the stencil / window records and the hierarchy rebuilt.  Takes
// over d_g and d_m (cudaMalloc'ed).  setup_ms runs from ev0, which the caller records.
static int apply_grounds(cs_b200_handle* h, void* d_g, unsigned char* d_m) {
  const size_t vb = std::max<size_t>(1, (size_t)h->nnz) * h->esize();
  auto cleanup = [&]() { cudaFree(d_g); cudaFree(d_m); };
  cudaFree(h->d_fg);                 // the previous call's finite grounds; this call's replace them
  h->d_fg = nullptr;
  cudaError_t e0 = cudaSuccess;
  if (!h->d_vals0) {
    e0 = cudaMalloc(&h->d_vals0, vb);
    if (e0 == cudaSuccess) e0 = cudaMemcpyAsync(h->d_vals0, h->d_vals, vb, cudaMemcpyDeviceToDevice, h->stream);
  } else {
    e0 = cudaMemcpyAsync(h->d_vals, h->d_vals0, vb, cudaMemcpyDeviceToDevice, h->stream);
  }
  if (e0 != cudaSuccess) { cleanup(); return set_err(h, CS_B200_ERR_CUDA, "CUDA error %s (pristine values)", cudaGetErrorString(e0)); }
  if (d_g || d_m) {
    const int g = (int)std::min<int64_t>((h->n + 255) / 256, (int64_t)h->num_sms * 32);
    with_type(h, [&](auto t) {
      using T = decltype(t);
      k_apply_grounds<T><<<g, 256, 0, h->stream>>>((int)h->n, h->d_rowptr, h->d_colidx, (T*)h->d_vals, (const T*)d_g, d_m);
    });
  }
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  if (e == cudaSuccess) {            // kept for the ground currents of cs_b200_solve_advanced
    h->d_fg = d_g;
    d_g = nullptr;
  }
  cleanup();
  if (e != cudaSuccess) return set_err(h, CS_B200_ERR_CUDA, "CUDA error %s applying the grounds", cudaGetErrorString(e));
  teardown_operators(h);
  csb_dev::SeedJob* no_job = nullptr;
  if (int rc = with_type(h, [&](auto t) { return build_operators<decltype(t)>(h, {}, no_job, nullptr); })) return rc;
  cudaEventRecord(h->ev1, h->stream);
  cudaEventSynchronize(h->ev1);
  float ms = 0;
  cudaEventElapsedTime(&ms, h->ev0, h->ev1);
  h->stats.setup_ms = ms;
  return CS_B200_OK;
}

int cs_b200_set_grounds(cs_b200_handle* h, const void* finite_g, const uint8_t* dirichlet) {
  if (!h) return CS_B200_ERR_ARG;
  if (int rc = grounds_supported(h)) return rc;
  cudaSetDevice(h->device);
  h->err.clear();
  const size_t es = h->esize();
  cudaEventRecord(h->ev0, h->stream);
  void* d_g = nullptr;
  unsigned char* d_m = nullptr;
  auto cleanup = [&]() { cudaFree(d_g); cudaFree(d_m); };
  if (finite_g) {
    cudaError_t e = cudaMalloc(&d_g, (size_t)h->n * es);
    if (e == cudaSuccess) e = h2d(h, d_g, finite_g, (size_t)h->n * es);
    if (e != cudaSuccess) { cleanup(); return set_err(h, CS_B200_ERR_CUDA, "CUDA error %s (finite grounds)", cudaGetErrorString(e)); }
  }
  if (dirichlet) {
    cudaError_t e = cudaMalloc(&d_m, (size_t)h->n);
    if (e == cudaSuccess) e = h2d(h, d_m, dirichlet, (size_t)h->n);
    if (e != cudaSuccess) { cleanup(); return set_err(h, CS_B200_ERR_CUDA, "CUDA error %s (Dirichlet mask)", cudaGetErrorString(e)); }
  }
  return apply_grounds(h, d_g, d_m);
}

int cs_b200_get_dims(const cs_b200_handle* h, int64_t* n, int64_t* nnz) {
  if (!h) return CS_B200_ERR_ARG;
  if (n) *n = h->n;
  if (nnz) *nnz = h->nnz;
  return CS_B200_OK;
}

void cs_b200_destroy(cs_b200_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  teardown_operators(h);
  if (h->owns_matrix) { cudaFree(h->d_rowptr); cudaFree(h->d_colidx); cudaFree(h->d_vals); }
  cudaFree(h->d_vals0);
  cudaFree(h->d_fg);
  cudaFree(h->d_plan);
  cudaFree(h->d_bptr); cudaFree(h->d_cum_branch); cudaFree(h->d_branch_stage);
  void* bufs[] = {h->d_dinv, h->d_bstart, h->X, h->R, h->R2, h->P, h->P2, h->AP, h->B, h->stage,
                  h->d_cum, h->d_max, h->d_ctl, h->d_partials, h->d_flush};
  for (void* b : bufs) if (b) cudaFree(b);
  if (h->h_ctl) cudaFreeHost(h->h_ctl);
  cudaFree(h->d_sp_rows); cudaFree(h->d_sp_vals); cudaFree(h->d_sp_ptr);
  cudaFree(h->d_probe); cudaFree(h->d_probe_out);
  cudaFree(h->d_rg_seg); cudaFree(h->d_rg_rows);
  for (int i = 0; i < 2; ++i) {
    cudaFree(h->io_in[i]); cudaFree(h->io_out[i]);
    cudaEvent_t evs[] = {h->ev_in[i], h->ev_used[i], h->ev_ready[i], h->ev_out[i]};
    for (cudaEvent_t e : evs) if (e) cudaEventDestroy(e);
  }
  if (h->s_in) cudaStreamDestroy(h->s_in);
  if (h->s_out) cudaStreamDestroy(h->s_out);
  for (cudaEvent_t e : h->prof_ev) cudaEventDestroy(e);
  if (h->ev0) cudaEventDestroy(h->ev0);
  if (h->ev1) cudaEventDestroy(h->ev1);
  if (h->ev2) cudaEventDestroy(h->ev2);
  if (h->ev3) cudaEventDestroy(h->ev3);
  if (h->stream) cudaStreamDestroy(h->stream);
  delete h;
}

int cs_b200_reset_currents(cs_b200_handle* h) {
  if (!h) return CS_B200_ERR_ARG;
  cudaSetDevice(h->device);
  CK(h, cudaMemsetAsync(h->d_cum, 0, (size_t)h->n_pad * h->esize(), h->stream));
  const int g = (int)std::min<int64_t>(4096, (h->n_pad + 255) / 256);
  with_type(h, [&](auto t) {
    using T = decltype(t);
    k_fill<T><<<g, 256, 0, h->stream>>>((T*)h->d_max, (size_t)h->n_pad, T(-9999));
  });
  if (h->d_cum_branch)
    CK(h, cudaMemsetAsync(h->d_cum_branch, 0, (size_t)std::max<int64_t>(h->nb, 1) * h->esize(), h->stream));
  CK(h, cudaGetLastError());
  CK(h, cudaStreamSynchronize(h->stream));
  return CS_B200_OK;
}

int cs_b200_read_currents(cs_b200_handle* h, void* cum, void* max) {
  if (!h) return CS_B200_ERR_ARG;
  cudaSetDevice(h->device);
  if (cum) CK(h, cudaMemcpyAsync(cum, h->d_cum, (size_t)h->n * h->esize(), cudaMemcpyDeviceToHost, h->stream));
  if (max) CK(h, cudaMemcpyAsync(max, h->d_max, (size_t)h->n * h->esize(), cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  return CS_B200_OK;
}

int cs_b200_read_branch_currents(cs_b200_handle* h, void* cum_branch) {
  if (!h || !cum_branch) return set_err(h, CS_B200_ERR_ARG, "bad read_branch_currents arguments");
  cudaSetDevice(h->device);
  if (int rc = ensure_branch_index(h)) return rc;
  const size_t bytes = (size_t)h->nb * h->esize();
  if (h->d_cum_branch)
    CK(h, cudaMemcpyAsync(cum_branch, h->d_cum_branch, bytes, cudaMemcpyDeviceToHost, h->stream));
  else
    std::memset(cum_branch, 0, bytes);   // no call has accumulated branch currents yet
  CK(h, cudaStreamSynchronize(h->stream));
  return CS_B200_OK;
}

int cs_b200_branch_index(cs_b200_handle* h, int64_t* nb, int64_t* lo, int64_t* hi) {
  if (!h || !nb) return set_err(h, CS_B200_ERR_ARG, "bad branch_index arguments");
  cudaSetDevice(h->device);
  if (int rc = ensure_branch_index(h)) return rc;
  *nb = h->nb;
  if ((!lo && !hi) || h->nb == 0) return CS_B200_OK;
  DevScratch ends;
  CK(h, cudaMalloc(&ends.p, (size_t)h->nb * 2 * sizeof(long long)));
  long long* d_lo = (long long*)ends.p;
  long long* d_hi = d_lo + h->nb;
  const int g = (int)std::min<int64_t>((h->n + 255) / 256, (int64_t)h->num_sms * 32);
  k_branch_ends<<<g, 256, 0, h->stream>>>((int)h->n, h->d_rowptr, h->d_colidx, h->d_bptr, d_lo, d_hi);
  CK(h, cudaGetLastError());
  if (lo) CK(h, cudaMemcpyAsync(lo, d_lo, (size_t)h->nb * sizeof(int64_t), cudaMemcpyDeviceToHost, h->stream));
  if (hi) CK(h, cudaMemcpyAsync(hi, d_hi, (size_t)h->nb * sizeof(int64_t), cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  return CS_B200_OK;
}

// The labels of cs_b200_components on the device: ncomp, and with `out` non-null each row's label in out (n int32
// on the device; the stream is synchronised on return).
static int label_components(cs_b200_handle* h, int64_t* ncomp, int* out) {
  const int n = (int)h->n;
  *ncomp = 0;
  if (n == 0) return CS_B200_OK;
  // scratch from the stream-ordered pool, released before return: parent, root flags, their exclusive scan,
  // each row's root, then its label (n each, the last one in `out` when given) and cub's temporary storage
  size_t tb = 0;
  CK(h, cub::DeviceScan::ExclusiveSum(nullptr, tb, (const int*)nullptr, (int*)nullptr, n, h->stream));
  const size_t ib = (size_t)n * sizeof(int), ia = (ib + 255) & ~(size_t)255;
  const size_t off_root = ia, off_idx = 2 * ia, off_lab = 3 * ia, off_tmp = 4 * ia;
  char* s = nullptr;
  CK(h, cudaMallocAsync((void**)&s, off_tmp + std::max<size_t>(tb, 1), h->stream));
  int* parent = (int*)s;
  int* root = (int*)(s + off_root);
  int* idx = (int*)(s + off_idx);
  int* lab = out ? out : (int*)(s + off_lab);
  const int g = (int)std::min<int64_t>((h->n + 255) / 256, (int64_t)h->num_sms * 32);
  constexpr int CHUNK = 16;
  const int ge = (int)std::max<int64_t>(1, std::min<int64_t>((h->nnz / CHUNK + 255) / 256, (int64_t)h->num_sms * 32));
  const void* vals = h->d_vals0 ? h->d_vals0 : h->d_vals;    // pristine values: grounds do not split
  k_cc_init<<<g, 256, 0, h->stream>>>(n, parent);
  with_type(h, [&](auto t) {
    using T = decltype(t);
    k_cc_hook<T><<<ge, 256, 0, h->stream>>>(n, (int)h->nnz, h->d_rowptr, h->d_colidx, (const T*)vals, parent, CHUNK);
  });
  k_cc_compress<<<g, 256, 0, h->stream>>>(n, parent, lab, root);
  cudaError_t e = cub::DeviceScan::ExclusiveSum(s + off_tmp, tb, root, idx, n, h->stream);
  int total = 0, last_flag = 0;
  if (e == cudaSuccess) {
    if (out) k_cc_label<<<g, 256, 0, h->stream>>>(n, lab, idx);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpyAsync(&total, idx + n - 1, sizeof(int), cudaMemcpyDeviceToHost, h->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(&last_flag, root + n - 1, sizeof(int), cudaMemcpyDeviceToHost, h->stream);
  cudaFreeAsync(s, h->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
  if (e != cudaSuccess) return set_err(h, CS_B200_ERR_CUDA, "CUDA error %s (components)", cudaGetErrorString(e));
  h->stats.kernel_launches += out ? 5 : 4;
  *ncomp = (int64_t)total + last_flag;
  return CS_B200_OK;
}

int cs_b200_components(cs_b200_handle* h, int64_t* ncomp, int32_t* comp_of) {
  if (!h || !ncomp) return set_err(h, CS_B200_ERR_ARG, "bad components arguments");
  cudaSetDevice(h->device);
  h->err.clear();
  *ncomp = 0;
  if (h->n == 0) return CS_B200_OK;
  int* lab = nullptr;
  if (comp_of) CK(h, cudaMallocAsync((void**)&lab, (size_t)h->n * sizeof(int), h->stream));
  int rc = label_components(h, ncomp, lab);
  if (rc == CS_B200_OK && comp_of) {
    cudaError_t e = cudaMemcpyAsync(comp_of, lab, (size_t)h->n * sizeof(int), cudaMemcpyDeviceToHost, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (e != cudaSuccess) rc = set_err(h, CS_B200_ERR_CUDA, "CUDA error %s (components)", cudaGetErrorString(e));
  }
  if (lab) { cudaFreeAsync(lab, h->stream); cudaStreamSynchronize(h->stream); }
  return rc;
}

int cs_b200_plan_advanced(cs_b200_handle* h, int64_t nrows, int64_t ncols, const int32_t* nodemap,
                          const void* src, const void* gnd, int dtype, int policy,
                          int64_t* ncol, int64_t* nsolved, int64_t* nset_rows, int64_t* nsrc_rows,
                          int* finite_applied) {
  if (!h) return CS_B200_ERR_ARG;
  if (!nodemap || !src || !gnd || !ncol || !nsolved || !nset_rows || !nsrc_rows || !finite_applied)
    return set_err(h, CS_B200_ERR_ARG, "cs_b200_plan_advanced: a NULL argument");
  if (dtype != CS_B200_F32 && dtype != CS_B200_F64)
    return set_err(h, CS_B200_ERR_ARG, "cs_b200_plan_advanced: bad dtype %d", dtype);
  if (policy < 0 || policy > 3)
    return set_err(h, CS_B200_ERR_ARG, "cs_b200_plan_advanced: bad policy %d (0 keepall ... 3 rmvall)", policy);
  // at most 2^30 cells: every index, grid-stride step and launch size below stays inside int32
  if (nrows <= 0 || ncols <= 0 || nrows > (int64_t(1) << 30) / ncols)
    return set_err(h, CS_B200_ERR_ARG, "cs_b200_plan_advanced: a %lld x %lld raster does not fit (2^30 cells at most)",
                   (long long)nrows, (long long)ncols);
  cudaSetDevice(h->device);
  h->err.clear();
  cudaFree(h->d_plan);                // a second plan replaces the first
  h->d_plan = nullptr;
  h->plan_ncol = h->plan_nset = h->plan_nsrc = 0;
  const int ncell = (int)(nrows * ncols), n = (int)h->n;
  const size_t ms = dtype == CS_B200_F64 ? 8 : 4;
  cudaStream_t st = h->stream;
  const int g = (int)std::min<int64_t>((std::max(ncell, n) + 255) / 256, (int64_t)h->num_sms * 32);
  PoolScratch sc(st);
  int *d_nm, *cnt, *ptr, *val, *val2, *flags;
  unsigned *key, *key2;
  void *d_src, *d_gnd;
  double *s, *gv;
  CK(h, sc.get(&d_nm, ncell));
  CK(h, sc.get((char**)&d_src, ncell * ms));
  CK(h, sc.get((char**)&d_gnd, ncell * ms));
  CK(h, sc.get(&key, ncell)); CK(h, sc.get(&key2, ncell));
  CK(h, sc.get(&val, ncell)); CK(h, sc.get(&val2, ncell));
  CK(h, sc.get(&cnt, (size_t)n + 1)); CK(h, sc.get(&ptr, (size_t)n + 1));
  CK(h, sc.get(&s, n)); CK(h, sc.get(&gv, n));
  CK(h, sc.get(&flags, 2));
  void* d_f = nullptr;               // the finite grounds: the handle keeps them when they are applied
  CK(h, cudaMalloc(&d_f, std::max<size_t>((size_t)n, 1) * h->esize()));
  struct FreeF { void*& p; ~FreeF() { cudaFree(p); } } free_f{d_f};
  CK(h, cudaMemcpyAsync(d_nm, nodemap, (size_t)ncell * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(h, cudaMemcpyAsync(d_src, src, (size_t)ncell * ms, cudaMemcpyHostToDevice, st));
  CK(h, cudaMemcpyAsync(d_gnd, gnd, (size_t)ncell * ms, cudaMemcpyHostToDevice, st));
  CK(h, cudaMemsetAsync(cnt, 0, ((size_t)n + 1) * sizeof(int), st));
  CK(h, cudaMemsetAsync(flags, 0, 2 * sizeof(int), st));
  // expand: every cell keyed by its node in row-major order; stable radix sort: each node's cells in np.add.at's
  // order; compress: the node's range from the exclusive scan of the cell counts
  k_adv_cells<<<g, 256, 0, st>>>(ncell, (int)nrows, (int)ncols, n, d_nm, key, val, cnt, flags);
  CK(h, cudaGetLastError());
  const int kb = nbits_for((unsigned)n);
  size_t tb = 0, tb2 = 0;
  CK(h, cub::DeviceRadixSort::SortPairs(nullptr, tb, key, key2, val, val2, ncell, 0, kb, st));
  CK(h, cub::DeviceScan::ExclusiveSum(nullptr, tb2, cnt, ptr, n + 1, st));
  char* tmp;
  CK(h, sc.get(&tmp, std::max(tb, tb2)));
  CK(h, cub::DeviceRadixSort::SortPairs(tmp, tb, key, key2, val, val2, ncell, 0, kb, st));
  CK(h, cub::DeviceScan::ExclusiveSum(tmp, tb2, cnt, ptr, n + 1, st));
  with_type(h, [&](auto t) {
    using T = decltype(t);
    if (dtype == CS_B200_F64)
      k_adv_node_values<double, T><<<g, 256, 0, st>>>(n, (int)nrows, (int)ncols, ptr, val2, (const double*)d_src,
                                                      (const double*)d_gnd, policy, s, gv, (T*)d_f, flags);
    else
      k_adv_node_values<float, T><<<g, 256, 0, st>>>(n, (int)nrows, (int)ncols, ptr, val2, (const float*)d_src,
                                                     (const float*)d_gnd, policy, s, gv, (T*)d_f, flags);
  });
  CK(h, cudaGetLastError());
  int hf[2] = {0, 0};
  CK(h, cudaMemcpyAsync(hf, flags, sizeof hf, cudaMemcpyDeviceToHost, st));
  CK(h, cudaStreamSynchronize(st));
  h->stats.kernel_launches += 2;
  if (hf[0] & 1) return set_err(h, CS_B200_ERR_ARG, "cs_b200_plan_advanced: a node map entry outside [0, %d]", n);
  if (hf[0] & 2) return set_err(h, CS_B200_ERR_ARG, "cs_b200_plan_advanced: a node of the handle has no cell");
  if (hf[1])                         // finite grounds to apply: the handle must take them before any plan is kept
    if (int rc = grounds_supported(h)) return rc;
  // components of the pristine operator; each component's rows ascending (stable sort of 0 ... n-1 by label)
  int64_t nc64 = 0;
  int *lab, *lab2, *rows, *ccnt, *cptr;
  CK(h, sc.get(&lab, n)); CK(h, sc.get(&lab2, n)); CK(h, sc.get(&rows, n));
  if (int rc = label_components(h, &nc64, lab)) return rc;
  const int ncomp = (int)nc64;
  CK(h, sc.get(&ccnt, (size_t)ncomp + 1)); CK(h, sc.get(&cptr, (size_t)ncomp + 1));
  CK(h, cudaMemsetAsync(ccnt, 0, ((size_t)ncomp + 1) * sizeof(int), st));
  k_adv_rows<<<g, 256, 0, st>>>(n, lab, key, val, ccnt);
  CK(h, cudaGetLastError());
  const int lb = nbits_for((unsigned)ncomp);
  size_t tb4 = 0;
  CK(h, cub::DeviceRadixSort::SortPairs(nullptr, tb4, key, key2, val, rows, n, 0, lb, st));
  char* tmp4;
  CK(h, sc.get(&tmp4, tb4));
  CK(h, cub::DeviceRadixSort::SortPairs(tmp4, tb4, key, key2, val, rows, n, 0, lb, st));
  CK(h, cub::DeviceScan::ExclusiveSum(tmp, tb2, ccnt, cptr, ncomp + 1, st));
  // the nonzero terms of each component's two sums, compacted in position order, for numpy's summation tree
  auto cub2 = [&](auto&& call) -> cudaError_t {   // cub's size query, its scratch, then the call
    size_t bytes = 0;
    cudaError_t e = call((void*)nullptr, bytes);
    char* t = nullptr;
    if (e == cudaSuccess) e = sc.get(&t, bytes);
    return e == cudaSuccess ? call((void*)t, bytes) : e;
  };
  int *nzs, *nzg, *ninf, *nsrcc, *zs_ptr, *zg_ptr, *zs_pos, *zg_pos, *nsel;
  unsigned char *fs, *fgz;
  for (int** a : {&nzs, &nzg, &ninf, &nsrcc, &zs_ptr, &zg_ptr}) {
    CK(h, sc.get(a, (size_t)ncomp + 1));
    CK(h, cudaMemsetAsync(*a, 0, ((size_t)ncomp + 1) * sizeof(int), st));
  }
  CK(h, sc.get(&zs_pos, n)); CK(h, sc.get(&zg_pos, n)); CK(h, sc.get(&nsel, 1));
  CK(h, sc.get(&fs, n)); CK(h, sc.get(&fgz, n));
  const unsigned* labs = key2;                    // each sorted position's label
  k_adv_counts<<<g, 256, 0, st>>>(n, rows, labs, s, gv, nzs, nzg, ninf, nsrcc, fs, fgz);
  CK(h, cudaGetLastError());
  CK(h, cub2([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, nzs, zs_ptr, ncomp + 1, st); }));
  CK(h, cub2([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, nzg, zg_ptr, ncomp + 1, st); }));
  CK(h, cub2([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, val, fs, zs_pos, nsel, n, st); }));
  CK(h, cub2([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, val, fgz, zg_pos, nsel, n, st); }));
  long long *solved, *iscol, *nset, *nsrc, *xsolved, *colx, *setx, *srcx;
  for (long long** a : {&solved, &iscol, &nset, &nsrc, &xsolved, &colx, &setx, &srcx}) CK(h, sc.get(a, (size_t)ncomp + 1));
  for (long long* a : {solved, iscol, nset, nsrc}) CK(h, cudaMemsetAsync(a + ncomp, 0, sizeof(long long), st));
  const int gs = (int)std::max<int64_t>(1, std::min<int64_t>((ncomp + ADV_SUM_THREADS - 1) / ADV_SUM_THREADS,
                                                             (int64_t)h->num_sms * 32));
  k_adv_sums<<<gs, ADV_SUM_THREADS, 0, st>>>(ncomp, cptr, rows, s, gv, zs_ptr, zs_pos, zg_ptr, zg_pos, ninf, nsrcc,
                                             solved, iscol, nset, nsrc);
  CK(h, cudaGetLastError());
  long long tot[4];
  {
    long long* in[4] = {solved, iscol, nset, nsrc};
    long long* outx[4] = {xsolved, colx, setx, srcx};
    for (int i = 0; i < 4; ++i) {
      CK(h, cub2([&](void* t, size_t& b) { return cub::DeviceScan::ExclusiveSum(t, b, in[i], outx[i], ncomp + 1, st); }));
      CK(h, cudaMemcpyAsync(tot + i, outx[i] + ncomp, sizeof(long long), cudaMemcpyDeviceToHost, st));
    }
  }
  CK(h, cudaStreamSynchronize(st));
  const PlanView sz(nullptr, tot[1], tot[2], tot[3], n);
  CK(h, cudaMalloc(&h->d_plan, std::max<size_t>(sz.bytes, 1)));
  const PlanView pv(h->d_plan, tot[1], tot[2], tot[3], n);
  CK(h, cudaMemsetAsync(pv.set_ptr, 0, sizeof(long long), st));
  CK(h, cudaMemsetAsync(pv.src_ptr, 0, sizeof(long long), st));
  CK(h, cudaMemsetAsync(pv.col_of_row, 0xff, (size_t)n * sizeof(int), st));
  const int gc = (int)std::max<int64_t>(1, std::min<int64_t>((ncomp + 255) / 256, (int64_t)h->num_sms * 32));
  k_adv_ptrs<<<gc, 256, 0, st>>>(ncomp, iscol, colx, setx, nset, srcx, nsrc, pv.col_comp, pv.set_ptr, pv.src_ptr);
  CK(h, cudaGetLastError());
  // fs / fgz are done with: they take the set and source flags; zs_pos / zg_pos the selected rows
  k_adv_mark<<<g, 256, 0, st>>>(n, rows, labs, s, gv, iscol, colx, pv.col_of_row, fs, fgz);
  CK(h, cudaGetLastError());
  CK(h, cub2([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, rows, fs, zs_pos, nsel, n, st); }));
  CK(h, cub2([&](void* t, size_t& b) { return cub::DeviceSelect::Flagged(t, b, rows, fgz, zg_pos, nsel, n, st); }));
  const int gn = (int)std::max<int64_t>(1, std::min<int64_t>((tot[2] + tot[3] + 255) / 256, (int64_t)h->num_sms * 32));
  k_adv_widen<<<gn, 256, 0, st>>>((int)tot[2], zs_pos, (int)tot[3], zg_pos, s, pv.set_rows, pv.src_rows, pv.src_vals);
  CK(h, cudaGetLastError());
  CK(h, cudaStreamSynchronize(st));
  h->stats.kernel_launches += 5;
  h->plan_ncol = tot[1];
  h->plan_nset = tot[2];
  h->plan_nsrc = tot[3];
  *ncol = tot[1];
  *nsolved = tot[0];
  *nset_rows = tot[2];
  *nsrc_rows = tot[3];
  *finite_applied = hf[1];
  if (!hf[1]) return CS_B200_OK;     // no finite ground: the operator stays as it is
  cudaEventRecord(h->ev0, st);
  void* fg = d_f;
  d_f = nullptr;
  return apply_grounds(h, fg, nullptr);
}

int cs_b200_read_advanced_plan(cs_b200_handle* h, int64_t* col_comp, int64_t* set_ptr, int64_t* set_rows,
                               int64_t* src_ptr, int64_t* src_rows, double* src_vals, int32_t* col_of_row) {
  if (!h) return CS_B200_ERR_ARG;
  if (!h->d_plan) return set_err(h, CS_B200_ERR_ARG, "cs_b200_read_advanced_plan: no plan (cs_b200_plan_advanced)");
  if (!col_comp || !set_ptr || !set_rows || !src_ptr || !src_rows || !src_vals || !col_of_row)
    return set_err(h, CS_B200_ERR_ARG, "cs_b200_read_advanced_plan: a NULL argument");
  cudaSetDevice(h->device);
  const int64_t nc = h->plan_ncol, ns = h->plan_nset, nv = h->plan_nsrc;
  const PlanView pv(h->d_plan, nc, ns, nv, h->n);
  const cudaMemcpyKind d2h = cudaMemcpyDeviceToHost;
  CK(h, cudaMemcpyAsync(col_comp, pv.col_comp, (size_t)nc * 8, d2h, h->stream));
  CK(h, cudaMemcpyAsync(set_ptr, pv.set_ptr, (size_t)(nc + 1) * 8, d2h, h->stream));
  CK(h, cudaMemcpyAsync(set_rows, pv.set_rows, (size_t)ns * 8, d2h, h->stream));
  CK(h, cudaMemcpyAsync(src_ptr, pv.src_ptr, (size_t)(nc + 1) * 8, d2h, h->stream));
  CK(h, cudaMemcpyAsync(src_rows, pv.src_rows, (size_t)nv * 8, d2h, h->stream));
  CK(h, cudaMemcpyAsync(src_vals, pv.src_vals, (size_t)nv * 8, d2h, h->stream));
  CK(h, cudaMemcpyAsync(col_of_row, pv.col_of_row, (size_t)h->n * 4, d2h, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  cudaFree(h->d_plan);
  h->d_plan = nullptr;
  h->plan_ncol = h->plan_nset = h->plan_nsrc = 0;
  return CS_B200_OK;
}

int cs_b200_currents_device_ptrs(cs_b200_handle* h, void** d_cum, void** d_max) {
  if (!h) return CS_B200_ERR_ARG;
  if (d_cum) *d_cum = h->d_cum;
  if (d_max) *d_max = h->d_max;
  return CS_B200_OK;
}

int cs_b200_stream(cs_b200_handle* h, void** stream) {
  if (!h || !stream) return CS_B200_ERR_ARG;
  *stream = (void*)h->stream;
  return CS_B200_OK;
}

int cs_b200_profile_spmm(cs_b200_handle* h, int enable, double* total_ms, int64_t* launches) {
  if (!h) return CS_B200_ERR_ARG;
  if (total_ms) *total_ms = h->prof_ms;
  if (launches) *launches = h->prof_launches;
  if (enable >= 0) {
    h->profile = enable ? 1 : 0;
    h->prof_ms = 0.0;
    h->prof_launches = 0;
    h->prof_used = 0;
    h->prof_bytes = 0.0;
    h->prof_slot.clear();
    h->prof_pair_bytes.clear();
    for (int i = 0; i < PROF_CLASSES; ++i) { h->prof_slot_ms[i] = 0.0; h->prof_slot_bytes[i] = 0.0; h->prof_slot_launches[i] = 0; }
  }
  return CS_B200_OK;
}

int cs_b200_profile_classes(cs_b200_handle* h, double* ms18, double* bytes18, int64_t* launches18) {
  return cs_b200_profile_classes_n(h, 18, ms18, bytes18, launches18);
}

int cs_b200_profile_classes_n(cs_b200_handle* h, int nslots, double* ms, double* bytes, int64_t* launches) {
  if (!h || nslots < 0) return CS_B200_ERR_ARG;
  for (int i = 0; i < std::min(nslots, PROF_CLASSES); ++i) {
    if (ms) ms[i] = h->prof_slot_ms[i];
    if (bytes) bytes[i] = h->prof_slot_bytes[i];
    if (launches) launches[i] = h->prof_slot_launches[i];
  }
  return CS_B200_OK;
}

int cs_b200_profile_bytes(cs_b200_handle* h, double* algorithmic_bytes) {
  if (!h || !algorithmic_bytes) return CS_B200_ERR_ARG;
  *algorithmic_bytes = h->prof_bytes;
  return CS_B200_OK;
}

int cs_b200_get_stats(const cs_b200_handle* h, cs_b200_stats* out) {
  if (!h || !out) return CS_B200_ERR_ARG;
  *out = h->stats;
  return CS_B200_OK;
}

int cs_b200_spmv(cs_b200_handle* h, const void* x, void* y, int reps, double* ms_per_rep) {
  if (!h || !x || !y || reps < 1) return set_err(h, CS_B200_ERR_ARG, "bad spmv arguments");
  begin_call(h);
  const size_t bytes = (size_t)h->n * h->esize();
  CK(h, cudaMemcpyAsync(h->X, x, bytes, cudaMemcpyHostToDevice, h->stream));
  CK(h, cudaEventRecord(h->ev2, h->stream));
  with_type(h, [&](auto t) {
    using T = decltype(t);
    for (int r = 0; r < reps; ++r) launch_spmm<T, 1, SP_PLAIN>(h, (const T*)h->X, (T*)h->AP, nullptr);
  });
  CK(h, cudaGetLastError());
  CK(h, cudaEventRecord(h->ev3, h->stream));
  CK(h, cudaMemcpyAsync(y, h->AP, bytes, cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  float ms = 0;
  CK(h, cudaEventElapsedTime(&ms, h->ev2, h->ev3));
  if (ms_per_rep) *ms_per_rep = ms / reps;
  h->stats.kernel_ms = ms;
  h->stats.h2d_bytes = h->stats.d2h_bytes = (double)bytes;
  end_call(h);
  return CS_B200_OK;
}

int cs_b200_spmm(cs_b200_handle* h, int k, const void* x, void* y) {
  const bool add = getenv("CS_B200_SPMM_ADD") != nullptr;   // debug: Y = X + A X through SP_ADD
  if (!h || !x || !y || (k != 1 && k != 2 && k != 4 && k != 8) || k > h->ktmax)
    return set_err(h, CS_B200_ERR_ARG, "bad spmm arguments");
  begin_call(h);
  const size_t bytes = (size_t)h->n * k * h->esize();
  const size_t nelem = (size_t)h->n_pad * k;
  const int tg = copy_grid(nelem);
  CK(h, cudaMemcpyAsync(h->stage, x, bytes, cudaMemcpyHostToDevice, h->stream));
  CK(h, cudaMemsetAsync(h->X, 0, nelem * h->esize(), h->stream));
  const int rc = with_type_width(h, k, [&](auto t, auto KT) -> int {
    using T = decltype(t);
    k_cm_to_panel<T, KT><<<tg, 256, 0, h->stream>>>((int)h->n, (size_t)h->n, (const T*)h->stage, (T*)h->X, KT);
    if (add) {
      CK(h, cudaMemcpyAsync(h->AP, h->X, nelem * h->esize(), cudaMemcpyDeviceToDevice, h->stream));
      launch_spmm<T, KT, SP_ADD>(h, (const T*)h->X, (T*)h->AP, (const T*)h->AP);
    } else {
      launch_spmm<T, KT, SP_PLAIN>(h, (const T*)h->X, (T*)h->AP, nullptr);
    }
    k_panel_to_cm<T, KT><<<tg, 256, 0, h->stream>>>((int)h->n, (size_t)h->n, (const T*)h->AP, (T*)h->stage, h->d_ctl, 0);
    return CS_B200_OK;
  });
  if (rc) return rc;
  CK(h, cudaGetLastError());
  CK(h, cudaMemcpyAsync(y, h->stage, bytes, cudaMemcpyDeviceToHost, h->stream));
  CK(h, cudaStreamSynchronize(h->stream));
  end_call(h);
  return CS_B200_OK;
}

int cs_b200_apply_precond(cs_b200_handle* h, int k, const void* r, void* z, double* rz) {
  if (!h || !r || !z || (k != 1 && k != 2 && k != 4 && k != 8) || k > h->ktmax)
    return set_err(h, CS_B200_ERR_ARG, "bad apply_precond arguments");
  if (!h->amg) return set_err(h, CS_B200_ERR_UNSUPPORTED, "apply_precond: the handle has no multigrid preconditioner");
  begin_call(h);
  const int rc = with_type_width(h, k, [&](auto t, auto KT) { return apply_precond_t<decltype(t), KT>(h, r, z, rz); });
  end_call(h);
  return rc;
}

int cs_b200_bench_spmm(cs_b200_handle* h, int k, int reps, int flush_l2, double* ms_per_rep) {
  if (!h || reps < 1 || (k != 1 && k != 2 && k != 4 && k != 8) || k > h->ktmax)
    return set_err(h, CS_B200_ERR_ARG, "bad bench_spmm arguments");
  begin_call(h);
  if (flush_l2) { int rc = ensure_flush(h); if (rc) return rc; }
  const size_t pe = (size_t)h->n_pad * k;
  with_type(h, [&](auto t) {
    using T = decltype(t);
    k_fill<T><<<copy_grid(pe), 256, 0, h->stream>>>((T*)h->X, pe, T(1));
  });
  double total = 0;
  auto one = [&]() {
    with_type_width(h, k, [&](auto t, auto KT) {
      using T = decltype(t);
      launch_spmm<T, KT, SP_PLAIN>(h, (const T*)h->X, (T*)h->AP, nullptr);
    });
  };
  one();  // warm-up
  if (flush_l2) {
    for (int r = 0; r < reps; ++r) {
      k_flush<<<h->num_sms * 8, 256, 0, h->stream>>>(h->d_flush, h->flush_elems);
      CK(h, cudaEventRecord(h->ev2, h->stream));
      one();
      CK(h, cudaEventRecord(h->ev3, h->stream));
      CK(h, cudaEventSynchronize(h->ev3));
      float ms = 0;
      CK(h, cudaEventElapsedTime(&ms, h->ev2, h->ev3));
      total += ms;
    }
  } else {
    CK(h, cudaEventRecord(h->ev2, h->stream));
    for (int r = 0; r < reps; ++r) one();
    CK(h, cudaEventRecord(h->ev3, h->stream));
    CK(h, cudaEventSynchronize(h->ev3));
    float ms = 0;
    CK(h, cudaEventElapsedTime(&ms, h->ev2, h->ev3));
    total = ms;
  }
  CK(h, cudaGetLastError());
  if (ms_per_rep) *ms_per_rep = total / reps;
  h->stats.kernel_ms = total;
  end_call(h);
  return CS_B200_OK;
}

int cs_b200_bench_cg_iter(cs_b200_handle* h, int k, int reps, double* ms_per_rep) {
  if (!h || reps < 1 || (k != 1 && k != 2 && k != 4 && k != 8) || k > h->ktmax)
    return set_err(h, CS_B200_ERR_ARG, "bad bench_cg_iter arguments");
  begin_call(h);
  PanelCtl* hc = h->h_ctl;
  std::memset(hc, 0, sizeof(PanelCtl));
  for (int c = 0; c < k; ++c) {
    hc->src[c] = (c * 7919) % h->n;
    hc->dst[c] = h->n - 1 - (c * 104729) % (h->n / 2 + 1);
    if (hc->dst[c] == hc->src[c]) hc->dst[c] = (hc->src[c] + 1) % h->n;
    hc->weight[c] = 1.0;
  }
  CK(h, cudaMemcpyAsync(h->d_ctl, hc, sizeof(PanelCtl), cudaMemcpyHostToDevice, h->stream));
  const size_t nelem = (size_t)h->n_pad * k;
  CK(h, cudaMemsetAsync(h->B, 0, nelem * h->esize(), h->stream));
  const int rc = with_type_width(h, k, [&](auto t, auto KT) -> int {
    using T = decltype(t);
    k_pair_rhs<T, KT><<<1, 32, 0, h->stream>>>((T*)h->B, h->d_ctl);
    k_cg_init<T, KT><<<ew_grid<T, KT>(h), NT, 0, h->stream>>>(nelem, (const T*)h->B, (const T*)h->d_dinv, (T*)h->X,
                                                              (T*)h->R, (T*)h->P, h->d_ctl, h->d_partials, 0.0, 0.0,
                                                              1 << 30);
    for (int w = 0; w < 3; ++w) launch_iteration<T, KT>(h);
    CK(h, cudaEventRecord(h->ev2, h->stream));
    for (int r = 0; r < reps; ++r) launch_iteration<T, KT>(h);
    return CS_B200_OK;
  });
  if (rc) return rc;
  CK(h, cudaEventRecord(h->ev3, h->stream));
  CK(h, cudaEventSynchronize(h->ev3));
  CK(h, cudaGetLastError());
  float ms = 0;
  CK(h, cudaEventElapsedTime(&ms, h->ev2, h->ev3));
  if (ms_per_rep) *ms_per_rep = ms / reps;
  h->stats.kernel_ms = ms;
  end_call(h);
  return CS_B200_OK;
}

int cs_b200_solve_rhs(cs_b200_handle* h, int64_t k, const void* rhs, void* lhs, double rtol,
                      int64_t itmax, int64_t* iters, double* relres) {
  if (!h || k < 1 || !rhs || !lhs || !(rtol >= 0) || itmax < 0)
    return set_err(h, CS_B200_ERR_ARG, "bad solve_rhs arguments");
  return solve_call(h, [&](auto t, ColumnDriver& cols) {
    using T = decltype(t);
    return solve_rhs_t<T>(h, k, (const T*)rhs, (T*)lhs, rtol, itmax, iters, relres, cols);
  });
}

// the pairs of cs_b200_solve_pairs / cs_b200_solve_pairs_branch (`who`)
static int check_pairs(cs_b200_handle* h, const char* who, int64_t k, const int64_t* src, const int64_t* dst,
                       const void* R, double rtol, int64_t itmax) {
  if (!h || k < 1 || !src || !dst || !R || !(rtol >= 0) || itmax < 0)
    return set_err(h, CS_B200_ERR_ARG, "bad %s arguments", who);
  for (int64_t c = 0; c < k; ++c)
    if (src[c] < 0 || src[c] >= h->n || dst[c] < 0 || dst[c] >= h->n || src[c] == dst[c])
      return set_err(h, CS_B200_ERR_ARG, "pair %lld: src/dst out of range or equal (%lld, %lld)",
                     (long long)c, (long long)src[c], (long long)dst[c]);
  return CS_B200_OK;
}

int cs_b200_solve_pairs(cs_b200_handle* h, int64_t k, const int64_t* src, const int64_t* dst,
                        const double* weight, double rtol, int64_t itmax, void* R, void* volt,
                        void* curr, int accumulate, int64_t* iters, double* relres) {
  if (int rc = check_pairs(h, "solve_pairs", k, src, dst, R, rtol, itmax)) return rc;
  return solve_call(h, [&](auto t, ColumnDriver& cols) {
    using T = decltype(t);
    return cols.run(0, k, [&](auto kt, int64_t c0) {
      return pairs_panel<T, kt>(h, c0, src, dst, weight, rtol, itmax, (T*)R, (T*)volt, (T*)curr, accumulate,
                                iters, relres, cols);
    });
  });
}

int cs_b200_solve_pairs_branch(cs_b200_handle* h, int64_t k, const int64_t* src, const int64_t* dst,
                               const double* weight, double rtol, int64_t itmax, void* R, void* volt,
                               void* curr, int accumulate, int64_t* iters, double* relres, void* branch) {
  if (int rc = check_pairs(h, "solve_pairs_branch", k, src, dst, R, rtol, itmax)) return rc;
  return solve_call(h, [&](auto t, ColumnDriver& cols) {
    using T = decltype(t);
    if (int rc = ensure_branch_index(h)) return rc;
    return cols.run(0, k, [&](auto kt, int64_t c0) {
      if (int rc = pairs_panel<T, kt>(h, c0, src, dst, weight, rtol, itmax, (T*)R, (T*)volt, (T*)curr, accumulate,
                                      iters, relres, cols))
        return rc;
      if (!accumulate && !curr) launch_cur_max<T, kt>(h);   // pairs_panel ran it only for the node currents
      return branch_pass<T, kt>(h, c0, (T*)branch, accumulate, kt);
    });
  });
}

int cs_b200_solve_sources(cs_b200_handle* h, int64_t k, const int64_t* colptr, const int64_t* rows,
                          const double* vals, const int64_t* ref, const double* weight,
                          double rtol, int64_t itmax, int64_t nprobe, const int64_t* probe,
                          void* probe_volt, void* volt, void* curr, int accumulate,
                          int64_t* iters, double* relres) {
  if (!h || k < 1 || !colptr || !ref || !(rtol >= 0) || itmax < 0 || nprobe < 0 ||
      (nprobe > 0 && !probe) || colptr[0] != 0)
    return set_err(h, CS_B200_ERR_ARG, "bad solve_sources arguments");
  for (int64_t c = 0; c < k; ++c) {
    if (colptr[c + 1] < colptr[c] || ref[c] < 0 || ref[c] >= h->n)
      return set_err(h, CS_B200_ERR_ARG, "column %lld: bad colptr or reference row", (long long)c);
  }
  if (colptr[k] > 0 && (!rows || !vals)) return set_err(h, CS_B200_ERR_ARG, "rows/vals missing");
  for (int64_t e = 0; e < colptr[k]; ++e)
    if (rows[e] < 0 || rows[e] >= h->n)
      return set_err(h, CS_B200_ERR_ARG, "entry %lld: row %lld out of range", (long long)e, (long long)rows[e]);
  for (int64_t i = 0; i < nprobe; ++i)
    if (probe[i] < 0 || probe[i] >= h->n) return set_err(h, CS_B200_ERR_ARG, "probe row out of range");
  return solve_call(h, [&](auto t, ColumnDriver& cols) {
    using T = decltype(t);
    if (nprobe > 0 && probe_volt)
      if (int rc = upload_probe(h, nprobe, probe)) return rc;
    return cols.run(0, k, [&](auto kt, int64_t c0) {
      return sources_panel<T, kt>(h, c0, colptr, rows, vals, ref, weight, rtol, itmax, nprobe, (T*)probe_volt,
                                  (T*)volt, (T*)curr, accumulate, iters, relres, cols);
    });
  });
}

int cs_b200_solve_pairs_superposed(cs_b200_handle* h, int64_t np, const int64_t* nodes, int64_t k,
                                   const int64_t* pi, const int64_t* pj, const double* weight,
                                   double rtol, int64_t itmax, void* R, void* volt, void* curr,
                                   int accumulate, int64_t* point_iters, double* relres) {
  if (!h || np < 2 || !nodes || k < 1 || !pi || !pj || !R || !(rtol >= 0) || itmax < 0)
    return set_err(h, CS_B200_ERR_ARG, "bad solve_pairs_superposed arguments");
  for (int64_t x = 0; x < np; ++x) {
    if (nodes[x] < 0 || nodes[x] >= h->n)
      return set_err(h, CS_B200_ERR_ARG, "focal node %lld out of range", (long long)x);
    if (x > 0 && nodes[x] == nodes[0])
      return set_err(h, CS_B200_ERR_ARG, "focal node %lld repeats the reference node", (long long)x);
  }
  for (int64_t c = 0; c < k; ++c)
    if (pi[c] < 0 || pi[c] >= np || pj[c] < 0 || pj[c] >= np || nodes[pi[c]] == nodes[pj[c]])
      return set_err(h, CS_B200_ERR_ARG, "pair %lld: indices out of range or equal nodes", (long long)c);
  return solve_call(h, [&](auto t, ColumnDriver& cols) {
    using T = decltype(t);
    return solve_pairs_superposed_t<T>(h, np, nodes, k, pi, pj, weight, rtol, itmax, (T*)R, (T*)volt, (T*)curr,
                                       accumulate, point_iters, relres, cols);
  });
}

// the sets of one CSR (set_ptr[nsets+1], set_rows): non-empty, sorted, unique, rows in range
static int check_sets(cs_b200_handle* h, int64_t nsets, const int64_t* set_ptr, const int64_t* set_rows) {
  if (set_ptr[0] != 0) return set_err(h, CS_B200_ERR_ARG, "set_ptr[0] must be 0");
  for (int64_t s = 0; s < nsets; ++s) {
    if (set_ptr[s + 1] <= set_ptr[s]) return set_err(h, CS_B200_ERR_ARG, "set %lld is empty", (long long)s);
    for (int64_t e = set_ptr[s]; e < set_ptr[s + 1]; ++e) {
      if (set_rows[e] < 0 || (h && set_rows[e] >= h->n) || set_rows[e] > INT32_MAX)
        return set_err(h, CS_B200_ERR_ARG, "set %lld: row %lld out of range", (long long)s, (long long)set_rows[e]);
      if (e > set_ptr[s] && set_rows[e] <= set_rows[e - 1])
        return set_err(h, CS_B200_ERR_ARG, "set %lld: rows not sorted and unique", (long long)s);
    }
  }
  return CS_B200_OK;
}

int cs_b200_solve_region_pairs(cs_b200_handle* h, int64_t nsets, const int64_t* set_ptr,
                               const int64_t* set_rows, int64_t k, const int64_t* set_a,
                               const int64_t* set_b, const double* weight, double rtol, int64_t itmax,
                               void* R, void* volt, void* curr, int accumulate,
                               int64_t* iters, double* relres) {
  // the sets are checked before the handle so that malformed input is reported the same way with or
  // without a device; row ranges need the handle's n
  if (k < 1 || nsets < 1 || !set_ptr || !set_rows || !set_a || !set_b || !R || !(rtol >= 0) || itmax < 0)
    return set_err(h, CS_B200_ERR_ARG, "bad solve_region_pairs arguments");
  if (int rc = check_sets(h, nsets, set_ptr, set_rows)) return rc;
  for (int64_t c = 0; c < k; ++c) {
    const int64_t a = set_a[c], b = set_b[c];
    if (a < 0 || a >= nsets || b < 0 || b >= nsets)
      return set_err(h, CS_B200_ERR_ARG, "column %lld: set index out of range (%lld, %lld)", (long long)c,
                     (long long)a, (long long)b);
    // sorted merge: the two sets of a column must not share a row
    int64_t i = set_ptr[a], j = set_ptr[b];
    while (i < set_ptr[a + 1] && j < set_ptr[b + 1]) {
      if (set_rows[i] == set_rows[j])
        return set_err(h, CS_B200_ERR_ARG, "column %lld: sets %lld and %lld overlap at row %lld", (long long)c,
                       (long long)a, (long long)b, (long long)set_rows[i]);
      if (set_rows[i] < set_rows[j]) ++i; else ++j;
    }
  }
  return solve_call(h, [&](auto t, ColumnDriver& cols) {
    using T = decltype(t);
    return cols.run(0, k, [&](auto kt, int64_t c0) {
      return region_panel<T, kt>(h, c0, set_ptr, set_rows, set_a, set_b, weight, rtol, itmax, (T*)R, (T*)volt,
                                 (T*)curr, accumulate, iters, relres, cols);
    });
  });
}

// the columns of cs_b200_solve_grounded / cs_b200_solve_advanced (`who`): everything is checked before
// the handle, as in cs_b200_solve_region_pairs; row ranges need its n.  gset[c] = -1 (no direct grounds)
// is accepted only when `floating_ok`.
static int check_grounded_columns(cs_b200_handle* h, const char* who, int64_t nsets, const int64_t* set_ptr,
                                  const int64_t* set_rows, int64_t k, const int64_t* gset, const int64_t* src_ptr,
                                  const int64_t* src_rows, const double* src_vals, double rtol, int64_t itmax,
                                  bool floating_ok) {
  if (k < 1 || nsets < (floating_ok ? 0 : 1) || !set_ptr || (nsets > 0 && !set_rows) || !gset || !src_ptr ||
      !src_rows || !src_vals || !(rtol >= 0) || itmax < 0)
    return set_err(h, CS_B200_ERR_ARG, "bad %s arguments", who);
  if (int rc = check_sets(h, nsets, set_ptr, set_rows)) return rc;
  if (src_ptr[0] != 0) return set_err(h, CS_B200_ERR_ARG, "src_ptr[0] must be 0");
  for (int64_t c = 0; c < k; ++c) {
    const int64_t s = gset[c];
    if (s < (floating_ok ? -1 : 0) || s >= nsets)
      return set_err(h, CS_B200_ERR_ARG, "column %lld: set index %lld out of range", (long long)c, (long long)s);
    if (src_ptr[c + 1] <= src_ptr[c])
      return set_err(h, CS_B200_ERR_ARG, "column %lld has no sources", (long long)c);
    if (src_ptr[c + 1] - src_ptr[0] > INT32_MAX)
      return set_err(h, CS_B200_ERR_ARG, "too many source entries");
    for (int64_t e = src_ptr[c]; e < src_ptr[c + 1]; ++e) {
      const int64_t r = src_rows[e];
      if (r < 0 || (h && r >= h->n) || r > INT32_MAX)
        return set_err(h, CS_B200_ERR_ARG, "column %lld: source row %lld out of range", (long long)c, (long long)r);
      if (s >= 0 && std::binary_search(set_rows + set_ptr[s], set_rows + set_ptr[s + 1], r))
        return set_err(h, CS_B200_ERR_ARG, "column %lld: source row %lld is on its ground set %lld", (long long)c,
                       (long long)r, (long long)s);
    }
  }
  return CS_B200_OK;
}

int cs_b200_solve_grounded(cs_b200_handle* h, int64_t nsets, const int64_t* set_ptr, const int64_t* set_rows,
                           int64_t k, const int64_t* gset, const int64_t* src_ptr, const int64_t* src_rows,
                           const double* src_vals, const double* weight, double rtol, int64_t itmax,
                           void* src_volt, void* volt, void* curr, int accumulate, int64_t* iters,
                           double* relres) {
  if (int rc = check_grounded_columns(h, "solve_grounded", nsets, set_ptr, set_rows, k, gset, src_ptr, src_rows,
                                      src_vals, rtol, itmax, false))
    return rc;
  return solve_call(h, [&](auto t, ColumnDriver& cols) {
    using T = decltype(t);
    return cols.run(0, k, [&](auto kt, int64_t c0) {
      return grounded_panel<T, kt>(h, c0, set_ptr, set_rows, gset, src_ptr, src_rows, src_vals, weight, rtol,
                                   itmax, (T*)src_volt, (T*)volt, (T*)curr, accumulate, iters, relres, cols,
                                   nullptr);
    });
  });
}

int cs_b200_solve_advanced(cs_b200_handle* h, int64_t nsets, const int64_t* set_ptr, const int64_t* set_rows,
                           int64_t k, const int64_t* gset, const int64_t* src_ptr, const int64_t* src_rows,
                           const double* src_vals, const double* weight, double rtol, int64_t itmax, void* volt,
                           void* curr, int accumulate, int64_t* iters, double* relres) {
  if (int rc = check_grounded_columns(h, "solve_advanced", nsets, set_ptr, set_rows, k, gset, src_ptr, src_rows,
                                      src_vals, rtol, itmax, true))
    return rc;
  for (int64_t c = 0; c < k; ++c)
    if (gset[c] < 0 && !(h && h->d_fg))
      return set_err(h, CS_B200_ERR_ARG, "column %lld has no direct grounds and the handle no finite grounds "
                     "(cs_b200_set_grounds)", (long long)c);
  return solve_call(h, [&](auto t, ColumnDriver& cols) {
    using T = decltype(t);
    return cols.run(0, k, [&](auto kt, int64_t c0) {
      return grounded_panel<T, kt>(h, c0, set_ptr, set_rows, gset, src_ptr, src_rows, src_vals, weight, rtol,
                                   itmax, (T*)nullptr, (T*)volt, (T*)curr, accumulate, iters, relres, cols,
                                   h->d_fg);
    });
  });
}

int cs_b200_solve_advanced_network(cs_b200_handle* h, int64_t nsets, const int64_t* set_ptr,
                                   const int64_t* set_rows, int64_t k, const int64_t* gset, const int64_t* src_ptr,
                                   const int64_t* src_rows, const double* src_vals, const int64_t* owner,
                                   double rtol, int64_t itmax, void* volt, void* curr, void* branch,
                                   int64_t* iters, double* relres) {
  if (int rc = check_grounded_columns(h, "solve_advanced_network", nsets, set_ptr, set_rows, k, gset, src_ptr,
                                      src_rows, src_vals, rtol, itmax, true))
    return rc;
  if (!owner) return set_err(h, CS_B200_ERR_ARG, "bad solve_advanced_network arguments (owner)");
  for (int64_t c = 0; c < k; ++c)
    if (gset[c] < 0 && !(h && h->d_fg))
      return set_err(h, CS_B200_ERR_ARG, "column %lld has no direct grounds and the handle no finite grounds "
                     "(cs_b200_set_grounds)", (long long)c);
  if (h) {                           // owner has the handle's n rows
    for (int64_t r = 0; r < h->n; ++r)
      if (owner[r] < -1 || owner[r] >= k)
        return set_err(h, CS_B200_ERR_ARG, "owner[%lld] = %lld is not a column or -1", (long long)r,
                       (long long)owner[r]);
    for (int64_t c = 0; c < k; ++c) {
      for (int64_t e = src_ptr[c]; e < src_ptr[c + 1]; ++e)
        if (owner[src_rows[e]] != c)
          return set_err(h, CS_B200_ERR_ARG, "column %lld: source row %lld is owned by column %lld", (long long)c,
                         (long long)src_rows[e], (long long)owner[src_rows[e]]);
      if (gset[c] >= 0)
        for (int64_t e = set_ptr[gset[c]]; e < set_ptr[gset[c] + 1]; ++e)
          if (owner[set_rows[e]] != c)
            return set_err(h, CS_B200_ERR_ARG, "column %lld: ground row %lld is owned by column %lld",
                           (long long)c, (long long)set_rows[e], (long long)owner[set_rows[e]]);
    }
  }
  return solve_call(h, [&](auto t, ColumnDriver& cols) {
    using T = decltype(t);
    return advanced_network_t<T>(h, set_ptr, set_rows, k, gset, src_ptr, src_rows, src_vals, owner, rtol, itmax,
                                 (T*)volt, (T*)curr, (T*)branch, iters, relres, cols);
  });
}

}  // extern "C"
// ---------------------------------------------------------------------------------------------
// multi-GPU: NCCL behind the C ABI (loaded at run time, so a single-GPU user needs no NCCL)
// ---------------------------------------------------------------------------------------------
#include <dlfcn.h>

namespace {

struct NcclId { char internal[128]; };
typedef void* ncclComm_p;
// enums of nccl.h (stable across NCCL 2.x)
enum { NCCL_INT8 = 0, NCCL_INT32 = 2, NCCL_INT64 = 4, NCCL_FLOAT32 = 7, NCCL_FLOAT64 = 8 };
enum { NCCL_SUM = 0, NCCL_MAX = 2 };

struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(NcclId*) = nullptr;
  int (*CommInitRank)(ncclComm_p*, int, NcclId, int) = nullptr;
  int (*CommDestroy)(ncclComm_p) = nullptr;
  int (*Broadcast)(const void*, void*, size_t, int, int, ncclComm_p, cudaStream_t) = nullptr;
  int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_p, cudaStream_t) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, ncclComm_p, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
  std::string err;
};

NcclApi& nccl_api() {
  static NcclApi api;
  if (api.lib || !api.err.empty()) return api;
  const char* names[] = {std::getenv("CS_B200_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
  for (const char* nm : names) {
    if (!nm) continue;
    api.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
    if (api.lib) break;
  }
  if (!api.lib) { api.err = std::string("cannot load NCCL (libnccl.so.2): ") + dlerror(); return api; }
  auto sym = [&](const char* s) { void* p = dlsym(api.lib, s); if (!p) api.err = std::string("NCCL symbol missing: ") + s; return p; };
  api.GetUniqueId = (int (*)(NcclId*))sym("ncclGetUniqueId");
  api.CommInitRank = (int (*)(ncclComm_p*, int, NcclId, int))sym("ncclCommInitRank");
  api.CommDestroy = (int (*)(ncclComm_p))sym("ncclCommDestroy");
  api.Broadcast = (int (*)(const void*, void*, size_t, int, int, ncclComm_p, cudaStream_t))sym("ncclBroadcast");
  api.AllReduce = (int (*)(const void*, void*, size_t, int, int, ncclComm_p, cudaStream_t))sym("ncclAllReduce");
  api.AllGather = (int (*)(const void*, void*, size_t, int, ncclComm_p, cudaStream_t))sym("ncclAllGather");
  api.GetErrorString = (const char* (*)(int))sym("ncclGetErrorString");
  return api;
}

thread_local std::string g_comm_error;

}  // namespace

struct cs_b200_comm {
  int device = 0, rank = 0, nranks = 1;
  ncclComm_p comm = nullptr;
  cudaStream_t stream = nullptr;
  std::string err;
};

namespace {
int comm_err(cs_b200_comm* c, int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (c) c->err = buf; else g_comm_error = buf;
  return code;
}
#define CKN(c, call)                                                                                  \
  do {                                                                                                \
    int _r = (call);                                                                                  \
    if (_r != 0) return comm_err(c, CS_B200_ERR_CUDA, "NCCL error %s (%s)", nccl_api().GetErrorString(_r), #call); \
  } while (0)
#define CKU(c, call)                                                                                  \
  do {                                                                                                \
    cudaError_t _e = (call);                                                                          \
    if (_e != cudaSuccess) return comm_err(c, CS_B200_ERR_CUDA, "CUDA error %s (%s)", cudaGetErrorString(_e), #call); \
  } while (0)
}  // namespace

extern "C" {

int cs_b200_comm_unique_id(void* id128) {
  if (!id128) return comm_err(nullptr, CS_B200_ERR_ARG, "id128 is NULL");
  NcclApi& api = nccl_api();
  if (!api.err.empty()) return comm_err(nullptr, CS_B200_ERR_UNSUPPORTED, "%s", api.err.c_str());
  NcclId id;
  CKN(nullptr, api.GetUniqueId(&id));
  std::memcpy(id128, &id, sizeof id);
  return CS_B200_OK;
}

int cs_b200_comm_init(int device, int rank, int nranks, const void* id128, cs_b200_comm** out) {
  if (!out || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return comm_err(nullptr, CS_B200_ERR_ARG, "bad comm_init arguments");
  *out = nullptr;
  NcclApi& api = nccl_api();
  if (!api.err.empty()) return comm_err(nullptr, CS_B200_ERR_UNSUPPORTED, "%s", api.err.c_str());
  CKU(nullptr, cudaSetDevice(device));
  cs_b200_comm* c = new cs_b200_comm();
  c->device = device; c->rank = rank; c->nranks = nranks;
  NcclId id;
  std::memcpy(&id, id128, sizeof id);
  int r = api.CommInitRank(&c->comm, nranks, id, rank);
  if (r != 0) { comm_err(nullptr, CS_B200_ERR_CUDA, "NCCL error %s (ncclCommInitRank)", api.GetErrorString(r)); delete c; return CS_B200_ERR_CUDA; }
  cudaError_t e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) { comm_err(nullptr, CS_B200_ERR_CUDA, "CUDA error %s creating the comm stream", cudaGetErrorString(e)); api.CommDestroy(c->comm); delete c; return CS_B200_ERR_CUDA; }
  *out = c;
  return CS_B200_OK;
}

void cs_b200_comm_destroy(cs_b200_comm* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->stream) { cudaStreamSynchronize(c->stream); cudaStreamDestroy(c->stream); }
  if (c->comm) nccl_api().CommDestroy(c->comm);
  delete c;
}

const char* cs_b200_comm_last_error(const cs_b200_comm* c) { return c ? c->err.c_str() : g_comm_error.c_str(); }

int cs_b200_comm_barrier(cs_b200_comm* c) {
  if (!c) return CS_B200_ERR_ARG;
  cudaSetDevice(c->device);
  int* d = nullptr;
  CKU(c, cudaMalloc(&d, sizeof(int)));
  cudaMemsetAsync(d, 0, sizeof(int), c->stream);
  int r = nccl_api().AllReduce(d, d, 1, NCCL_INT32, NCCL_SUM, c->comm, c->stream);
  cudaError_t e = cudaStreamSynchronize(c->stream);
  cudaFree(d);
  if (r != 0) return comm_err(c, CS_B200_ERR_CUDA, "NCCL error %s (barrier)", nccl_api().GetErrorString(r));
  CKU(c, e);
  return CS_B200_OK;
}

int cs_b200_comm_max_double(cs_b200_comm* c, double* v, int count) {
  if (!c || !v || count < 1) return CS_B200_ERR_ARG;
  cudaSetDevice(c->device);
  double* d = nullptr;
  CKU(c, cudaMalloc(&d, (size_t)count * sizeof(double)));
  cudaMemcpyAsync(d, v, (size_t)count * sizeof(double), cudaMemcpyHostToDevice, c->stream);
  int r = nccl_api().AllReduce(d, d, (size_t)count, NCCL_FLOAT64, NCCL_MAX, c->comm, c->stream);
  cudaMemcpyAsync(v, d, (size_t)count * sizeof(double), cudaMemcpyDeviceToHost, c->stream);
  cudaError_t e = cudaStreamSynchronize(c->stream);
  cudaFree(d);
  if (r != 0) return comm_err(c, CS_B200_ERR_CUDA, "NCCL error %s (max_double)", nccl_api().GetErrorString(r));
  CKU(c, e);
  return CS_B200_OK;
}

int cs_b200_comm_reduce_currents(cs_b200_comm* c, cs_b200_handle* h) {
  if (!c || !h || h->device != c->device) return comm_err(c, CS_B200_ERR_ARG, "bad reduce_currents arguments");
  cudaSetDevice(c->device);
  const int dt = h->dtype == CS_B200_F64 ? NCCL_FLOAT64 : NCCL_FLOAT32;
  // on the handle's own stream: ordered right behind the last accumulation kernel, no host sync between
  CKN(c, nccl_api().AllReduce(h->d_cum, h->d_cum, (size_t)h->n, dt, NCCL_SUM, c->comm, h->stream));
  CKN(c, nccl_api().AllReduce(h->d_max, h->d_max, (size_t)h->n, dt, NCCL_MAX, c->comm, h->stream));
  CKU(c, cudaStreamSynchronize(h->stream));
  return CS_B200_OK;
}

int cs_b200_comm_gather_pairs(cs_b200_comm* c, int64_t k_total, const int64_t* my_idx, int64_t k_mine,
                              const double* my_R, double* R_all) {
  if (!c || k_total < 1 || k_mine < 0 || (k_mine > 0 && (!my_idx || !my_R)) || !R_all)
    return comm_err(c, CS_B200_ERR_ARG, "bad gather_pairs arguments");
  cudaSetDevice(c->device);
  // fixed-size slots: ceil(k_total / nranks) (index, value) pairs per rank, index -1 = empty
  const int64_t slot = (k_total + c->nranks - 1) / c->nranks;
  if (k_mine > slot) return comm_err(c, CS_B200_ERR_ARG, "rank %d holds %lld pairs, more than ceil(k_total / nranks) = %lld", c->rank, (long long)k_mine, (long long)slot);
  std::vector<double> send((size_t)2 * slot, -1.0), recv((size_t)2 * slot * c->nranks);
  for (int64_t i = 0; i < k_mine; ++i) { send[2 * i] = (double)my_idx[i]; send[2 * i + 1] = my_R[i]; }
  double *ds = nullptr, *dr = nullptr;
  CKU(c, cudaMalloc(&ds, send.size() * sizeof(double)));
  cudaError_t e = cudaMalloc(&dr, recv.size() * sizeof(double));
  if (e != cudaSuccess) { cudaFree(ds); CKU(c, e); }
  cudaMemcpyAsync(ds, send.data(), send.size() * sizeof(double), cudaMemcpyHostToDevice, c->stream);
  int r = nccl_api().AllGather(ds, dr, send.size(), NCCL_FLOAT64, c->comm, c->stream);
  cudaMemcpyAsync(recv.data(), dr, recv.size() * sizeof(double), cudaMemcpyDeviceToHost, c->stream);
  e = cudaStreamSynchronize(c->stream);
  cudaFree(ds); cudaFree(dr);
  if (r != 0) return comm_err(c, CS_B200_ERR_CUDA, "NCCL error %s (gather_pairs)", nccl_api().GetErrorString(r));
  CKU(c, e);
  for (int64_t i = 0; i < k_total; ++i) R_all[i] = -1.0;
  for (size_t q = 0; q + 1 < recv.size(); q += 2) {
    const int64_t idx = (int64_t)recv[q];
    if (idx >= 0 && idx < k_total) R_all[idx] = recv[q + 1];
  }
  return CS_B200_OK;
}

int cs_b200_create_bcast(cs_b200_comm* c, int root, int64_t n, int64_t nnz, const void* rowptr,
                         const void* colidx, const void* vals, int index_bits, int index_base,
                         int dtype, const cs_b200_opts* opts, cs_b200_handle** out) {
  if (!out) return comm_err(c, CS_B200_ERR_ARG, "out is NULL");
  *out = nullptr;
  if (!c || root < 0 || root >= c->nranks || n <= 0 || nnz <= 0 || (dtype != CS_B200_F32 && dtype != CS_B200_F64) ||
      nnz >= (int64_t)1 << 31 || n >= (int64_t)1 << 31 || (index_bits != 32 && index_bits != 64) ||
      (index_base != 0 && index_base != 1))
    return comm_err(c, CS_B200_ERR_ARG, "bad create_bcast arguments");
  const bool is_root = c->rank == root;
  if (is_root && (!rowptr || !colidx || !vals)) return comm_err(c, CS_B200_ERR_ARG, "the root rank must pass the matrix");
  const csb_dev::HostPattern hp = is_root ? csb_dev::HostPattern{rowptr, colidx, index_bits, index_base} : csb_dev::HostPattern{};
  return create_handle(n, nnz, dtype, c->device, opts, hp, &c->err, out, [&](cs_b200_handle* h, Seeds& seeds) -> int {
    int rc = upload_host_csr(h, is_root ? rowptr : nullptr, colidx, vals, index_bits, index_base);
    if (rc) return rc;
    // one broadcast of the CSR (SURVEY.md 8e), on the handle's stream behind the upload
    NcclApi& api = nccl_api();
    const size_t es = h->esize();
#define CKBN(call)                                                                                 \
  do {                                                                                             \
    int _r = (call);                                                                               \
    if (_r != 0) return set_err(h, CS_B200_ERR_CUDA, "NCCL error %s (%s)", api.GetErrorString(_r), #call); \
  } while (0)
    CKBN(api.Broadcast(h->d_rowptr, h->d_rowptr, (size_t)(n + 1), NCCL_INT32, root, c->comm, h->stream));
    CKBN(api.Broadcast(h->d_colidx, h->d_colidx, (size_t)nnz, NCCL_INT32, root, c->comm, h->stream));
    CKBN(api.Broadcast(h->d_vals, h->d_vals, (size_t)nnz * es, NCCL_INT8, root, c->comm, h->stream));
#undef CKBN
    if (!seeds.wanted) return CS_B200_OK;
    // the root's ordered aggregation seeds travel the same way (n ints) instead of every rank
    // downloading the pattern and repeating the pass
    CK(h, cudaMalloc(&seeds.d_seed, (size_t)(n + 1) * sizeof(int)));
    if (is_root) {
      const int* seed = nullptr;
      int64_t cnt = 0;
      const int nagg = csb_dev::seed_wait(seeds.job, &seed, &cnt);
      CK(h, cudaMemcpyAsync(seeds.d_seed, seed, (size_t)n * sizeof(int), cudaMemcpyHostToDevice, h->stream));
      CK(h, cudaMemcpyAsync(seeds.d_seed + n, &nagg, sizeof(int), cudaMemcpyHostToDevice, h->stream));
      CK(h, cudaStreamSynchronize(h->stream));
    }
    int r = api.Broadcast(seeds.d_seed, seeds.d_seed, (size_t)(n + 1), NCCL_INT32, root, c->comm, h->stream);
    int nagg = 0;
    cudaError_t e = cudaMemcpyAsync(&nagg, seeds.d_seed + n, sizeof(int), cudaMemcpyDeviceToHost, h->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(h->stream);
    if (r != 0 || e != cudaSuccess)
      return set_err(h, CS_B200_ERR_CUDA, "broadcast of the aggregation seeds failed (%s)", r != 0 ? api.GetErrorString(r) : cudaGetErrorString(e));
    seeds.dev.d_seed = seeds.d_seed;
    seeds.dev.nagg = nagg;
    return CS_B200_OK;
  });
}

}  // extern "C"

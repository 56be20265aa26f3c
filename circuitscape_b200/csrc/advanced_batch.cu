// advanced_batch.cu -- many small advanced-mode problems in one launch: the moving-window solve of
// compute_omniscape_current (src/utils.jl:145-257) for a stack of conductance windows.
//
// The handle-based solver keeps one large operator resident and amortises an AMG setup over many
// right-hand sides; a window is the opposite shape (thousands of independent operators of ~10^4
// cells, one right-hand side each).  So each window is one CTA that runs the whole advanced-mode
// kernel (src/raster/advanced.jl:151-305 with the raster branch of src/out.jl:178-207) on its own:
//   1. valid cells (g > 0; NODATA, 0 and NaN are not nodes), outputs zeroed
//   2. conflict resolution, policy rmvsrc (src/raster/advanced.jl:119-149)
//   3. connected-component labels: hooking with atomicMin + pointer jumping; label = smallest cell
//   4. skip rule (sum(sources) == 0 or sum(grounds) == 0), candidates flagged with integer ops first
//   5. Jacobi-preconditioned CG per solved component, in order of its smallest cell, with the
//      Krylov stop rule sqrt(r'z) <= atol + rtol sqrt(r0'z0)
//   6. true-residual gate ||b - A x|| / ||b|| on the reduced system (Inf grounds deleted)
//   7. node currents max(inflow, outflow) with the 1e-8 cut relative to the component's maxima
// The operator is never stored: edge weights come from the conductances through ras::weight and the
// Dirichlet (Inf-ground) cells are held at 0.  Window data is window-major, column-major inside a
// window (cell r + c * nrows), so a CTA's passes are coalesced down raster columns.  Every
// reduction is a fixed-order CTA tree and there are no floating-point atomics, so a window's
// result depends on its own data and shape only: repeat runs and any split into batches give
// bit-identical outputs.
#include "../../include/cs_b200.h"

#include <cuda_runtime.h>

#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_select.cuh>

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <vector>

#include "raster_assembly.cuh"

int set_handleless_error(int code, const char* msg);   // cs_b200.cu: the text of cs_b200_last_error(NULL)

namespace {

int set_err(int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  return set_handleless_error(code, buf);
}

constexpr int BT = 256;               // threads per window
constexpr int NWARP = BT / 32;
constexpr int NVEC = 5;               // x, r, p, q, diag
constexpr double kNodata = -9999.0;
constexpr double kCut = 1e-8;         // src/out.jl:281-287
constexpr double kGate = 1e-4;        // src/core.jl:641

enum WinStatus { WIN_OK = 0, WIN_MAXITER = 1, WIN_RESIDUAL = 2 };

struct WinOut {
  double relres;         // max over the window's solved components
  double fail_relres;    // first component that failed the gate (or ran into itmax)
  long long iters;       // summed over the window's solved components
  int fail_iters;
  int status;            // WinStatus
};

struct Shape {
  int nrows, ncols, ncell, four;
};

// visit the valid stencil neighbours of cell i: f(j, diagonal).  Slot k -> (dr, dc) = (k % 3 - 1,
// k / 3 - 1) as in raster_assembly.cuh, so FORWARD (k > 4) visits exactly the neighbours j > i.
template <bool FORWARD, typename T, class F>
__device__ __forceinline__ void for_nbrs(const Shape& s, const T* __restrict__ g, int i, F&& f) {
  const int r = i % s.nrows, c = i / s.nrows;
#pragma unroll
  for (int k = FORWARD ? 5 : 0; k < 9; ++k) {
    if (k == 4) continue;
    const int dr = k % 3 - 1, dc = k / 3 - 1;
    const bool diagonal = dr != 0 && dc != 0;
    if (s.four && diagonal) continue;
    const int rr = r + dr, cc = c + dc;
    if (rr < 0 || rr >= s.nrows || cc < 0 || cc >= s.ncols) continue;
    const int j = cc * s.nrows + rr;
    const double gj = (double)g[j];
    if (gj > 0.0) f(j, gj, diagonal);
  }
}

// fixed-order CTA reductions (shuffle tree per warp, then the warps in order); every thread gets the result
__device__ __forceinline__ double block_sum(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = sh[0];
    for (int w = 1; w < NWARP; ++w) t += sh[w];
    sh[NWARP] = t;
  }
  __syncthreads();
  return sh[NWARP];
}

__device__ __forceinline__ double dmax(double a, double b) { return a > b ? a : b; }

__device__ __forceinline__ double block_max(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = dmax(v, __shfl_down_sync(0xffffffffu, v, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = sh[0];
    for (int w = 1; w < NWARP; ++w) t = dmax(t, sh[w]);
    sh[NWARP] = t;
  }
  __syncthreads();
  return sh[NWARP];
}

__device__ __forceinline__ int find_root(const volatile int* lab, int x) {
  int p = lab[x];
  while (p != x) { x = p; p = lab[x]; }
  return x;
}

// source of a node after resolve_conflicts(..., "rmvsrc"): dropped where the cell is also grounded
__device__ __forceinline__ double node_source(double s, double gnd) { return (s != 0.0 && gnd != 0.0) ? 0.0 : s; }

// ground after resolve_conflicts: Inf grounds under a positive source are dropped (a no-op once
// rmvsrc has zeroed those sources, kept so the rule reads as the reference's)
__device__ __forceinline__ double node_ground(double s, double gnd) {
  return (isinf(gnd) && node_source(s, gnd) > 0.0) ? 0.0 : gnd;
}

// the finite-ground conductance of a node (Inf grounds are Dirichlet nodes, not conductances)
__device__ __forceinline__ double node_finite(double gnd) { return isfinite(gnd) ? gnd : 0.0; }

__device__ __forceinline__ double cut(double b, double mx) { return fabs(b / mx) < kCut ? 0.0 : b; }

template <typename T>
__global__ void __launch_bounds__(BT)
k_advanced_batch(Shape s, const T* __restrict__ g_all, const T* __restrict__ src_all,
                 const T* __restrict__ gnd_all, double rtol, double atol, long long itmax,
                 double* __restrict__ cur_all, double* __restrict__ volt_all, double* __restrict__ vec_all,
                 int* __restrict__ lab_all, int* __restrict__ flag_all, int* __restrict__ list_all,
                 WinOut* __restrict__ out) {
  using Scan = cub::BlockScan<int, BT>;
  __shared__ typename Scan::TempStorage scan_tmp;
  __shared__ double red[NWARP + 1];

  const int n = s.ncell;
  const int64_t base = (int64_t)blockIdx.x * n;
  const T* __restrict__ g = g_all + base;
  const T* __restrict__ src = src_all + base;
  const T* __restrict__ gnd = gnd_all + base;
  double* __restrict__ cur = cur_all + base;
  double* __restrict__ volt = volt_all ? volt_all + base : nullptr;
  double* __restrict__ X = vec_all + (int64_t)blockIdx.x * NVEC * n;
  double* __restrict__ R = X + n;
  double* __restrict__ P = R + n;
  double* __restrict__ Q = P + n;
  double* __restrict__ D = Q + n;      // diagonal of the reduced operator; 0 = not an unknown
  int* lab = lab_all + base;            // read and hooked concurrently: no __restrict__
  int* __restrict__ flag = flag_all + base;
  int* __restrict__ list = list_all + base;
  volatile int* vlab = lab;

  // 1. valid cells, outputs zeroed
  for (int i = threadIdx.x; i < n; i += BT) {
    lab[i] = (double)g[i] > 0.0 ? i : -1;
    flag[i] = 0;
    cur[i] = 0.0;
    if (volt) volt[i] = 0.0;
  }
  __syncthreads();

  // 3. component labels.  Hook the larger of two roots under the smaller (labels only decrease and
  // always point to a smaller cell, so there are no cycles and the final root is the component's
  // smallest cell), then compress every path; repeat until a pass sees no edge between two trees.
  for (;;) {
    int changed = 0;
    for (int i = threadIdx.x; i < n; i += BT) {
      if (lab[i] < 0) continue;
      for_nbrs<true>(s, g, i, [&](int j, double, bool) {
        const int ri = find_root(vlab, i), rj = find_root(vlab, j);
        if (ri != rj) {
          atomicMin(&lab[max(ri, rj)], min(ri, rj));
          changed = 1;
        }
      });
    }
    changed = __syncthreads_or(changed);
    for (int i = threadIdx.x; i < n; i += BT)
      if (lab[i] >= 0) vlab[i] = find_root(vlab, i);
    __syncthreads();
    if (!changed) break;
  }

  // 2 + 4. after rmvsrc: flag every root whose component has a nonzero source (1) / ground (2)
  for (int i = threadIdx.x; i < n; i += BT) {
    const int root = lab[i];
    if (root < 0) continue;
    const double si = (double)src[i], gi = (double)gnd[i];
    int f = 0;
    if (node_source(si, gi) != 0.0) f |= 1;
    if (node_ground(si, gi) != 0.0) f |= 2;
    if (f) atomicOr(&flag[root], f);
  }
  __syncthreads();

  // candidate roots in ascending cell order
  int ncand = 0;
  for (int b0 = 0; b0 < n; b0 += BT) {
    const int i = b0 + threadIdx.x;
    const int is = (i < n && lab[i] == i && flag[i] == 3) ? 1 : 0;
    int pos, total;
    Scan(scan_tmp).ExclusiveSum(is, pos, total);
    if (is) list[ncand + pos] = i;
    ncand += total;
    __syncthreads();
  }

  WinOut wo{0.0, 0.0, 0, 0, WIN_OK};
  for (int ci = 0; ci < ncand; ++ci) {
    const int root = list[ci];
    // 4. the exact rule of src/raster/advanced.jl:194-196 on the component's own sums
    double ss = 0.0, gs = 0.0;
    for (int i = threadIdx.x; i < n; i += BT) {
      if (lab[i] != root) continue;
      const double si = (double)src[i], gi = (double)gnd[i];
      ss += node_source(si, gi);
      gs += node_ground(si, gi);
    }
    ss = block_sum(ss, red);
    gs = block_sum(gs, red);
    if (ss == 0.0 || gs == 0.0) continue;
    // multiple_solver adds the finite grounds unless the component's first entry is the NODATA
    // sentinel (src/raster/advanced.jl:284-285); the first node is the root cell
    const bool use_fin = node_finite((double)gnd[root]) != kNodata;

    // 5. reduced system: unknowns = the component's cells that are not Inf grounds
    double rz = 0.0, bb = 0.0;
    for (int i = threadIdx.x; i < n; i += BT) {
      double d = 0.0, b = 0.0;
      const double gi = (double)g[i], grd = (double)gnd[i];
      if (lab[i] == root && !(grd == INFINITY)) {
        for_nbrs<false>(s, g, i, [&](int, double gj, bool dg) { d += ras::weight(gi, gj, dg, false); });
        if (use_fin) d += node_finite(grd);
        b = node_source((double)src[i], grd);
      }
      const double z = d != 0.0 ? b / d : 0.0;
      D[i] = d;
      X[i] = 0.0;
      R[i] = b;
      P[i] = z;
      rz += b * z;
      bb += b * b;
    }
    rz = block_sum(rz, red);
    bb = block_sum(bb, red);
    const double tol = atol + rtol * sqrt(rz);
    long long it = 0;
    bool active = rz > 0.0 && sqrt(rz) > tol && itmax > 0;
    while (active) {
      double pq = 0.0;
      for (int i = threadIdx.x; i < n; i += BT) {
        const double d = D[i];
        if (d == 0.0) continue;
        const double gi = (double)g[i];
        double q = d * P[i];
        for_nbrs<false>(s, g, i, [&](int j, double gj, bool dg) { q -= ras::weight(gi, gj, dg, false) * P[j]; });
        Q[i] = q;
        pq += P[i] * q;
      }
      const double alpha = rz / block_sum(pq, red);
      double rn = 0.0;
      for (int i = threadIdx.x; i < n; i += BT) {
        const double d = D[i];
        if (d == 0.0) continue;
        X[i] += alpha * P[i];
        const double r = R[i] - alpha * Q[i];
        R[i] = r;
        rn += r * (r / d);
      }
      rn = block_sum(rn, red);
      ++it;
      if (!(sqrt(rn) > tol) || it >= itmax) {
        active = false;
        rz = rn;
        break;
      }
      const double beta = rn / rz;
      rz = rn;
      for (int i = threadIdx.x; i < n; i += BT) {
        const double d = D[i];
        if (d != 0.0) P[i] = R[i] / d + beta * P[i];
      }
      __syncthreads();
    }

    // 6. true residual of the reduced system
    double rr = 0.0;
    for (int i = threadIdx.x; i < n; i += BT) {
      const double d = D[i];
      if (d == 0.0) continue;
      const double gi = (double)g[i];
      double ax = d * X[i];
      for_nbrs<false>(s, g, i, [&](int j, double gj, bool dg) { ax -= ras::weight(gi, gj, dg, false) * X[j]; });
      const double res = node_source((double)src[i], (double)gnd[i]) - ax;
      rr += res * res;
    }
    rr = block_sum(rr, red);
    const double relres = bb > 0.0 ? sqrt(rr / bb) : 0.0;
    wo.iters += it;
    wo.relres = dmax(wo.relres, relres);
    int st = WIN_OK;
    if (!(relres < kGate)) st = WIN_RESIDUAL;
    else if (it >= itmax && sqrt(rz) > tol) st = WIN_MAXITER;
    if (st > wo.status) {
      wo.status = st;
      wo.fail_relres = relres;
      wo.fail_iters = (int)min(it, (long long)INT_MAX);
    }

    // 7. node currents (src/out.jl:178-207): branch currents e = w (v_lo - v_hi) over the edges
    // lo < hi, cut at 1e-8 of the component's max of e (inflow) and of -e (outflow) separately
    double mp = -INFINITY, mq = -INFINITY;
    for (int i = threadIdx.x; i < n; i += BT) {
      if (lab[i] != root) continue;
      const double gi = (double)g[i], vi = X[i];
      for_nbrs<true>(s, g, i, [&](int j, double gj, bool dg) {
        const double e = ras::weight(gi, gj, dg, false) * (vi - X[j]);
        mp = dmax(mp, e);
        mq = dmax(mq, -e);
      });
    }
    mp = block_max(mp, red);
    mq = block_max(mq, red);
    for (int i = threadIdx.x; i < n; i += BT) {
      if (lab[i] != root) continue;
      const double gi = (double)g[i], vi = X[i];
      double in = 0.0, outf = 0.0;
      for_nbrs<false>(s, g, i, [&](int j, double gj, bool dg) {
        const double w = ras::weight(gi, gj, dg, false);
        const double e = j > i ? w * (vi - X[j]) : w * (X[j] - vi);
        const double ep = cut(e, mp), eq = cut(-e, mq);
        if (j < i) { in += ep > 0.0 ? ep : 0.0; outf += eq > 0.0 ? eq : 0.0; }
        else       { in += -ep > 0.0 ? -ep : 0.0; outf += -eq > 0.0 ? -eq : 0.0; }
      });
      if (use_fin) {
        const double fg = node_finite((double)gnd[i]) * vi;
        in += fg < 0.0 ? -fg : 0.0;
        outf += fg > 0.0 ? fg : 0.0;
      }
      cur[i] = in > outf ? in : outf;
      if (volt) volt[i] = vi;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) out[blockIdx.x] = wo;
}

template <typename T>
cudaError_t launch(int nwin, Shape s, const void* g, const void* src, const void* gnd, double rtol, double atol,
                   long long itmax, double* cur, double* volt, double* vec, int* lab, int* flag, int* list,
                   WinOut* out, cudaStream_t st) {
  k_advanced_batch<T><<<nwin, BT, 0, st>>>(s, (const T*)g, (const T*)src, (const T*)gnd, rtol, atol, itmax, cur,
                                           volt, vec, lab, flag, list, out);
  return cudaGetLastError();
}

size_t align256(size_t b) { return (b + 255) / 256 * 256; }

// ---------------------------------------------------------------------------------------------------
// Moving windows cut from one resident landscape (cs_b200_solve_moving_windows).  Per batch of
// consecutive windows: k_window_cut writes the g / src / gnd stacks k_advanced_batch reads, the batch
// is solved, and k_window_accumulate adds the staged currents into the landscape map.  The map is
// split into TILE x TILE tiles; each tile is one CTA that owns its cells and adds the windows touching
// it in window order, from lists built expand - sort - compress: every window writes (tile, window)
// for the tiles its square overlaps (k_window_tiles), a stable radix sort by tile keeps window order
// inside a tile, and k_tile_bounds marks where each tile's run starts and ends.  The map stays on the
// device across batches and each cell is one fixed chain of fp64 adds from +0.0, so the result does
// not depend on the batch split.  cs_b200_solve_omniscape runs the same loop: k_block_targets and a cub
// select find the targets first, k_window_cut's Omniscape modes normalise each window's sources (and cut
// a flow-potential window beside each conductance window), the tile lists serve both maps, and
// k_omniscape_finish writes the normalised map and the NODATA mask.
// ---------------------------------------------------------------------------------------------------
constexpr int TILE = 32;
constexpr int TILE_COLS = BT / TILE;            // tile columns one CTA pass covers
constexpr int TILE_PASSES = TILE / TILE_COLS;   // cells per thread

struct Land {
  int nrows, ncols;    // landscape, column-major
  int radius, side;    // side = 2 radius + 1
  int circular;
  int tiles_r, ntiles; // tiles down a column, tiles in all
  int span;            // most tiles a window overlaps along one axis
};

// What k_window_cut writes.  CUT_WINDOW: the window of cs_b200_solve_moving_windows (per-window scale and
// ground).  CUT_OMNI: Omniscape's conductance window -- sources s' outside the target's block, scaled to
// sum to the target's amps (the scale is reduced here and stored per target), a direct ground at the
// centre.  CUT_FLOW: the flow-potential window of the same target -- g = 1 on every landscape cell in the
// square (and disc), the CUT_OMNI sources (its stored scale), a direct ground at the centre.
enum CutMode { CUT_WINDOW = 0, CUT_OMNI = 1, CUT_FLOW = 2 };

struct BlockRule {          // Omniscape's source rule (CUT_OMNI, CUT_FLOW)
  double theta;             // source threshold
  int half;                 // (block size - 1) / 2
  const double* amps;       // per target
  double* scale;            // per target: written by CUT_OMNI, read by CUT_FLOW
};

// effective source strength s' of a landscape cell: s where s > theta, s is finite and g > 0, else 0
template <typename T>
__device__ __forceinline__ double eff_strength(T s, T g, double theta) {
  const double sd = (double)s;
  return (sd > theta && isfinite(sd) && (double)g > 0.0) ? sd : 0.0;
}

// window w's g / src / gnd in k_advanced_batch's layout (window-major, column-major inside)
template <int MODE, typename T>
__global__ void __launch_bounds__(BT)
k_window_cut(Land L, int w0, const T* __restrict__ G, const T* __restrict__ S, const int* __restrict__ trow,
             const int* __restrict__ tcol, const double* __restrict__ scale, const double* __restrict__ gnd,
             BlockRule br, T* __restrict__ g_all, T* __restrict__ src_all, T* __restrict__ gnd_all) {
  const int w = w0 + blockIdx.x, R = L.radius, W = L.side, n = W * W;
  const int r0 = trow[w] - R, c0 = tcol[w] - R;
  double sc;
  if constexpr (MODE == CUT_WINDOW) {
    sc = scale ? scale[w] : 1.0;
  } else if constexpr (MODE == CUT_FLOW) {
    sc = br.scale[w];
  } else {
    // the window's source sum: s' over the landscape cells in the disc outside the target's block, a
    // strided fp64 partial per thread, then the fixed-order CTA tree
    __shared__ double red[NWARP + 1];
    double part = 0.0;
    for (int i = threadIdx.x; i < n; i += BT) {
      const int dr = i % W - R, dc = i / W - R, r = r0 + R + dr, c = c0 + R + dc;
      if (r >= 0 && r < L.nrows && c >= 0 && c < L.ncols && (!L.circular || dr * dr + dc * dc <= R * R) &&
          (abs(dr) > br.half || abs(dc) > br.half)) {
        const int64_t j = (int64_t)c * L.nrows + r;
        part += eff_strength(S[j], G[j], br.theta);
      }
    }
    const double sum = block_sum(part, red);
    sc = sum > 0.0 ? br.amps[w] / sum : 0.0;
    if (threadIdx.x == 0) br.scale[w] = sc;
  }
  const T gc = MODE == CUT_WINDOW && gnd ? (T)gnd[w] : (T)INFINITY;
  const int64_t base = (int64_t)blockIdx.x * n;
  for (int i = threadIdx.x; i < n; i += BT) {
    const int dr = i % W - R, dc = i / W - R, r = r0 + R + dr, c = c0 + R + dc;
    T gv = 0, sv = 0, nv = 0;
    if (r >= 0 && r < L.nrows && c >= 0 && c < L.ncols && (!L.circular || dr * dr + dc * dc <= R * R)) {
      const int64_t j = (int64_t)c * L.nrows + r;
      const T gl = G[j];
      if constexpr (MODE == CUT_WINDOW) {
        if ((double)gl > 0.0) {
          gv = gl;
          sv = (T)(sc * (double)S[j]);
          if (dr == 0 && dc == 0) nv = gc;
        }
      } else if (MODE == CUT_FLOW || (double)gl > 0.0) {
        gv = MODE == CUT_FLOW ? (T)1 : gl;
        if (abs(dr) > br.half || abs(dc) > br.half) sv = (T)(sc * eff_strength(S[j], gl, br.theta));
        if (dr == 0 && dc == 0) nv = gc;
      }
    }
    g_all[base + i] = gv;
    src_all[base + i] = sv;
    gnd_all[base + i] = nv;
  }
}

// Omniscape's targets: one thread per block centre (candidate k = i + j * ni, block-column-major), the
// amps summed sequentially in fp64 over the block clipped to the landscape, column outer, row inner
template <typename T>
__global__ void k_block_targets(int nrows, int ncols, int bsz, int ni, int ncand, double theta,
                                const T* __restrict__ G, const T* __restrict__ S, int* __restrict__ crow,
                                int* __restrict__ ccol, double* __restrict__ camps, char* __restrict__ flag) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= ncand) return;
  const int half = (bsz - 1) / 2, tr = half + (k % ni) * bsz, tc = half + (k / ni) * bsz;
  const int r1 = min(tr + half, nrows - 1), c1 = min(tc + half, ncols - 1);
  double a = 0.0;
  for (int c = tc - half; c <= c1; ++c)
    for (int r = tr - half; r <= r1; ++r) {
      const int64_t j = (int64_t)c * nrows + r;
      a += eff_strength(S[j], G[j], theta);
    }
  crow[k] = tr;
  ccol[k] = tc;
  camps[k] = a;
  flag[k] = a > 0.0 ? 1 : 0;
}

// the returned maps: normalized = fp > 0 ? cum / fp : 0, then NODATA (-9999) in every map where g is NaN
// or -9999; fp and norm are null without flow potential
template <typename T>
__global__ void k_omniscape_finish(int64_t cells, const T* __restrict__ G, double* __restrict__ cum,
                                   double* __restrict__ fp, double* __restrict__ norm) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= cells) return;
  const double g = (double)G[i];
  const bool mask = isnan(g) || g == kNodata;
  if (fp) {
    const double f = fp[i];
    norm[i] = mask ? kNodata : (f > 0.0 ? cum[i] / f : 0.0);
    if (mask) fp[i] = kNodata;
  }
  if (mask) cum[i] = kNodata;
}

// (tile, window-in-batch) for every tile window w0 + wl overlaps; span^2 slots per window, the unused
// ones keyed ntiles so that they sort behind every tile
__global__ void k_window_tiles(Land L, int w0, int nb, const int* __restrict__ trow, const int* __restrict__ tcol,
                               unsigned* __restrict__ key, int* __restrict__ val) {
  const int per = L.span * L.span;
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= (int64_t)nb * per) return;
  const int wl = (int)(p / per), k = (int)(p % per), w = w0 + wl;
  const int r0 = max(trow[w] - L.radius, 0), r1 = min(trow[w] + L.radius, L.nrows - 1);
  const int c0 = max(tcol[w] - L.radius, 0), c1 = min(tcol[w] + L.radius, L.ncols - 1);
  const int ti = r0 / TILE + k % L.span, tj = c0 / TILE + k / L.span;
  key[p] = (ti <= r1 / TILE && tj <= c1 / TILE) ? (unsigned)(ti + tj * L.tiles_r) : (unsigned)L.ntiles;
  val[p] = wl;
}

// run [beg[t], end[t]) of tile t in the sorted pairs (beg = end = 0 for a tile no window touches)
__global__ void k_tile_bounds(int np, const unsigned* __restrict__ key, unsigned ntiles, int* __restrict__ beg,
                              int* __restrict__ end) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= np) return;
  const unsigned k = key[i];
  if (k >= ntiles) return;
  if (i == 0 || key[i - 1] != k) beg[k] = i;
  if (i == np - 1 || key[i + 1] != k) end[k] = i + 1;
}

// one CTA per tile: each thread owns TILE_PASSES cells of the tile and adds the staged window currents
// of the tile's windows in window order
__global__ void __launch_bounds__(BT)
k_window_accumulate(Land L, int w0, const int* __restrict__ trow, const int* __restrict__ tcol,
                    const int* __restrict__ beg, const int* __restrict__ end, const int* __restrict__ wins,
                    const double* __restrict__ cur_all, double* __restrict__ cum) {
  const int t = blockIdx.x, b = beg[t], e = end[t];
  if (b == e) return;
  const int W = L.side, n = W * W;
  const int r = (t % L.tiles_r) * TILE + threadIdx.x % TILE;
  const int cbase = (t / L.tiles_r) * TILE + threadIdx.x / TILE;
  const bool rin = r < L.nrows;
  double acc[TILE_PASSES];
#pragma unroll
  for (int k = 0; k < TILE_PASSES; ++k) {
    const int c = cbase + k * TILE_COLS;
    acc[k] = rin && c < L.ncols ? cum[(int64_t)c * L.nrows + r] : 0.0;
  }
  for (int q = b; q < e; ++q) {
    const int wl = wins[q], w = w0 + wl;
    const int dr = r - (trow[w] - L.radius), dc0 = cbase - (tcol[w] - L.radius);
    const double* __restrict__ cur = cur_all + (int64_t)wl * n;
#pragma unroll
    for (int k = 0; k < TILE_PASSES; ++k) {
      const int dc = dc0 + k * TILE_COLS;
      if (rin && cbase + k * TILE_COLS < L.ncols && dr >= 0 && dr < W && dc >= 0 && dc < W)
        acc[k] += cur[dr + dc * W];
    }
  }
#pragma unroll
  for (int k = 0; k < TILE_PASSES; ++k) {
    const int c = cbase + k * TILE_COLS;
    if (rin && c < L.ncols) cum[(int64_t)c * L.nrows + r] = acc[k];
  }
}

// device buffers of one call, freed when it returns
struct DevBufs {
  std::vector<void*> ptrs;
  ~DevBufs() {
    for (void* q : ptrs) cudaFree(q);
  }
  template <typename X>
  cudaError_t get(X** out, size_t count) {
    void* q = nullptr;
    const cudaError_t e = cudaMalloc(&q, count ? count * sizeof(X) : 1);
    if (e == cudaSuccess) ptrs.push_back(q);
    *out = (X*)q;
    return e;
  }
};

struct Stream {
  cudaStream_t s = nullptr;
  ~Stream() {
    if (s) cudaStreamDestroy(s);
  }
};

#define CKM(call)                                                                                \
  do {                                                                                           \
    cudaError_t _e = (call);                                                                     \
    if (_e != cudaSuccess)                                                                       \
      return set_err(CS_B200_ERR_CUDA, "CUDA error %s at %s:%d (%s)", cudaGetErrorString(_e), \
                     __FILE__, __LINE__, #call);                                                 \
  } while (0)

// Omniscape's block rule and flow potential on top of the moving-window loop (cs_b200_solve_omniscape)
struct OmniJob {
  int bsz;                      // block size (odd)
  double theta;                 // source threshold
  bool flow;                    // also cut, solve and accumulate the flow-potential window of every target
  double *fp, *norm;            // host maps (flow only)
  std::vector<double> amps, scale;   // per target, filled by the call
  std::vector<WinOut> wo_fp;         // per target's flow-potential window, filled by the call
};

// the batches of cs_b200_solve_moving_windows (om null: trow / tcol are the targets) and of
// cs_b200_solve_omniscape (om set: trow / tcol receive the targets found on the device).  Batches are as
// many targets as fit `budget` at `per` bytes per window, every window of a target counted; wo receives
// every (conductance) window's WinOut.
template <typename T>
int moving_windows(const Land& L, size_t budget, size_t per_win, const void* g, const void* src,
                   std::vector<int>& trow, std::vector<int>& tcol, const double* scale, const double* gnd, int four,
                   double rtol, long long itmax, double* cum, std::vector<WinOut>& wo, OmniJob* om) {
  const size_t cells = (size_t)L.nrows * L.ncols, ncell = (size_t)L.side * L.side, per = (size_t)L.span * L.span;
  const Shape s{L.side, L.side, (int)ncell, four};
  const double atol = std::sqrt(2.220446049250313e-16);   // sqrt(eps(Float64)), as cs_b200_solve_advanced_batch
  const int kinds = om && om->flow ? 2 : 1;               // windows per target
  int nbits = 1;
  while (nbits < 32 && (1ull << nbits) <= (unsigned long long)L.ntiles) ++nbits;   // keys 0 .. ntiles
  Stream st;
  DevBufs d;
  T *dG, *dS, *wg, *ws, *wn;
  double *dcum, *dfp = nullptr, *dnorm = nullptr, *dscale = nullptr, *dgnd = nullptr, *damps = nullptr, *wcur, *wvec;
  int *dtr, *dtc, *wlab, *wflag, *wlist, *val_in, *val_out, *beg, *end;
  unsigned *key_in, *key_out;
  WinOut* dout;
  unsigned char* tmp = nullptr;
  size_t tmp_bytes = 0;
  CKM(cudaStreamCreateWithFlags(&st.s, cudaStreamNonBlocking));
  CKM(d.get(&dG, cells));
  CKM(d.get(&dS, cells));
  CKM(d.get(&dcum, cells));
  if (kinds == 2) {
    CKM(d.get(&dfp, cells));
    CKM(d.get(&dnorm, cells));
  }
  CKM(cudaMemcpyAsync(dG, g, cells * sizeof(T), cudaMemcpyHostToDevice, st.s));
  CKM(cudaMemcpyAsync(dS, src, cells * sizeof(T), cudaMemcpyHostToDevice, st.s));
  CKM(cudaMemsetAsync(dcum, 0, cells * sizeof(double), st.s));
  if (dfp) CKM(cudaMemsetAsync(dfp, 0, cells * sizeof(double), st.s));

  int nwin = (int)trow.size();
  if (!om) {
    CKM(d.get(&dtr, (size_t)nwin));
    CKM(d.get(&dtc, (size_t)nwin));
    if (scale) CKM(d.get(&dscale, (size_t)nwin));
    if (gnd) CKM(d.get(&dgnd, (size_t)nwin));
    CKM(cudaMemcpyAsync(dtr, trow.data(), (size_t)nwin * sizeof(int), cudaMemcpyHostToDevice, st.s));
    CKM(cudaMemcpyAsync(dtc, tcol.data(), (size_t)nwin * sizeof(int), cudaMemcpyHostToDevice, st.s));
    if (scale) CKM(cudaMemcpyAsync(dscale, scale, (size_t)nwin * sizeof(double), cudaMemcpyHostToDevice, st.s));
    if (gnd) CKM(cudaMemcpyAsync(dgnd, gnd, (size_t)nwin * sizeof(double), cudaMemcpyHostToDevice, st.s));
  } else {
    // the block centres, then the ones with amps > 0 compacted in candidate order
    const int half = (om->bsz - 1) / 2;
    const int ni = L.nrows > half ? (L.nrows - 1 - half) / om->bsz + 1 : 0;
    const int nj = L.ncols > half ? (L.ncols - 1 - half) / om->bsz + 1 : 0;
    const int ncand = ni * nj;
    int *crow, *ccol, *dnum;
    double* camps;
    char* cflag;
    CKM(d.get(&crow, (size_t)ncand));
    CKM(d.get(&ccol, (size_t)ncand));
    CKM(d.get(&camps, (size_t)ncand));
    CKM(d.get(&cflag, (size_t)ncand));
    CKM(d.get(&dtr, (size_t)ncand));
    CKM(d.get(&dtc, (size_t)ncand));
    CKM(d.get(&damps, (size_t)ncand));
    CKM(d.get(&dscale, (size_t)ncand));
    CKM(d.get(&dnum, 1));
    size_t sel_i = 0, sel_d = 0;
    CKM(cub::DeviceSelect::Flagged(nullptr, sel_i, crow, cflag, dtr, dnum, ncand, st.s));
    CKM(cub::DeviceSelect::Flagged(nullptr, sel_d, camps, cflag, damps, dnum, ncand, st.s));
    unsigned char* sel_tmp;
    CKM(d.get(&sel_tmp, std::max(sel_i, sel_d)));
    int nt = 0;
    if (ncand > 0) {
      k_block_targets<T><<<(ncand + BT - 1) / BT, BT, 0, st.s>>>(L.nrows, L.ncols, om->bsz, ni, ncand, om->theta, dG,
                                                                 dS, crow, ccol, camps, cflag);
      CKM(cudaGetLastError());
      CKM(cub::DeviceSelect::Flagged(sel_tmp, sel_i, crow, cflag, dtr, dnum, ncand, st.s));
      CKM(cub::DeviceSelect::Flagged(sel_tmp, sel_i, ccol, cflag, dtc, dnum, ncand, st.s));
      CKM(cub::DeviceSelect::Flagged(sel_tmp, sel_d, camps, cflag, damps, dnum, ncand, st.s));
      CKM(cudaMemcpyAsync(&nt, dnum, sizeof(int), cudaMemcpyDeviceToHost, st.s));
      CKM(cudaStreamSynchronize(st.s));
    }
    nwin = nt;
    trow.resize((size_t)nt);
    tcol.resize((size_t)nt);
    om->amps.resize((size_t)nt);
    om->scale.resize((size_t)nt);
    wo.resize((size_t)nt);
    om->wo_fp.resize((size_t)nt);
    CKM(cudaMemcpyAsync(trow.data(), dtr, (size_t)nt * sizeof(int), cudaMemcpyDeviceToHost, st.s));
    CKM(cudaMemcpyAsync(tcol.data(), dtc, (size_t)nt * sizeof(int), cudaMemcpyDeviceToHost, st.s));
    CKM(cudaMemcpyAsync(om->amps.data(), damps, (size_t)nt * sizeof(double), cudaMemcpyDeviceToHost, st.s));
  }

  // targets per batch
  const int bw = (int)std::max<size_t>(1, std::min({budget / (per_win * kinds), (size_t)nwin, INT_MAX / per}));
  CKM(d.get(&wg, kinds * bw * ncell));
  CKM(d.get(&ws, kinds * bw * ncell));
  CKM(d.get(&wn, kinds * bw * ncell));
  CKM(d.get(&wcur, kinds * bw * ncell));
  CKM(d.get(&wvec, kinds * bw * ncell * NVEC));
  CKM(d.get(&wlab, kinds * bw * ncell));
  CKM(d.get(&wflag, kinds * bw * ncell));
  CKM(d.get(&wlist, kinds * bw * ncell));
  CKM(d.get(&dout, (size_t)(kinds * bw)));
  CKM(d.get(&key_in, bw * per));
  CKM(d.get(&key_out, bw * per));
  CKM(d.get(&val_in, bw * per));
  CKM(d.get(&val_out, bw * per));
  CKM(d.get(&beg, (size_t)L.ntiles));
  CKM(d.get(&end, (size_t)L.ntiles));
  CKM(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, key_in, key_out, val_in, val_out, (int)(bw * per), 0,
                                      nbits, st.s));
  CKM(d.get(&tmp, tmp_bytes));

  const BlockRule br{om ? om->theta : 0.0, om ? (om->bsz - 1) / 2 : 0, damps, dscale};
  for (int w0 = 0; w0 < nwin; w0 += bw) {
    const int nb = std::min(bw, nwin - w0), np = (int)(nb * per);
    const size_t second = (size_t)nb * ncell;   // the flow-potential windows follow the batch's conductance windows
    if (!om) {
      k_window_cut<CUT_WINDOW, T><<<nb, BT, 0, st.s>>>(L, w0, dG, dS, dtr, dtc, dscale, dgnd, br, wg, ws, wn);
    } else {
      k_window_cut<CUT_OMNI, T><<<nb, BT, 0, st.s>>>(L, w0, dG, dS, dtr, dtc, nullptr, nullptr, br, wg, ws, wn);
      if (kinds == 2) {
        CKM(cudaGetLastError());
        k_window_cut<CUT_FLOW, T><<<nb, BT, 0, st.s>>>(L, w0, dG, dS, dtr, dtc, nullptr, nullptr, br, wg + second,
                                                       ws + second, wn + second);
      }
    }
    CKM(cudaGetLastError());
    CKM((launch<T>(kinds * nb, s, wg, ws, wn, rtol, atol, itmax, wcur, nullptr, wvec, wlab, wflag, wlist, dout,
                   st.s)));
    k_window_tiles<<<(np + BT - 1) / BT, BT, 0, st.s>>>(L, w0, nb, dtr, dtc, key_in, val_in);
    CKM(cudaGetLastError());
    size_t tb = tmp_bytes;
    CKM(cub::DeviceRadixSort::SortPairs(tmp, tb, key_in, key_out, val_in, val_out, np, 0, nbits, st.s));
    CKM(cudaMemsetAsync(beg, 0, (size_t)L.ntiles * sizeof(int), st.s));
    CKM(cudaMemsetAsync(end, 0, (size_t)L.ntiles * sizeof(int), st.s));
    k_tile_bounds<<<(np + BT - 1) / BT, BT, 0, st.s>>>(np, key_out, (unsigned)L.ntiles, beg, end);
    CKM(cudaGetLastError());
    k_window_accumulate<<<L.ntiles, BT, 0, st.s>>>(L, w0, dtr, dtc, beg, end, val_out, wcur, dcum);
    CKM(cudaGetLastError());
    CKM(cudaMemcpyAsync(wo.data() + w0, dout, (size_t)nb * sizeof(WinOut), cudaMemcpyDeviceToHost, st.s));
    if (kinds == 2) {   // the same tile lists place the flow-potential windows
      k_window_accumulate<<<L.ntiles, BT, 0, st.s>>>(L, w0, dtr, dtc, beg, end, val_out, wcur + second, dfp);
      CKM(cudaGetLastError());
      CKM(cudaMemcpyAsync(om->wo_fp.data() + w0, dout + nb, (size_t)nb * sizeof(WinOut), cudaMemcpyDeviceToHost,
                          st.s));
    }
  }
  if (om) {
    k_omniscape_finish<T><<<(unsigned)((cells + BT - 1) / BT), BT, 0, st.s>>>((int64_t)cells, dG, dcum, dfp, dnorm);
    CKM(cudaGetLastError());
    CKM(cudaMemcpyAsync(om->scale.data(), dscale, (size_t)nwin * sizeof(double), cudaMemcpyDeviceToHost, st.s));
    if (dfp) {
      CKM(cudaMemcpyAsync(om->fp, dfp, cells * sizeof(double), cudaMemcpyDeviceToHost, st.s));
      CKM(cudaMemcpyAsync(om->norm, dnorm, cells * sizeof(double), cudaMemcpyDeviceToHost, st.s));
    }
  }
  CKM(cudaMemcpyAsync(cum, dcum, cells * sizeof(double), cudaMemcpyDeviceToHost, st.s));
  CKM(cudaStreamSynchronize(st.s));
  return CS_B200_OK;
}

// the Land of a landscape and radius (tile grid and the most tiles a window overlaps along one axis)
Land make_land(int64_t nrows, int64_t ncols, int64_t radius, int circular) {
  Land L;
  L.nrows = (int)nrows;
  L.ncols = (int)ncols;
  L.radius = (int)radius;
  L.side = 2 * L.radius + 1;
  L.circular = circular ? 1 : 0;
  L.tiles_r = (L.nrows + TILE - 1) / TILE;
  L.ntiles = L.tiles_r * ((L.ncols + TILE - 1) / TILE);
  L.span = std::min((L.side + TILE - 1) / TILE + 1, std::max(L.tiles_r, L.ntiles / L.tiles_r));
  return L;
}

// device bytes of one window's stack, solver.advanced_batch_bytes(ncell, itemsize, False): the inputs,
// the current raster, NVEC fp64 CG vectors, three int32 label arrays and its WinOut
size_t window_bytes(const Land& L, int dtype) {
  const size_t isz = dtype == CS_B200_F64 ? 8 : 4, ncell = (size_t)L.side * L.side;
  return ncell * (3 * isz + 8 + NVEC * 8 + 3 * 4) + sizeof(WinOut);
}

}  // namespace

#define CKB(call)                                                                              \
  do {                                                                                         \
    cudaError_t _e = (call);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      rc = set_err(CS_B200_ERR_CUDA, "CUDA error %s at %s:%d (%s)", cudaGetErrorString(_e), \
                   __FILE__, __LINE__, #call);                                                 \
      goto done;                                                                               \
    }                                                                                          \
  } while (0)

extern "C" int cs_b200_solve_advanced_batch(int64_t nwin, int64_t nrows, int64_t ncols, const void* g,
                                            const void* src, const void* gnd, int dtype, int four_neighbors,
                                            int device, double rtol, int64_t itmax, void* cur, void* volt,
                                            int64_t* iters, double* relres, int64_t* first_failed) {
  if (first_failed) *first_failed = -1;
  if (nwin < 0 || nrows < 1 || ncols < 1)
    return set_err(CS_B200_ERR_ARG, "bad batch shape (nwin=%lld nrows=%lld ncols=%lld)",
                   (long long)nwin, (long long)nrows, (long long)ncols);
  if (nrows > INT_MAX / ncols || nwin > INT_MAX)
    return set_err(CS_B200_ERR_ARG, "batch too large (nwin=%lld, %lld x %lld cells per window)",
                   (long long)nwin, (long long)nrows, (long long)ncols);
  if (dtype != CS_B200_F32 && dtype != CS_B200_F64) return set_err(CS_B200_ERR_ARG, "bad dtype %d", dtype);
  if (!(rtol >= 0.0) || itmax < 0)
    return set_err(CS_B200_ERR_ARG, "bad rtol %g / itmax %lld", rtol, (long long)itmax);
  if (nwin > 0 && (!g || !src || !gnd || !cur))
    return set_err(CS_B200_ERR_ARG, "g, src, gnd and cur must not be NULL");
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return set_err(CS_B200_ERR_CUDA, "no CUDA device available (%s): libcsb200 has no CPU fallback",
                   cudaGetErrorString(e));
  if (device < 0 || device >= ndev)
    return set_err(CS_B200_ERR_ARG, "device %d out of range (0..%d)", device, ndev - 1);
  if (nwin == 0) return CS_B200_OK;

  int rc = CS_B200_OK;
  const Shape s{(int)nrows, (int)ncols, (int)(nrows * ncols), four_neighbors ? 1 : 0};
  const size_t cells = (size_t)nwin * s.ncell;
  const size_t isz = dtype == CS_B200_F64 ? 8 : 4;
  const size_t b_in = align256(cells * isz), b_out = align256(cells * 8), b_vec = align256(cells * 8 * NVEC),
               b_int = align256(cells * 4), b_win = align256((size_t)nwin * sizeof(WinOut));
  unsigned char* dbuf = nullptr;
  cudaStream_t st = nullptr;
  std::vector<WinOut> wo((size_t)nwin);
  const long long itm = (long long)itmax;
  const double atol = std::sqrt(2.220446049250313e-16);   // sqrt(eps(Float64)), Krylov.jl's default
  double *d_cur, *d_volt, *d_vec;
  int *d_lab, *d_flag, *d_list;
  WinOut* d_out;
  unsigned char* p;
  int64_t bad = -1;
  int worst = WIN_OK;

  CKB(cudaSetDevice(device));
  CKB(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  CKB(cudaMalloc(&dbuf, 3 * b_in + 2 * b_out + b_vec + 3 * b_int + b_win));
  p = dbuf + 3 * b_in;
  d_cur = (double*)p;   p += b_out;
  d_volt = volt ? (double*)p : nullptr; p += b_out;
  d_vec = (double*)p;   p += b_vec;
  d_lab = (int*)p;      p += b_int;
  d_flag = (int*)p;     p += b_int;
  d_list = (int*)p;     p += b_int;
  d_out = (WinOut*)p;
  CKB(cudaMemcpyAsync(dbuf, g, cells * isz, cudaMemcpyHostToDevice, st));
  CKB(cudaMemcpyAsync(dbuf + b_in, src, cells * isz, cudaMemcpyHostToDevice, st));
  CKB(cudaMemcpyAsync(dbuf + 2 * b_in, gnd, cells * isz, cudaMemcpyHostToDevice, st));
  if (dtype == CS_B200_F64)
    CKB((launch<double>((int)nwin, s, dbuf, dbuf + b_in, dbuf + 2 * b_in, rtol, atol, itm, d_cur, d_volt, d_vec,
                        d_lab, d_flag, d_list, d_out, st)));
  else
    CKB((launch<float>((int)nwin, s, dbuf, dbuf + b_in, dbuf + 2 * b_in, rtol, atol, itm, d_cur, d_volt, d_vec,
                       d_lab, d_flag, d_list, d_out, st)));
  CKB(cudaMemcpyAsync(cur, d_cur, cells * 8, cudaMemcpyDeviceToHost, st));
  if (volt) CKB(cudaMemcpyAsync(volt, d_volt, cells * 8, cudaMemcpyDeviceToHost, st));
  CKB(cudaMemcpyAsync(wo.data(), d_out, (size_t)nwin * sizeof(WinOut), cudaMemcpyDeviceToHost, st));
  CKB(cudaStreamSynchronize(st));

  for (int64_t w = 0; w < nwin; ++w) {
    if (iters) iters[w] = wo[w].iters;
    if (relres) relres[w] = wo[w].relres;
    if (wo[w].status > worst) { worst = wo[w].status; bad = w; }
  }
  if (worst == WIN_RESIDUAL) {
    rc = set_err(CS_B200_ERR_RESIDUAL,
                 "CUDA PCG solver residual %g exceeds tolerance %g for window %lld (%d iterations)",
                 wo[bad].fail_relres, kGate, (long long)bad, wo[bad].fail_iters);
  } else if (worst == WIN_MAXITER) {
    rc = set_err(CS_B200_ERR_MAXITER,
                 "CUDA PCG solver reached itmax = %lld before rtol for window %lld (residual %g)",
                 (long long)itmax, (long long)bad, wo[bad].fail_relres);
  }
  if (first_failed) *first_failed = bad;
done:
  if (dbuf) cudaFree(dbuf);
  if (st) cudaStreamDestroy(st);
  return rc;
}

extern "C" int cs_b200_solve_moving_windows(int64_t nrows, int64_t ncols, const void* g, const void* src, int dtype,
                                            int64_t nwin, const int64_t* target_rows, const int64_t* target_cols,
                                            int64_t radius, int circular, const double* source_scale,
                                            const double* ground, int four_neighbors, int device, double rtol,
                                            int64_t itmax, int64_t max_batch_bytes, double* cum, int64_t* iters,
                                            double* relres, int64_t* first_failed) {
  if (first_failed) *first_failed = -1;
  if (nrows < 1 || ncols < 1 || nrows > INT_MAX / ncols)
    return set_err(CS_B200_ERR_ARG, "bad landscape shape %lld x %lld (at most INT_MAX cells)", (long long)nrows,
                   (long long)ncols);
  if (radius < 0 || 2 * radius + 1 > 46340)   // (2R+1)^2 cells per window must fit an int
    return set_err(CS_B200_ERR_ARG, "bad radius %lld (0 <= radius, (2 radius + 1)^2 <= INT_MAX)", (long long)radius);
  if (nwin < 0 || nwin > INT_MAX) return set_err(CS_B200_ERR_ARG, "bad window count %lld", (long long)nwin);
  if (dtype != CS_B200_F32 && dtype != CS_B200_F64) return set_err(CS_B200_ERR_ARG, "bad dtype %d", dtype);
  if (!(rtol >= 0.0) || itmax < 0)
    return set_err(CS_B200_ERR_ARG, "bad rtol %g / itmax %lld", rtol, (long long)itmax);
  if (max_batch_bytes <= 0) return set_err(CS_B200_ERR_ARG, "bad max_batch_bytes %lld", (long long)max_batch_bytes);
  if (!g || !src || !cum || (nwin > 0 && (!target_rows || !target_cols)))
    return set_err(CS_B200_ERR_ARG, "g, src, cum, target_rows and target_cols must not be NULL");
  std::vector<int> trow((size_t)nwin), tcol((size_t)nwin);
  for (int64_t w = 0; w < nwin; ++w) {
    if (target_rows[w] < 0 || target_rows[w] >= nrows || target_cols[w] < 0 || target_cols[w] >= ncols)
      return set_err(CS_B200_ERR_ARG, "target %lld at (%lld, %lld) outside the %lld x %lld landscape", (long long)w,
                     (long long)target_rows[w], (long long)target_cols[w], (long long)nrows, (long long)ncols);
    if (ground && !(ground[w] > 0.0))
      return set_err(CS_B200_ERR_ARG, "ground[%lld] = %g: target grounds must be > 0 (Inf = direct)", (long long)w,
                     ground[w]);
    if (source_scale && !std::isfinite(source_scale[w]))
      return set_err(CS_B200_ERR_ARG, "source_scale[%lld] = %g is not finite", (long long)w, source_scale[w]);
    trow[w] = (int)target_rows[w];
    tcol[w] = (int)target_cols[w];
  }
  const size_t cells = (size_t)nrows * ncols;
  std::fill(cum, cum + cells, 0.0);
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return set_err(CS_B200_ERR_CUDA, "no CUDA device available (%s): libcsb200 has no CPU fallback",
                   cudaGetErrorString(e));
  if (device < 0 || device >= ndev)
    return set_err(CS_B200_ERR_ARG, "device %d out of range (0..%d)", device, ndev - 1);
  if (nwin == 0) return CS_B200_OK;

  const Land L = make_land(nrows, ncols, radius, circular);
  std::vector<WinOut> wo((size_t)nwin);
  e = cudaSetDevice(device);
  if (e != cudaSuccess) return set_err(CS_B200_ERR_CUDA, "cudaSetDevice(%d): %s", device, cudaGetErrorString(e));
  const int rc = dtype == CS_B200_F64
                     ? moving_windows<double>(L, (size_t)max_batch_bytes, window_bytes(L, dtype), g, src, trow, tcol,
                                              source_scale, ground, four_neighbors ? 1 : 0, rtol, (long long)itmax,
                                              cum, wo, nullptr)
                     : moving_windows<float>(L, (size_t)max_batch_bytes, window_bytes(L, dtype), g, src, trow, tcol,
                                             source_scale, ground, four_neighbors ? 1 : 0, rtol, (long long)itmax,
                                             cum, wo, nullptr);
  if (rc != CS_B200_OK) return rc;

  int64_t bad = -1;
  int worst = WIN_OK;
  for (int64_t w = 0; w < nwin; ++w) {
    if (iters) iters[w] = wo[w].iters;
    if (relres) relres[w] = wo[w].relres;
    if (wo[w].status > worst) { worst = wo[w].status; bad = w; }
  }
  if (first_failed) *first_failed = bad;
  if (worst == WIN_RESIDUAL)
    return set_err(CS_B200_ERR_RESIDUAL,
                   "CUDA PCG solver residual %g exceeds tolerance %g for window %lld (%d iterations)",
                   wo[bad].fail_relres, kGate, (long long)bad, wo[bad].fail_iters);
  if (worst == WIN_MAXITER)
    return set_err(CS_B200_ERR_MAXITER,
                   "CUDA PCG solver reached itmax = %lld before rtol for window %lld (residual %g)",
                   (long long)itmax, (long long)bad, wo[bad].fail_relres);
  return CS_B200_OK;
}

extern "C" int cs_b200_solve_omniscape(int64_t nrows, int64_t ncols, const void* g, const void* src, int dtype,
                                       int64_t radius, int64_t block_size, double source_threshold,
                                       int flow_potential, int four_neighbors, int device, double rtol, int64_t itmax,
                                       int64_t max_batch_bytes, double* cum, double* fp, double* normalized,
                                       int64_t max_targets, int64_t* ntargets, int64_t* target_rows,
                                       int64_t* target_cols, double* amps, double* scale, int64_t* iters,
                                       double* relres, int64_t* fp_iters, double* fp_relres, int64_t* first_failed) {
  if (first_failed) *first_failed = -1;
  if (ntargets) *ntargets = 0;
  if (nrows < 1 || ncols < 1 || nrows > INT_MAX / ncols)
    return set_err(CS_B200_ERR_ARG, "bad landscape shape %lld x %lld (at most INT_MAX cells)", (long long)nrows,
                   (long long)ncols);
  if (radius < 0 || 2 * radius + 1 > 46340)   // (2R+1)^2 cells per window must fit an int
    return set_err(CS_B200_ERR_ARG, "bad radius %lld (0 <= radius, (2 radius + 1)^2 <= INT_MAX)", (long long)radius);
  if (block_size < 1 || block_size % 2 == 0 || block_size > INT_MAX)
    return set_err(CS_B200_ERR_ARG, "bad block_size %lld (an odd number >= 1)", (long long)block_size);
  if (!(source_threshold >= 0.0))
    return set_err(CS_B200_ERR_ARG, "bad source_threshold %g (>= 0)", source_threshold);
  if (dtype != CS_B200_F32 && dtype != CS_B200_F64) return set_err(CS_B200_ERR_ARG, "bad dtype %d", dtype);
  if (!(rtol >= 0.0) || itmax < 0)
    return set_err(CS_B200_ERR_ARG, "bad rtol %g / itmax %lld", rtol, (long long)itmax);
  if (max_batch_bytes <= 0) return set_err(CS_B200_ERR_ARG, "bad max_batch_bytes %lld", (long long)max_batch_bytes);
  if (!g || !src || !cum || !ntargets || !target_rows || !target_cols || !amps || !scale)
    return set_err(CS_B200_ERR_ARG, "g, src, cum, ntargets, target_rows, target_cols, amps and scale must not be NULL");
  if (flow_potential && (!fp || !normalized))
    return set_err(CS_B200_ERR_ARG, "fp and normalized must not be NULL with flow_potential");
  const int64_t half = (block_size - 1) / 2;
  const int64_t ncand = (nrows > half ? (nrows - 1 - half) / block_size + 1 : 0) *
                        (ncols > half ? (ncols - 1 - half) / block_size + 1 : 0);
  if (max_targets < ncand)
    return set_err(CS_B200_ERR_ARG, "max_targets %lld is below the %lld block centres", (long long)max_targets,
                   (long long)ncand);
  const size_t cells = (size_t)nrows * ncols;
  std::fill(cum, cum + cells, 0.0);
  if (flow_potential) {
    std::fill(fp, fp + cells, 0.0);
    std::fill(normalized, normalized + cells, 0.0);
  }
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return set_err(CS_B200_ERR_CUDA, "no CUDA device available (%s): libcsb200 has no CPU fallback",
                   cudaGetErrorString(e));
  if (device < 0 || device >= ndev)
    return set_err(CS_B200_ERR_ARG, "device %d out of range (0..%d)", device, ndev - 1);

  const Land L = make_land(nrows, ncols, radius, 1);
  OmniJob om{(int)block_size, source_threshold, flow_potential != 0, fp, normalized, {}, {}, {}};
  std::vector<int> trow, tcol;
  std::vector<WinOut> wo;
  e = cudaSetDevice(device);
  if (e != cudaSuccess) return set_err(CS_B200_ERR_CUDA, "cudaSetDevice(%d): %s", device, cudaGetErrorString(e));
  const int rc = dtype == CS_B200_F64
                     ? moving_windows<double>(L, (size_t)max_batch_bytes, window_bytes(L, dtype), g, src, trow, tcol,
                                              nullptr, nullptr, four_neighbors ? 1 : 0, rtol, (long long)itmax, cum,
                                              wo, &om)
                     : moving_windows<float>(L, (size_t)max_batch_bytes, window_bytes(L, dtype), g, src, trow, tcol,
                                             nullptr, nullptr, four_neighbors ? 1 : 0, rtol, (long long)itmax, cum,
                                             wo, &om);
  if (rc != CS_B200_OK) return rc;

  const int64_t nt = (int64_t)trow.size();
  *ntargets = nt;
  int64_t bad = -1;
  int worst = WIN_OK;
  bool bad_fp = false;
  for (int64_t t = 0; t < nt; ++t) {
    target_rows[t] = trow[t];
    target_cols[t] = tcol[t];
    amps[t] = om.amps[t];
    scale[t] = om.scale[t];
    if (iters) iters[t] = wo[t].iters;
    if (relres) relres[t] = wo[t].relres;
    if (wo[t].status > worst) { worst = wo[t].status; bad = t; bad_fp = false; }
    if (!om.flow) continue;
    if (fp_iters) fp_iters[t] = om.wo_fp[t].iters;
    if (fp_relres) fp_relres[t] = om.wo_fp[t].relres;
    if (om.wo_fp[t].status > worst) { worst = om.wo_fp[t].status; bad = t; bad_fp = true; }
  }
  if (first_failed) *first_failed = bad;
  const WinOut* f = bad < 0 ? nullptr : bad_fp ? &om.wo_fp[bad] : &wo[bad];
  const char* kind = bad_fp ? "flow-potential" : "conductance";
  if (worst == WIN_RESIDUAL)
    return set_err(CS_B200_ERR_RESIDUAL,
                   "CUDA PCG solver residual %g exceeds tolerance %g for target %lld, %s window (%d iterations)",
                   f->fail_relres, kGate, (long long)bad, kind, f->fail_iters);
  if (worst == WIN_MAXITER)
    return set_err(CS_B200_ERR_MAXITER,
                   "CUDA PCG solver reached itmax = %lld before rtol for target %lld, %s window (residual %g)",
                   (long long)itmax, (long long)bad, kind, f->fail_relres);
  return CS_B200_OK;
}

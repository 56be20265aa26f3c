// setup_device.hpp -- interface of the DEVICE-side setup (setup_device.cu): the smoothed-aggregation
// hierarchy (role of `smoothed_aggregation(matrix; ...)`, src/core.jl:164-167, once per connected
// component) and the windowed row-block records of every operator, built on the GPU from a CSR
// that already lives there.  Round 1 built both on the host (amg_host.hpp / win_host.hpp, still
// available through cs_b200_opts.setup = 1 and used as the reference in the tests).
//
// What runs where:
//   host    the aggregation seed pass only -- the greedy "root + free neighbourhood" rule in index
//           order (amg_host.hpp `aggregate`, phase 1).  It is the lexicographically-first maximal
//           independent set of the distance-2 graph: inherently ordered, 0.26 s for 1.6e7 nodes on
//           one core, and it tiles rasters into regular 3x3 aggregates.  The parallel MIS(2)
//           variants tried instead (profiles/r2_aggregation_study.md) produce 12-13-node
//           aggregates and cost 50 % more PCG iterations, so the ordered rule stayed; it runs on a
//           helper thread while the matrix uploads and the device does everything else.
//   device  diagonal / lambda_max(D^-1 A) by power iteration, the rest of the aggregation, tentative
//           and smoothed prolongator, P^T, the Galerkin product P^T A P (expand - radix sort -
//           compress SpGEMM, deterministic: no floating-point atomics), row blocks, windowed
//           records, fp32 copies.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <future>
#include <memory>
#include <string>
#include <vector>

namespace csb_dev {

struct DCsr {                      // device CSR, int32 indices, fp64 values (setup arithmetic)
  int64_t nrows = 0, ncols = 0, nnz = 0;
  int* ptr = nullptr;
  int* idx = nullptr;
  double* val = nullptr;
};
void free_csr(DCsr& m);

struct DLevel {
  DCsr A;                          // level 0: aliases the caller's arrays when `borrowed`
  DCsr P, R;                       // to / from the next coarser level (empty on the coarsest)
  double* dinv = nullptr;          // 1 / diag(A), n entries
  double omega = 2.0 / 3.0;
  bool borrowed = false;
};

struct DHierarchy {
  std::vector<DLevel> levels;
  std::vector<double> coarse_pinv; // host, dense n_c x n_c (row-major); empty if n_c > 320 (after coarse_pinv_wait)
  std::shared_ptr<std::future<std::vector<double>>> pinv_job;   // the eigen-solve, on a helper thread
  double operator_complexity = 1.0;
  double ms_agg_host = 0, ms_total = 0;
};
void free_hierarchy(DHierarchy& h);
void coarse_pinv_wait(DHierarchy& h);   // joins the helper thread; fills coarse_pinv

// Host copy of the finest pattern for the ordered aggregation pass (any index width / base, exactly
// what the caller handed to cs_b200_create); null pointers => the pattern is downloaded.
struct HostPattern {
  const void* rowptr = nullptr;
  const void* colidx = nullptr;
  int index_bits = 32;
  int index_base = 0;
};

// The ordered seed pass of level 0 can be started before the matrix is even on the device (it only
// reads the caller's host arrays): seed_start launches it on a helper thread, build_hierarchy joins it.
struct SeedJob;
SeedJob* seed_start(int64_t n, const HostPattern& hp);
void seed_discard(SeedJob* job);   // waits for the thread and frees the job (error paths)

int seed_wait(SeedJob* job, const int** seed, int64_t* count);   // joins; *seed stays valid until seed_discard

// level-0 seeds already on the device (multi-GPU: the root's seed pass, broadcast over NCCL)
struct DeviceSeed {
  const int* d_seed = nullptr;     // n entries, -1 = free
  int nagg = 0;
};

// Build the hierarchy of A0 (device, fp64 values; borrowed, not freed).  `pre`: a job started with
// seed_start on the same pattern (consumed), or null; `dseed`: level-0 seeds resident on the device
// (takes precedence), or null.  Returns 0 or a cudaError_t
// (as int) / -1 with `err` set.
int build_hierarchy(cudaStream_t stream, const DCsr& A0, const HostPattern& hp, SeedJob* pre, const DeviceSeed* dseed,
                    int max_levels, int max_coarse, DHierarchy& out, std::string& err, bool verbose);

// Greedy row blocks (<= max_rows rows and <= nnz_cap entries; a longer row stands alone) -- the
// partition win_host.hpp::row_blocks / build_row_blocks compute sequentially.  *d_bstart: device,
// nblocks + 1 entries, cudaMalloc'ed.
int row_blocks(cudaStream_t stream, const int* d_rowptr, int64_t nrows, int max_rows, int nnz_cap, int** d_bstart,
               int* nblocks, std::string& err);

// Windowed row-block form of a device CSR with values of type T (float / double): block descriptors
// (csb_win::BlockMeta layout) and the packed records  [values | 1/diag | 16-bit local columns | row
// offsets].  d_dinv may be null.  meta / blob: cudaMalloc'ed (null when the operator is mostly
// scattered and keeps the plain kernel, as on the host path).
struct DWin {
  void* meta = nullptr;
  unsigned char* blob = nullptr;
  int nblocks = 0;
  int64_t windowed_blocks = 0;
};
template <typename T>
int build_windowed(cudaStream_t stream, const int* d_rowptr, const int* d_colidx, const T* d_vals, int64_t nrows,
                   int64_t ncols_pad, int wcap, const T* d_dinv, DWin& out, std::string& err);

// Stencil (DIA) form of a square device CSR: if every stored entry (i, j) has j - i in
// {0, +-1, +-nr, +-(nr -+ 1)} for one stride nr >= 3 (the raster stencil with column-major numbering,
// src/raster/pairwise.jl:316-367, and the regular coarse grids below it), *d_dia receives the 9
// diagonals (slot s = 3 (dc + 1) + (dr + 1), ld = n rounded up to 4, zero where there is no entry;
// cudaMalloc'ed) and *nr the stride; otherwise *d_dia stays null.
template <typename T>
int build_dia(cudaStream_t stream, const int* d_rowptr, const int* d_colidx, const T* d_vals, int64_t n, T** d_dia,
              int* nr, size_t* ld, std::string& err);

// Half form of a stencil from build_dia: if every lower slot s < 4 of row i holds the bit pattern of the upper
// slot 8 - s of row i + off(s) (off(s) = (s / 3 - 1) nr + s % 3 - 1), or +0 where that row lies outside [0, n),
// *d_dia is replaced by a cudaMalloc'ed copy of slots 4 ... 8 (same ld) and *half set to 1; otherwise both
// are left as they are (*half = 0).  Bit patterns, not values: -0 and NaN do not pass for +0 or each other.
template <typename T>
int halve_dia(cudaStream_t stream, T** d_dia, int64_t n, int nr, size_t ld, int* half, std::string& err);

// Raster -> Laplacian WITH short-circuit polygons on the device (src/raster/pairwise.jl:271-367 +
// src/core.jl:608-624): every cell of a polygon (NODATA cells too) takes the node of the polygon's first
// valid cell, labels are compacted in order, parallel cell adjacencies of merged nodes add up, adjacencies
// inside a node are dropped.  d_g: conductances (fp64, column-major cells; <= 0 / NaN = not a node of its
// own, and 0 for the averaging rules); d_poly: polygon id per cell (0 = none, ids <= max_poly) or null.
// out: CSR (fp64, cudaMalloc'ed); *d_nodemap: node id per cell (1-based, 0 = none; cudaMalloc'ed).
int assemble_raster_polygons(cudaStream_t stream, int64_t nrows, int64_t ncols, const double* d_g, const int* d_poly,
                             int max_poly, int four_neighbors, int avg_res, DCsr& out, int** d_nodemap,
                             std::string& err);

// ELL-4 copy of a device CSR whose rows all have <= 4 entries (the prolongator of a regular grid):
// *d_col / *d_val slot-major with leading dimension *ld (cudaMalloc'ed), padding (column 0, value 0);
// both stay null if some row is longer.
template <typename T>
int build_ell4(cudaStream_t stream, const int* d_rowptr, const int* d_colidx, const T* d_vals, int64_t nrows,
               int** d_col, T** d_val, size_t* ld, std::string& err);

// narrow caller indices (int32 / int64, base 0 / 1) to int32 0-based on the device
int narrow_indices(cudaStream_t stream, const void* d_src, int index_bits, int index_base, int64_t count, int* d_dst);
int convert_values(cudaStream_t stream, const double* d_in, float* d_out, int64_t count);
int convert_values(cudaStream_t stream, const float* d_in, double* d_out, int64_t count);

// release the stream-ordered scratch pool the setup used
void trim_pool(int device);

}  // namespace csb_dev

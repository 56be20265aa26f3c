// raster_assembly.cuh -- the step BEFORE the path (SURVEY.md 8f, rank 2): the Laplacian of a
// conductance raster assembled on the device, straight into the CSR the solver consumes.
//
// Restates, without polygons, what the reference does on the host:
//   construct_node_map   src/raster/pairwise.jl:271-281  cells with conductance > 0 are nodes,
//                                                        numbered column-major (= memory order
//                                                        of the Julia matrix)
//   construct_graph      src/raster/pairwise.jl:317-367  E/S/SE/NE neighbours, symmetrised;
//                                                        cardinal / diagonal averaging rules
//   laplacian!           src/core.jl:608-624             off-diagonals -g_ij, diagonal sum_j g_ij
// Three kernels around two prefix sums (cub::DeviceScan): valid flags -> node ids; stencil
// degree per node -> rowptr; fill.  Column indices come out sorted because the stencil is
// walked in memory order.  One thread per raster cell, cell index = r + c * nrows, so every
// global access is coalesced along a raster column.
#pragma once
#include <cstdint>
#include <cub/device/device_scan.cuh>

namespace ras {

// stencil slot k = 0..8 -> (dr, dc) = (k % 3 - 1, k / 3 - 1): ascending node id for column-major
// numbering; slot 4 is the cell itself

// src/raster/pairwise.jl:364-367  (values are conductances)
__device__ __forceinline__ double weight(double a, double b, bool diagonal, bool avg_res) {
  const double s2 = 1.4142135623730951;
  if (avg_res) return diagonal ? 1.0 / (s2 * (1.0 / a + 1.0 / b) / 2.0) : 1.0 / ((1.0 / a + 1.0 / b) / 2.0);
  return diagonal ? (a + b) / (2.0 * s2) : (a + b) / 2.0;
}

template <typename T>
__global__ void k_valid(int64_t ncell, const T* __restrict__ g, int* __restrict__ valid) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ncell; i += (int64_t)gridDim.x * blockDim.x)
    valid[i] = g[i] > T(0) ? 1 : 0;   // NODATA (-9999), 0 and NaN are not nodes
}

// rowcnt[node] = 1 (diagonal) + number of valid stencil neighbours.  Internal linkage: the header
// is included by more than one translation unit.
static __global__ void k_count(int nrows, int ncols, int four, const int* __restrict__ valid,
                        const int* __restrict__ nodeid, int* __restrict__ rowcnt) {
  const int64_t ncell = (int64_t)nrows * ncols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ncell; i += (int64_t)gridDim.x * blockDim.x) {
    if (!valid[i]) continue;
    const int r = (int)(i % nrows), c = (int)(i / nrows);
    int cnt = 1;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      if (k == 4) continue;
      const int dr = k % 3 - 1, dc = k / 3 - 1;
      if (four && dr != 0 && dc != 0) continue;
      const int rr = r + dr, cc = c + dc;
      if (rr < 0 || rr >= nrows || cc < 0 || cc >= ncols) continue;
      cnt += valid[(int64_t)cc * nrows + rr];
    }
    rowcnt[nodeid[i]] = cnt;
  }
}

template <typename T>
__global__ void k_fill(int nrows, int ncols, int four, int avg_res, const T* __restrict__ g,
                       const int* __restrict__ valid, const int* __restrict__ nodeid,
                       const int* __restrict__ rowptr, int* __restrict__ colidx, T* __restrict__ vals) {
  const int64_t ncell = (int64_t)nrows * ncols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ncell; i += (int64_t)gridDim.x * blockDim.x) {
    if (!valid[i]) continue;
    const int r = (int)(i % nrows), c = (int)(i / nrows);
    const int id = nodeid[i];
    const double gi = (double)g[i];
    int p = rowptr[id];
    int diag_pos = p;
    double deg = 0.0;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      if (k == 4) { diag_pos = p++; continue; }
      const int dr = k % 3 - 1, dc = k / 3 - 1;
      const bool diagonal = dr != 0 && dc != 0;
      if (four && diagonal) continue;
      const int rr = r + dr, cc = c + dc;
      if (rr < 0 || rr >= nrows || cc < 0 || cc >= ncols) continue;
      const int64_t j = (int64_t)cc * nrows + rr;
      if (!valid[j]) continue;
      const double w = weight(gi, (double)g[j], diagonal, avg_res != 0);
      colidx[p] = nodeid[j];
      vals[p] = (T)(-w);
      deg += w;
      ++p;
    }
    colidx[diag_pos] = id;
    vals[diag_pos] = (T)deg;
  }
}

// exclusive prefix sum of `count` ints on `stream` (temporary storage allocated and freed here)
inline cudaError_t exclusive_scan(const int* d_in, int* d_out, int64_t count, cudaStream_t stream) {
  void* tmp = nullptr;
  size_t bytes = 0;
  cudaError_t e = cub::DeviceScan::ExclusiveSum(nullptr, bytes, d_in, d_out, (int)count, stream);
  if (e != cudaSuccess) return e;
  e = cudaMalloc(&tmp, bytes ? bytes : 1);
  if (e != cudaSuccess) return e;
  e = cub::DeviceScan::ExclusiveSum(tmp, bytes, d_in, d_out, (int)count, stream);
  cudaError_t e2 = cudaStreamSynchronize(stream);
  cudaFree(tmp);
  return e != cudaSuccess ? e : e2;
}

}  // namespace ras

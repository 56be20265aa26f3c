// setup_device.cu -- device-side setup of libcsb200.so: smoothed-aggregation hierarchy, row blocks and
// windowed records built on the GPU (interface and rationale: setup_device.hpp).
//
// Everything here runs once per connected component ("construct preconditioner", src/core.jl:164-167);
// the arithmetic is fp64 whatever the handle's type.  Sparse products are expand - sort - compress:
// every scalar product a_ik * b_kj becomes an item keyed (i, j), a stable radix sort (cub) groups
// equal keys in generation order and one thread per distinct key sums its run front to back, so the
// result is bit-reproducible (no floating-point atomics anywhere).
#include "setup_device.hpp"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <future>
#include <limits>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "amg_host.hpp"   // dense_pinv for the <= 320-node coarsest operator
#include "win_host.hpp"   // BlockMeta layout + window geometry shared with the kernel

namespace csb_dev {

namespace {

constexpr int TPB = 256;
// Grid caps are multiples of the H100's 132 SMs.  Fixed rather than queried: the power iteration
// combines one partial per CTA, so a fixed grid keeps the setup bit-reproducible on any device.
constexpr int SMS = 132;

#define CKD(call)                                                                                   \
  do {                                                                                              \
    cudaError_t _e = (call);                                                                        \
    if (_e != cudaSuccess) {                                                                        \
      err = std::string("CUDA error ") + cudaGetErrorString(_e) + " at " + __FILE__ + ":" +        \
            std::to_string(__LINE__) + " (" + #call + ")";                                          \
      return -2;                                                                                    \
    }                                                                                               \
  } while (0)

inline int grid_for(int64_t n, int cap = SMS * 32) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((n + TPB - 1) / TPB, cap));
}

inline int bits_for(int64_t count) {   // bits needed to hold values 0 .. count-1 (>= 1)
  int b = 1;
  while (((int64_t)1 << b) < count) ++b;
  return b;
}

// stream-ordered scratch (cudaMallocAsync): freed when it goes out of scope, reused from the pool
template <typename T>
struct Scratch {
  T* p = nullptr;
  cudaStream_t s = nullptr;
  Scratch() = default;
  Scratch(const Scratch&) = delete;
  Scratch& operator=(const Scratch&) = delete;
  ~Scratch() { release(); }
  cudaError_t alloc(size_t count, cudaStream_t stream) {
    release();
    s = stream;
    return cudaMallocAsync((void**)&p, std::max<size_t>(count, 1) * sizeof(T), stream);
  }
  void release() {
    if (p) cudaFreeAsync(p, s);
    p = nullptr;
  }
  T* take() { T* q = p; p = nullptr; return q; }
};

void ensure_pool(int device) {
  static bool done[64] = {};
  if (done[device & 63]) return;
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    uint64_t thr = std::numeric_limits<uint64_t>::max();   // keep scratch between the phases of one setup
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  done[device & 63] = true;
}

struct Tick {
  bool on;
  cudaStream_t s;
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
  Tick(bool v, cudaStream_t st) : on(v), s(st) {}
  void operator()(const char* what, int level = -1) {
    if (!on) return;
    cudaStreamSynchronize(s);
    const auto t1 = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[cs_b200 setup/device] L%-2d %-26s %8.2f ms\n", level, what,
                 std::chrono::duration<double, std::milli>(t1 - t0).count());
    t0 = t1;
  }
};

// CS_B200_VERBOSE=2: host time between sub-steps (stream synchronised), to find non-kernel overheads
struct Stamp {
  bool on;
  cudaStream_t s;
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
  explicit Stamp(cudaStream_t st) : s(st) {
    const char* e = std::getenv("CS_B200_VERBOSE");
    on = e && std::atoi(e) >= 2;
  }
  void operator()(const char* what) {
    if (!on) return;
    cudaStreamSynchronize(s);
    const auto t1 = std::chrono::steady_clock::now();
    std::fprintf(stderr, "[cs_b200 setup/stamp]        %-34s %8.2f ms\n", what,
                 std::chrono::duration<double, std::milli>(t1 - t0).count());
    t0 = t1;
  }
};

// ---------------------------------------------------------------------------------------------
// small kernels
// ---------------------------------------------------------------------------------------------
template <typename I>
__global__ void k_narrow(const I* __restrict__ src, int base, int64_t count, int* __restrict__ dst) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
    dst[i] = (int)(src[i] - (I)base);
}

template <typename TI, typename TO>
__global__ void k_cvt(const TI* __restrict__ in, TO* __restrict__ out, int64_t count) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = (TO)in[i];
}

__global__ void k_fill_int(int* p, int64_t count, int v) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
    p[i] = v;
}

__global__ void k_zero_int(int* p, int64_t count) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
    p[i] = 0;
}

// dinv = 1/diag ; rho_inf = max_i sum_j |a_ij| / |a_ii|   (amg_host.hpp diag_and_rho, first loop)
__global__ void k_diag_rho(int n, const int* __restrict__ ptr, const int* __restrict__ idx,
                           const double* __restrict__ val, double* __restrict__ dinv,
                           unsigned long long* __restrict__ rho_bits) {
  double local = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double d = 0.0, s = 0.0;
    for (int j = ptr[i]; j < ptr[i + 1]; ++j) {
      const double v = val[j];
      if (idx[j] == i) d += v;
      s += fabs(v);
    }
    if (d != 0.0) {
      dinv[i] = 1.0 / d;
      local = fmax(local, s / fabs(d));
    } else {
      dinv[i] = 0.0;
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) local = fmax(local, __shfl_xor_sync(0xffffffffu, local, off));
  // non-negative doubles order like their bit patterns: an integer max, order-independent
  if ((threadIdx.x & 31) == 0 && local > 0.0) atomicMax(rho_bits, (unsigned long long)__double_as_longlong(local));
}

// power iteration on D^-1 A (amg_host.hpp diag_and_rho): the iterate is x = s * u with the scale s kept
// in scal[0]; one launch computes y = D^-1 A x, the block partials of x'Ax, x'Dx and max|y|.
__global__ void k_power_init(int n, const double* __restrict__ dinv, double* __restrict__ u, double* scal) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    u[i] = dinv[i] != 0.0
               ? 1.0 + (double)(((unsigned long long)i * 2654435761ULL) % 1024ULL) / 1024.0 * ((i & 1) ? 1.0 : -1.0)
               : 0.0;
  if (blockIdx.x == 0 && threadIdx.x == 0) { scal[0] = 1.0; scal[1] = 0.0; scal[2] = 0.0; }
}

__global__ void __launch_bounds__(TPB)
k_power(int n, const int* __restrict__ ptr, const int* __restrict__ idx, const double* __restrict__ val,
        const double* __restrict__ dinv, const double* __restrict__ u, const double* __restrict__ scal,
        double* __restrict__ y, double* __restrict__ part) {
  __shared__ double sh[3][TPB / 32];
  const double s = scal[0];
  double sn = 0.0, sd = 0.0, sm = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double acc = 0.0;
    for (int j = ptr[i]; j < ptr[i + 1]; ++j) acc += val[j] * u[idx[j]];
    acc *= s;
    const double xi = s * u[i], di = dinv[i];
    sn += xi * acc;
    sd += di != 0.0 ? xi * xi / di : 0.0;
    const double yi = di * acc;
    y[i] = yi;
    sm = fmax(sm, fabs(yi));
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    sn += __shfl_xor_sync(0xffffffffu, sn, off);
    sd += __shfl_xor_sync(0xffffffffu, sd, off);
    sm = fmax(sm, __shfl_xor_sync(0xffffffffu, sm, off));
  }
  const int w = threadIdx.x >> 5;
  if ((threadIdx.x & 31) == 0) { sh[0][w] = sn; sh[1][w] = sd; sh[2][w] = sm; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0, b = 0.0, c = 0.0;
    for (int q = 0; q < TPB / 32; ++q) { a += sh[0][q]; b += sh[1][q]; c = fmax(c, sh[2][q]); }
    part[blockIdx.x] = a;
    part[gridDim.x + blockIdx.x] = b;
    part[2 * gridDim.x + blockIdx.x] = c;
  }
}

// one thread: fixed-order combine of the block partials; lam = x'Ax / x'Dx, next scale = 1 / max|y|
__global__ void k_power_final(int nblk, const double* __restrict__ part, double* scal) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (scal[2] != 0.0) return;                      // frozen (degenerate iterate), as the host loop's `break`
  double num = 0.0, den = 0.0, nrm = 0.0;
  for (int b = 0; b < nblk; ++b) { num += part[b]; den += part[nblk + b]; nrm = fmax(nrm, part[2 * nblk + b]); }
  if (!(den > 0.0)) { scal[2] = 1.0; return; }
  scal[1] = num / den;
  if (!(nrm > 0.0)) { scal[2] = 1.0; return; }
  scal[0] = 1.0 / nrm;
}

// aggregation phase 2 (amg_host.hpp `aggregate`): a node the seed pass left free joins the aggregate of
// its strongest already-seeded neighbour (first maximum in row order)
__global__ void k_agg_join(int n, const int* __restrict__ ptr, const int* __restrict__ idx,
                           const double* __restrict__ val, const int* __restrict__ seeded, int* __restrict__ agg,
                           int* __restrict__ cnt) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int a = seeded[i];
    if (a < 0) {
      double best = 0.0;
      for (int j = ptr[i]; j < ptr[i + 1]; ++j) {
        const int c = idx[j];
        if (c == i) continue;
        const int sc = seeded[c];
        if (sc < 0) continue;
        const double w = fabs(val[j]);
        if (w > best) { best = w; a = sc; }
      }
    }
    agg[i] = a;
    if (a >= 0) atomicAdd(&cnt[a], 1);
  }
}

// items of P = T - omega D^-1 (A T): row i owns slots ptr[i]+i .. ptr[i+1]+i (one per stored entry,
// then the T entry); entries whose column has no aggregate carry the sentinel column (dropped later)
__global__ void k_expand_P(int n, const int* __restrict__ ptr, const int* __restrict__ idx,
                           const double* __restrict__ val, const double* __restrict__ dinv, double omega,
                           const int* __restrict__ agg, const int* __restrict__ cnt, int cb, unsigned sentinel,
                           unsigned long long* __restrict__ keys, double* __restrict__ vals) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int a = ptr[i], b = ptr[i + 1];
    const double sc = omega * dinv[i];
    const unsigned long long hi = (unsigned long long)i << cb;
    int64_t o = (int64_t)a + i;
    for (int j = a; j < b; ++j, ++o) {
      const int c = agg[idx[j]];
      if (c >= 0) {
        keys[o] = hi | (unsigned)c;
        vals[o] = -sc * val[j] * (1.0 / sqrt((double)cnt[c]));
      } else {
        keys[o] = hi | sentinel;
        vals[o] = 0.0;
      }
    }
    const int mine = agg[i];
    if (mine >= 0) {
      keys[o] = hi | (unsigned)mine;
      vals[o] = 1.0 / sqrt((double)cnt[mine]);
    } else {
      keys[o] = hi | sentinel;
      vals[o] = 0.0;
    }
  }
}

__global__ void k_fill_erow(int n, const int* __restrict__ ptr, int* __restrict__ erow) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    for (int j = ptr[i]; j < ptr[i + 1]; ++j) erow[j] = i;
}

__global__ void k_cnt_products(int64_t nnz, const int* __restrict__ aidx, const int* __restrict__ bptr,
                               long long* __restrict__ cnt) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e <= nnz; e += (int64_t)gridDim.x * blockDim.x)
    cnt[e] = e < nnz ? (long long)(bptr[aidx[e] + 1] - bptr[aidx[e]]) : 0;
}

__global__ void k_expand_AB(int64_t nnz, const int* __restrict__ erow, const int* __restrict__ aidx,
                            const double* __restrict__ aval, const int* __restrict__ bptr,
                            const int* __restrict__ bidx, const double* __restrict__ bval,
                            const long long* __restrict__ off, int cb, unsigned long long* __restrict__ keys,
                            double* __restrict__ vals) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x) {
    const int k = aidx[e];
    const double av = aval[e];
    const unsigned long long hi = (unsigned long long)erow[e] << cb;
    long long o = off[e];
    for (int j = bptr[k]; j < bptr[k + 1]; ++j, ++o) {
      keys[o] = hi | (unsigned)bidx[j];
      vals[o] = av * bval[j];
    }
  }
}

// transpose items: key = (column, row)
__global__ void k_expand_T(int64_t nnz, const int* __restrict__ erow, const int* __restrict__ idx, int rb,
                           unsigned long long* __restrict__ keys) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nnz; e += (int64_t)gridDim.x * blockDim.x)
    keys[e] = ((unsigned long long)idx[e] << rb) | (unsigned)erow[e];
}

// flag[k] = 1 where a new (row, column) key starts (and the column is not the sentinel); flag[m] = 0
__global__ void k_heads(int64_t m, const unsigned long long* __restrict__ keys, unsigned long long colmask,
                        unsigned long long sentinel, int use_sentinel, int* __restrict__ flag) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k <= m; k += (int64_t)gridDim.x * blockDim.x) {
    int f = 0;
    if (k < m) {
      const unsigned long long key = keys[k];
      f = (k == 0 || keys[k - 1] != key) ? 1 : 0;
      if (use_sentinel && (key & colmask) == sentinel) f = 0;
    }
    flag[k] = f;
  }
}

// one thread per distinct key: sums its run front to back (generation order => deterministic)
__global__ void k_compress(int64_t m, const unsigned long long* __restrict__ keys, const double* __restrict__ vals,
                           const int* __restrict__ flag, const int* __restrict__ pos, int cb,
                           unsigned long long colmask, int* __restrict__ out_idx, double* __restrict__ out_val,
                           int* __restrict__ rowcnt) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < m; k += (int64_t)gridDim.x * blockDim.x) {
    if (!flag[k]) continue;
    const unsigned long long key = keys[k];
    double s = vals[k];
    for (int64_t q = k + 1; q < m && keys[q] == key; ++q) s += vals[q];
    const int p = pos[k];
    out_idx[p] = (int)(key & colmask);
    out_val[p] = s;
    atomicAdd(&rowcnt[(int)(key >> cb)], 1);
  }
}

__global__ void k_unpack_T(int64_t m, const unsigned long long* __restrict__ keys, int rb,
                           unsigned long long rowmask, int* __restrict__ out_idx, int* __restrict__ rowcnt) {
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < m; k += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long key = keys[k];
    out_idx[k] = (int)(key & rowmask);
    atomicAdd(&rowcnt[(int)(key >> rb)], 1);
  }
}

// ---------------------------------------------------------------------------------------------
// cub wrappers on scratch
// ---------------------------------------------------------------------------------------------
template <typename TIn, typename TOut>
int exclusive_scan(cudaStream_t s, const TIn* in, TOut* out, int64_t count, std::string& err) {
  size_t bytes = 0;
  CKD(cub::DeviceScan::ExclusiveSum(nullptr, bytes, in, out, count, s));
  Scratch<unsigned char> tmp;
  CKD(tmp.alloc(bytes, s));
  CKD(cub::DeviceScan::ExclusiveSum(tmp.p, bytes, in, out, count, s));
  return 0;
}

// stable sort of (key, value) pairs on the low `nbits` bits; results in keys_out / vals_out
int sort_pairs(cudaStream_t s, const unsigned long long* kin, unsigned long long* kout, const double* vin,
               double* vout, int64_t count, int nbits, std::string& err) {
  size_t bytes = 0;
  CKD(cub::DeviceRadixSort::SortPairs(nullptr, bytes, kin, kout, vin, vout, count, 0, nbits, s));
  Scratch<unsigned char> tmp;
  CKD(tmp.alloc(bytes, s));
  CKD(cub::DeviceRadixSort::SortPairs(tmp.p, bytes, kin, kout, vin, vout, count, 0, nbits, s));
  return 0;
}

// sorted (row, col) items -> CSR with duplicates summed.  keys/vals: sorted.  out: cudaMalloc'ed.
int compress_to_csr(cudaStream_t s, int64_t m, const unsigned long long* keys, const double* vals, int64_t nrows,
                    int64_t ncols, int cb, bool use_sentinel, unsigned sentinel, int64_t max_nnz, bool* overflow,
                    DCsr& out, std::string& err) {
  if (overflow) *overflow = false;
  const unsigned long long colmask = (((unsigned long long)1) << cb) - 1ULL;
  Scratch<int> flag, pos, rowcnt;
  CKD(flag.alloc((size_t)m + 1, s));
  CKD(pos.alloc((size_t)m + 1, s));
  CKD(rowcnt.alloc((size_t)nrows + 1, s));
  k_heads<<<grid_for(m + 1), TPB, 0, s>>>(m, keys, colmask, (unsigned long long)sentinel, use_sentinel ? 1 : 0, flag.p);
  CKD(cudaGetLastError());
  int rc = exclusive_scan(s, flag.p, pos.p, m + 1, err);
  if (rc) return rc;
  int total = 0;
  CKD(cudaMemcpyAsync(&total, pos.p + m, sizeof(int), cudaMemcpyDeviceToHost, s));
  CKD(cudaStreamSynchronize(s));
  out = DCsr{};
  out.nrows = nrows; out.ncols = ncols; out.nnz = total;
  if (max_nnz > 0 && (int64_t)total > max_nnz) {
    if (overflow) *overflow = true;
    return 0;
  }
  CKD(cudaMalloc(&out.ptr, (size_t)(nrows + 1) * sizeof(int)));
  CKD(cudaMalloc(&out.idx, std::max<size_t>(1, (size_t)total) * sizeof(int)));
  CKD(cudaMalloc(&out.val, std::max<size_t>(1, (size_t)total) * sizeof(double)));
  k_zero_int<<<grid_for(nrows + 1), TPB, 0, s>>>(rowcnt.p, nrows + 1);
  k_compress<<<grid_for(m), TPB, 0, s>>>(m, keys, vals, flag.p, pos.p, cb, colmask, out.idx, out.val, rowcnt.p);
  CKD(cudaGetLastError());
  rc = exclusive_scan(s, rowcnt.p, out.ptr, nrows + 1, err);
  return rc;
}

// C = A * B on the device.  product_budget: give up (overflow) before expanding if the number of
// scalar products exceeds it; max_nnz: give up after the sort if C would have more entries.
int spgemm(cudaStream_t s, const DCsr& A, const DCsr& B, int64_t product_budget, int64_t max_nnz, bool* overflow,
           DCsr& C, std::string& err) {
  *overflow = false;
  C = DCsr{};
  C.nrows = A.nrows; C.ncols = B.ncols;
  Stamp st(s);
  Scratch<int> erow;
  Scratch<long long> cnt, off;
  CKD(erow.alloc((size_t)A.nnz, s));
  CKD(cnt.alloc((size_t)A.nnz + 1, s));
  CKD(off.alloc((size_t)A.nnz + 1, s));
  st("spgemm: scratch alloc");
  k_fill_erow<<<grid_for(A.nrows), TPB, 0, s>>>((int)A.nrows, A.ptr, erow.p);
  k_cnt_products<<<grid_for(A.nnz + 1), TPB, 0, s>>>(A.nnz, A.idx, B.ptr, cnt.p);
  CKD(cudaGetLastError());
  int rc = exclusive_scan(s, cnt.p, off.p, A.nnz + 1, err);
  if (rc) return rc;
  long long m = 0;
  CKD(cudaMemcpyAsync(&m, off.p + A.nnz, sizeof(long long), cudaMemcpyDeviceToHost, s));
  CKD(cudaStreamSynchronize(s));
  st("spgemm: count + scan");
  if (m > product_budget || m >= (long long)std::numeric_limits<int>::max()) {
    *overflow = true;
    return 0;
  }
  cnt.release();
  const int cb = bits_for(B.ncols), rb = bits_for(A.nrows);
  Scratch<unsigned long long> k0, k1;
  Scratch<double> v0, v1;
  CKD(k0.alloc((size_t)m, s));
  CKD(k1.alloc((size_t)m, s));
  CKD(v0.alloc((size_t)m, s));
  CKD(v1.alloc((size_t)m, s));
  st("spgemm: item buffers alloc");
  k_expand_AB<<<grid_for(A.nnz), TPB, 0, s>>>(A.nnz, erow.p, A.idx, A.val, B.ptr, B.idx, B.val, off.p, cb, k0.p, v0.p);
  CKD(cudaGetLastError());
  st("spgemm: expand");
  rc = sort_pairs(s, k0.p, k1.p, v0.p, v1.p, m, cb + rb, err);
  if (rc) return rc;
  st("spgemm: sort");
  k0.release();
  v0.release();
  struct Tail { Stamp& st; ~Tail() { st("spgemm: compress"); } } tail{st};
  return compress_to_csr(s, m, k1.p, v1.p, A.nrows, B.ncols, cb, false, 0, max_nnz, overflow, C, err);
}

int transpose(cudaStream_t s, const DCsr& P, DCsr& R, std::string& err) {
  R = DCsr{};
  R.nrows = P.ncols; R.ncols = P.nrows; R.nnz = P.nnz;
  const int rb = bits_for(P.nrows), cb = bits_for(P.ncols);
  Scratch<int> erow, rowcnt;
  Scratch<unsigned long long> k0, k1;
  CKD(erow.alloc((size_t)P.nnz, s));
  CKD(k0.alloc((size_t)P.nnz, s));
  CKD(k1.alloc((size_t)P.nnz, s));
  CKD(rowcnt.alloc((size_t)R.nrows + 1, s));
  CKD(cudaMalloc(&R.ptr, (size_t)(R.nrows + 1) * sizeof(int)));
  CKD(cudaMalloc(&R.idx, std::max<size_t>(1, (size_t)P.nnz) * sizeof(int)));
  CKD(cudaMalloc(&R.val, std::max<size_t>(1, (size_t)P.nnz) * sizeof(double)));
  k_fill_erow<<<grid_for(P.nrows), TPB, 0, s>>>((int)P.nrows, P.ptr, erow.p);
  k_expand_T<<<grid_for(P.nnz), TPB, 0, s>>>(P.nnz, erow.p, P.idx, rb, k0.p);
  CKD(cudaGetLastError());
  int rc = sort_pairs(s, k0.p, k1.p, P.val, R.val, P.nnz, rb + cb, err);
  if (rc) return rc;
  k_zero_int<<<grid_for(R.nrows + 1), TPB, 0, s>>>(rowcnt.p, R.nrows + 1);
  k_unpack_T<<<grid_for(P.nnz), TPB, 0, s>>>(P.nnz, k1.p, rb, (((unsigned long long)1) << rb) - 1ULL, R.idx, rowcnt.p);
  CKD(cudaGetLastError());
  return exclusive_scan(s, rowcnt.p, R.ptr, R.nrows + 1, err);
}

// dinv, omega = (4/3) / rho with rho ~ lambda_max(D^-1 A) from 8 power iterations kept inside
// [0.7, 1] x ||D^-1 A||_inf  (amg_host.hpp diag_and_rho)
int diag_and_rho(cudaStream_t s, const DCsr& A, double* dinv, double* rho, std::string& err) {
  const int n = (int)A.nrows;
  const int g = grid_for(n, SMS * 8);
  Scratch<double> u, y, part, scal;
  Scratch<unsigned long long> rbits;
  CKD(u.alloc((size_t)n, s));
  CKD(y.alloc((size_t)n, s));
  CKD(part.alloc((size_t)3 * g, s));
  CKD(scal.alloc(4, s));
  CKD(rbits.alloc(1, s));
  CKD(cudaMemsetAsync(rbits.p, 0, sizeof(unsigned long long), s));
  k_diag_rho<<<g, TPB, 0, s>>>(n, A.ptr, A.idx, A.val, dinv, rbits.p);
  k_power_init<<<g, TPB, 0, s>>>(n, dinv, u.p, scal.p);
  double *a = u.p, *b = y.p;
  for (int it = 0; it < 8; ++it) {
    k_power<<<g, TPB, 0, s>>>(n, A.ptr, A.idx, A.val, dinv, a, scal.p, b, part.p);
    k_power_final<<<1, 32, 0, s>>>(g, part.p, scal.p);
    std::swap(a, b);
  }
  CKD(cudaGetLastError());
  double hs[4] = {0, 0, 0, 0};
  unsigned long long hb = 0;
  CKD(cudaMemcpyAsync(hs, scal.p, 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
  CKD(cudaMemcpyAsync(&hb, rbits.p, sizeof(hb), cudaMemcpyDeviceToHost, s));
  CKD(cudaStreamSynchronize(s));
  double rho_inf;
  std::memcpy(&rho_inf, &hb, sizeof(double));
  const double lam = hs[1];
  if (!(rho_inf > 0.0)) { *rho = 1.0; return 0; }
  *rho = lam > 0.0 ? std::min(rho_inf, std::max(lam, 0.7 * rho_inf)) : rho_inf;
  return 0;
}

// the ordered seed pass of the aggregation (amg_host.hpp `aggregate`, phase 1) on a host pattern of
// any index type: a node whose whole neighbourhood is still free seeds an aggregate and takes it
template <typename I>
int greedy_seed(int64_t n, const I* ptr, const I* idx, I base, std::vector<int>& agg) {
  agg.assign((size_t)n, -1);
  int nagg = 0;
  for (int64_t i = 0; i < n; ++i) {
    if (agg[i] >= 0) continue;
    const int64_t a = (int64_t)(ptr[i] - base), b = (int64_t)(ptr[i + 1] - base);
    bool any = false, all_free = true;
    for (int64_t j = a; j < b; ++j) {
      const int64_t c = (int64_t)(idx[j] - base);
      if (c == i) continue;
      any = true;
      if (agg[c] >= 0) { all_free = false; break; }
    }
    if (!any || !all_free) continue;
    agg[i] = nagg;
    for (int64_t j = a; j < b; ++j) {
      const int64_t c = (int64_t)(idx[j] - base);
      if (c != i) agg[c] = nagg;
    }
    ++nagg;
  }
  return nagg;
}

int greedy_seed_any(int64_t n, const HostPattern& hp, std::vector<int>& agg) {
  if (hp.index_bits == 64)
    return greedy_seed<int64_t>(n, (const int64_t*)hp.rowptr, (const int64_t*)hp.colidx, (int64_t)hp.index_base, agg);
  return greedy_seed<int32_t>(n, (const int32_t*)hp.rowptr, (const int32_t*)hp.colidx, (int32_t)hp.index_base, agg);
}

}  // namespace

struct SeedJob {
  std::future<int> fut;
  std::vector<int> seed;
};

SeedJob* seed_start(int64_t n, const HostPattern& hp) {
  SeedJob* job = new SeedJob();
  const HostPattern h = hp;
  job->fut = std::async(std::launch::async, [n, h, job]() { return greedy_seed_any(n, h, job->seed); });
  return job;
}

int seed_wait(SeedJob* job, const int** seed, int64_t* count) {
  const int nagg = job->fut.get();
  *seed = job->seed.data();
  *count = (int64_t)job->seed.size();
  return nagg;
}

void seed_discard(SeedJob* job) {
  if (!job) return;
  if (job->fut.valid()) job->fut.wait();
  delete job;
}

// ---------------------------------------------------------------------------------------------
// public helpers
// ---------------------------------------------------------------------------------------------
void free_csr(DCsr& m) {
  cudaFree(m.ptr);
  cudaFree(m.idx);
  cudaFree(m.val);
  m = DCsr{};
}

void coarse_pinv_wait(DHierarchy& h) {
  if (h.pinv_job && h.pinv_job->valid()) h.coarse_pinv = h.pinv_job->get();
  h.pinv_job.reset();
}

void free_hierarchy(DHierarchy& h) {
  coarse_pinv_wait(h);
  for (auto& L : h.levels) {
    if (!L.borrowed) free_csr(L.A);
    free_csr(L.P);
    free_csr(L.R);
    cudaFree(L.dinv);
  }
  h.levels.clear();
}

void trim_pool(int device) {
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) cudaMemPoolTrimTo(pool, 0);
}

int narrow_indices(cudaStream_t s, const void* d_src, int index_bits, int index_base, int64_t count, int* d_dst) {
  if (index_bits == 64)
    k_narrow<long long><<<grid_for(count), TPB, 0, s>>>((const long long*)d_src, index_base, count, d_dst);
  else
    k_narrow<int><<<grid_for(count), TPB, 0, s>>>((const int*)d_src, index_base, count, d_dst);
  return (int)cudaGetLastError();
}

int convert_values(cudaStream_t s, const double* d_in, float* d_out, int64_t count) {
  k_cvt<double, float><<<grid_for(count), TPB, 0, s>>>(d_in, d_out, count);
  return (int)cudaGetLastError();
}
int convert_values(cudaStream_t s, const float* d_in, double* d_out, int64_t count) {
  k_cvt<float, double><<<grid_for(count), TPB, 0, s>>>(d_in, d_out, count);
  return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// hierarchy
// ---------------------------------------------------------------------------------------------
int build_hierarchy(cudaStream_t s, const DCsr& A0, const HostPattern& hp0, SeedJob* pre, const DeviceSeed* dseed,
                    int max_levels, int max_coarse, DHierarchy& out, std::string& err, bool verbose) {
  struct JobGuard { SeedJob*& j; ~JobGuard() { seed_discard(j); j = nullptr; } } job_guard{pre};
  int dev = 0;
  cudaGetDevice(&dev);
  ensure_pool(dev);
  const auto t_begin = std::chrono::steady_clock::now();
  Tick tick(verbose, s);
  out.levels.clear();
  out.levels.emplace_back();
  out.levels.back().A = A0;
  out.levels.back().borrowed = true;

  // the ordered seed pass of level 0 runs on a helper thread while the device works on the diagonal
  // and the power iteration; without a host copy of the pattern it is downloaded first
  std::vector<int> h_ptr, h_idx;
  HostPattern hp = hp0;
  if (!pre && !dseed && A0.nrows > max_coarse && max_levels > 1 && (!hp.rowptr || !hp.colidx)) {
    h_ptr.resize((size_t)A0.nrows + 1);
    h_idx.resize((size_t)std::max<int64_t>(A0.nnz, 1));
    CKD(cudaMemcpyAsync(h_ptr.data(), A0.ptr, (size_t)(A0.nrows + 1) * sizeof(int), cudaMemcpyDeviceToHost, s));
    CKD(cudaMemcpyAsync(h_idx.data(), A0.idx, (size_t)A0.nnz * sizeof(int), cudaMemcpyDeviceToHost, s));
    CKD(cudaStreamSynchronize(s));
    hp = HostPattern{h_ptr.data(), h_idx.data(), 32, 0};
    tick("pattern download", 0);
  }

  for (;;) {
    const int l = (int)out.levels.size() - 1;
    DLevel& lv = out.levels.back();
    const int64_t n = lv.A.nrows;
    const bool coarsen = (int)out.levels.size() < max_levels && n > max_coarse;
    // host seed pass (async) || device diag + rho
    std::vector<int> seed;
    std::future<int> fut;
    const auto t_agg = std::chrono::steady_clock::now();
    const bool use_dev = coarsen && l == 0 && dseed != nullptr;
    const bool use_pre = coarsen && l == 0 && pre != nullptr && !use_dev;
    if (coarsen && !use_pre && !use_dev) {
      const HostPattern hpl = hp;
      fut = std::async(std::launch::async, [n, hpl, &seed]() { return greedy_seed_any(n, hpl, seed); });
    }
    CKD(cudaMalloc(&lv.dinv, std::max<size_t>(1, (size_t)n) * sizeof(double)));
    double rho = 1.0;
    int rc = diag_and_rho(s, lv.A, lv.dinv, &rho, err);
    if (rc) { if (fut.valid()) fut.wait(); return rc; }
    lv.omega = (4.0 / 3.0) / rho;
    tick("diag + lambda_max", l);
    if (!coarsen) break;
    int nagg;
    if (use_dev) {
      nagg = dseed->nagg;
    } else if (use_pre) {
      nagg = pre->fut.get();
      seed.swap(pre->seed);
    } else {
      nagg = fut.get();
    }
    out.ms_agg_host += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_agg).count();
    tick("seed pass (host) wait", l);
    if (nagg <= 0 || nagg >= n) break;

    // aggregates: upload seeds, join the rest on the device, count
    Scratch<int> d_seed, d_agg, d_cnt;
    CKD(d_seed.alloc((size_t)n, s));
    CKD(d_agg.alloc((size_t)n, s));
    CKD(d_cnt.alloc((size_t)nagg, s));
    if (!use_dev) CKD(cudaMemcpyAsync(d_seed.p, seed.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice, s));
    k_zero_int<<<grid_for(nagg), TPB, 0, s>>>(d_cnt.p, nagg);
    k_agg_join<<<grid_for(n), TPB, 0, s>>>((int)n, lv.A.ptr, lv.A.idx, lv.A.val, use_dev ? dseed->d_seed : d_seed.p,
                                            d_agg.p, d_cnt.p);
    CKD(cudaGetLastError());
    CKD(cudaStreamSynchronize(s));   // `seed` (pageable) must outlive the copy
    d_seed.release();

    // P = (I - omega D^-1 A) T  by expand / sort / compress
    DCsr P;
    {
      const int64_t m = lv.A.nnz + n;
      const int cb = bits_for((int64_t)nagg + 1), rb = bits_for(n);
      const unsigned sentinel = (unsigned)nagg;
      Scratch<unsigned long long> k0, k1;
      Scratch<double> v0, v1;
      CKD(k0.alloc((size_t)m, s));
      CKD(k1.alloc((size_t)m, s));
      CKD(v0.alloc((size_t)m, s));
      CKD(v1.alloc((size_t)m, s));
      k_expand_P<<<grid_for(n), TPB, 0, s>>>((int)n, lv.A.ptr, lv.A.idx, lv.A.val, lv.dinv, lv.omega, d_agg.p, d_cnt.p,
                                             cb, sentinel, k0.p, v0.p);
      CKD(cudaGetLastError());
      rc = sort_pairs(s, k0.p, k1.p, v0.p, v1.p, m, cb + rb, err);
      if (rc) return rc;
      k0.release();
      v0.release();
      bool over = false;
      rc = compress_to_csr(s, m, k1.p, v1.p, n, nagg, cb, true, sentinel, 0, &over, P, err);
      if (rc) return rc;
    }
    d_agg.release();
    d_cnt.release();
    tick("prolongator", l);

    // Galerkin product with the densification guard of the host path (expander-like graphs):
    // A P within 4 nnz(A), P^T A P within nnz(A); the product counts are bounded before expanding
    bool over = false;
    DCsr AP, R, Ac;
    const int64_t budget = std::min<int64_t>(16 * lv.A.nnz + (1 << 20), (int64_t)1500000000);
    rc = spgemm(s, lv.A, P, budget, 4 * lv.A.nnz, &over, AP, err);
    if (rc) { free_csr(P); return rc; }
    if (over) { free_csr(P); free_csr(AP); break; }
    tick("A * P", l);
    rc = transpose(s, P, R, err);
    if (rc) { free_csr(P); free_csr(AP); return rc; }
    tick("P^T", l);
    rc = spgemm(s, R, AP, budget, lv.A.nnz, &over, Ac, err);
    free_csr(AP);
    if (rc) { free_csr(P); free_csr(R); return rc; }
    if (over || Ac.nnz > lv.A.nnz) { free_csr(P); free_csr(R); free_csr(Ac); break; }
    tick("P^T (A P)", l);
    lv.P = P;
    lv.R = R;
    out.levels.emplace_back();
    out.levels.back().A = Ac;
    // pattern of the new level for its seed pass
    if ((int)out.levels.size() < max_levels && Ac.nrows > max_coarse) {
      h_ptr.resize((size_t)Ac.nrows + 1);
      h_idx.resize((size_t)std::max<int64_t>(Ac.nnz, 1));
      CKD(cudaMemcpyAsync(h_ptr.data(), Ac.ptr, (size_t)(Ac.nrows + 1) * sizeof(int), cudaMemcpyDeviceToHost, s));
      CKD(cudaMemcpyAsync(h_idx.data(), Ac.idx, (size_t)Ac.nnz * sizeof(int), cudaMemcpyDeviceToHost, s));
      CKD(cudaStreamSynchronize(s));
      hp = HostPattern{h_ptr.data(), h_idx.data(), 32, 0};
      tick("pattern download", l + 1);
    }
  }

  // exact coarse solve only while the dense eigen-solve stays cheap (amg_host.hpp build_hierarchy)
  const DCsr& C = out.levels.back().A;
  out.coarse_pinv.clear();
  if (C.nrows <= 320) {
    csb_amg::Csr hc;
    hc.nrows = hc.ncols = C.nrows;
    hc.ptr.resize((size_t)C.nrows + 1);
    hc.idx.resize((size_t)C.nnz);
    hc.val.resize((size_t)C.nnz);
    CKD(cudaMemcpyAsync(hc.ptr.data(), C.ptr, hc.ptr.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (C.nnz) {
      CKD(cudaMemcpyAsync(hc.idx.data(), C.idx, hc.idx.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
      CKD(cudaMemcpyAsync(hc.val.data(), C.val, hc.val.size() * sizeof(double), cudaMemcpyDeviceToHost, s));
    }
    CKD(cudaStreamSynchronize(s));
    // the dense eigen-solve (~0.1 s for 200 nodes on one core) runs on a helper thread while the
    // caller turns the levels into window records; joined by coarse_pinv_wait()
    out.pinv_job = std::make_shared<std::future<std::vector<double>>>(
        std::async(std::launch::async, [hc = std::move(hc)]() { return csb_amg::dense_pinv(hc); }));
    tick("coarse operator download", (int)out.levels.size() - 1);
  }
  double tot = 0.0;
  for (auto& L : out.levels) tot += (double)L.A.nnz;
  out.operator_complexity = tot / (double)std::max<int64_t>(1, out.levels[0].A.nnz);
  out.ms_total = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_begin).count();
  return 0;
}

// ---------------------------------------------------------------------------------------------
// row blocks: greedy blocks of <= max_rows rows and <= nnz_cap entries (a longer row stands alone), the
// rule of win_host.hpp::row_blocks -- restarted at every chunk of CHUNK rows so that the chunks are
// independent: one thread walks its chunk block by block (the end of a block is a binary search in
// rowptr), first to count, then to write.  At most one short block per chunk more than the global
// greedy partition (< 2 % for every operator of the hierarchy).
// ---------------------------------------------------------------------------------------------
namespace {

constexpr int RB_CHUNK = 2048;

__device__ __forceinline__ int block_end(const int* __restrict__ rowptr, int r, int limit, int max_rows, int cap) {
  const int base = rowptr[r];
  int lo = r + 1, hi = min(limit, r + max_rows);   // answer in [lo, hi]
  while (lo < hi) {                                 // largest r1 with rowptr[r1] - base <= cap
    const int mid = (lo + hi + 1) >> 1;
    if (rowptr[mid] - base <= cap) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void k_count_blocks(int n, const int* __restrict__ rowptr, int max_rows, int cap, int nchunk,
                               int* __restrict__ cnt) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c <= nchunk; c += gridDim.x * blockDim.x) {
    int k = 0;
    if (c < nchunk) {
      const int end = min(n, (c + 1) * RB_CHUNK);
      for (int r = c * RB_CHUNK; r < end; ++k) r = block_end(rowptr, r, end, max_rows, cap);
    }
    cnt[c] = k;
  }
}

__global__ void k_write_blocks(int n, const int* __restrict__ rowptr, int max_rows, int cap, int nchunk,
                               const int* __restrict__ off, int* __restrict__ bstart) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c <= nchunk; c += gridDim.x * blockDim.x) {
    if (c == nchunk) { bstart[off[nchunk]] = n; continue; }
    const int end = min(n, (c + 1) * RB_CHUNK);
    int k = off[c];
    for (int r = c * RB_CHUNK; r < end; ++k) {
      bstart[k] = r;
      r = block_end(rowptr, r, end, max_rows, cap);
    }
  }
}

}  // namespace

int row_blocks(cudaStream_t s, const int* d_rowptr, int64_t nrows, int max_rows, int nnz_cap, int** d_bstart,
               int* nblocks, std::string& err) {
  int dev = 0;
  cudaGetDevice(&dev);
  ensure_pool(dev);
  const int n = (int)nrows;
  *d_bstart = nullptr;
  *nblocks = 0;
  const int nchunk = (n + RB_CHUNK - 1) / RB_CHUNK;
  Scratch<int> cnt, off;
  CKD(cnt.alloc((size_t)nchunk + 1, s));
  CKD(off.alloc((size_t)nchunk + 1, s));
  const int g = grid_for((int64_t)nchunk + 1);
  k_count_blocks<<<g, 64, 0, s>>>(n, d_rowptr, max_rows, nnz_cap, nchunk, cnt.p);
  CKD(cudaGetLastError());
  int rc = exclusive_scan(s, cnt.p, off.p, (int64_t)nchunk + 1, err);
  if (rc) return rc;
  int total = 0;
  CKD(cudaMemcpyAsync(&total, off.p + nchunk, sizeof(int), cudaMemcpyDeviceToHost, s));
  CKD(cudaStreamSynchronize(s));
  CKD(cudaMalloc(d_bstart, (size_t)(total + 1) * sizeof(int)));
  k_write_blocks<<<g, 64, 0, s>>>(n, d_rowptr, max_rows, nnz_cap, nchunk, off.p, *d_bstart);
  CKD(cudaGetLastError());
  *nblocks = total;
  return 0;
}

// ---------------------------------------------------------------------------------------------
// windowed records (win_host.hpp `build`, restated per block on the device)
// ---------------------------------------------------------------------------------------------
namespace {

using csb_win::ALN;
using csb_win::BlockMeta;
using csb_win::MAXSEG;
using csb_win::MERGE_GAP;
using csb_win::NNZ_CAP;
using csb_win::RB;

__global__ void k_record_sizes(int nb, const int* __restrict__ bstart, const int* __restrict__ rowptr, int vsize,
                               int with_dinv, long long* __restrict__ size) {
  for (int b = blockIdx.x * blockDim.x + threadIdx.x; b <= nb; b += gridDim.x * blockDim.x) {
    long long sz = 0;
    if (b < nb) {
      const int r0 = bstart[b], r1 = bstart[b + 1];
      const int cnt = rowptr[r1] - rowptr[r0];
      if (cnt <= NNZ_CAP && (r1 - r0) <= RB)
        sz = (long long)((cnt + 7) / 8 * 8) * (vsize + 2) + (long long)((r1 - r0 + 1 + 7) / 8 * 8) * 2 +
             (with_dinv ? (long long)((r1 - r0 + 7) / 8 * 8) * vsize : 0);
    }
    size[b] = sz;
  }
}

constexpr int WB_T = 128;     // threads per CTA of k_win_build
constexpr int WB_SORT = 2048; // >= NNZ_CAP, power of two

template <typename T>
__global__ void __launch_bounds__(WB_T)
k_win_build(int nb, const int* __restrict__ bstart, const int* __restrict__ rowptr, const int* __restrict__ colidx,
            const T* __restrict__ vals, const T* __restrict__ dinv, long long ncols_pad, int wcap,
            const long long* __restrict__ blob_off, BlockMeta* __restrict__ meta, unsigned char* __restrict__ blob,
            int* __restrict__ nwin) {
  __shared__ int s_cols[WB_SORT];
  __shared__ int s_start[MAXSEG + 1];   // positions (in the sorted list) where a run starts
  __shared__ int s_nrun;
  __shared__ int s_lo[MAXSEG], s_len[MAXSEG], s_off[MAXSEG];
  __shared__ int s_nseg, s_total, s_self;
  const int tid = threadIdx.x;
  for (int b = blockIdx.x; b < nb; b += gridDim.x) {
    const int r0 = bstart[b], r1 = bstart[b + 1];
    const int s = rowptr[r0], e = rowptr[r1];
    const int cnt = e - s, nrows = r1 - r0;
    const bool fits = cnt <= NNZ_CAP && nrows <= RB && cnt > 0;
    __syncthreads();   // shared state of the previous block is dead
    if (tid == 0) { s_nrun = 0; s_nseg = 0; s_total = 0; s_self = -1; }
    if (fits) {
      int P = 32;
      while (P < cnt) P <<= 1;
      for (int i = tid; i < P; i += WB_T) s_cols[i] = i < cnt ? colidx[s + i] : 0x7fffffff;
      __syncthreads();
      for (int k = 2; k <= P; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
          for (int i = tid; i < P; i += WB_T) {
            const int ixj = i ^ j;
            if (ixj > i) {
              const int a = s_cols[i], c = s_cols[ixj];
              const bool up = (i & k) == 0;
              if ((a > c) == up) { s_cols[i] = c; s_cols[ixj] = a; }
            }
          }
          __syncthreads();
        }
      // run starts, enumerated in order by warp 0 (a new run starts where the gap to the previous
      // column reaches MERGE_GAP; duplicates have gap -1)
      if (tid < 32) {
        int nrun = 0;
        for (int base = 0; base < cnt; base += 32) {
          const int k = base + tid;
          bool st = false;
          if (k < cnt) st = (k == 0) || (s_cols[k] - (s_cols[k - 1] + 1) >= MERGE_GAP);
          const unsigned bal = __ballot_sync(0xffffffffu, st);
          if (st) {
            const int slot = nrun + __popc(bal & ((1u << tid) - 1u));
            if (slot <= MAXSEG) s_start[slot] = k;
          }
          nrun += __popc(bal);
        }
        if (tid == 0) s_nrun = nrun;
      }
      __syncthreads();
      if (tid == 0 && s_nrun <= MAXSEG) {
        const int nrun = s_nrun;
        int nseg = 0, total = 0;
        bool ok = true;
        for (int q = 0; q < nrun; ++q) {
          const int first = s_cols[s_start[q]];
          const int last = s_cols[(q + 1 < nrun ? s_start[q + 1] : cnt) - 1];
          const int a = first / ALN * ALN;
          int l = (last + 1 - a + ALN - 1) / ALN * ALN;
          if ((long long)a + l > ncols_pad) l = (int)(ncols_pad - a);
          if (nseg > 0 && a < s_lo[nseg - 1] + s_len[nseg - 1]) {   // alignment made it touch the previous one
            const int nl = a + l - s_lo[nseg - 1];
            total += nl - s_len[nseg - 1];
            s_len[nseg - 1] = nl;
          } else {
            if (nseg == MAXSEG) { ok = false; break; }
            s_lo[nseg] = a; s_len[nseg] = l; total += l; ++nseg;
          }
        }
        if (ok && total <= wcap) {
          int acc = 0;
          for (int q = 0; q < nseg; ++q) { s_off[q] = acc; acc += s_len[q]; }
          int self = -1;
          for (int q = 0; q < nseg; ++q)
            if (r0 >= s_lo[q] && r1 <= s_lo[q] + s_len[q]) { self = s_off[q] + (r0 - s_lo[q]); break; }
          s_nseg = nseg; s_total = total; s_self = self;
        }
      }
    }
    __syncthreads();
    const int nseg = s_nseg;
    if (tid == 0) {
      BlockMeta m;
      m.row0 = r0; m.nrows = nrows; m.nnz = cnt; m.ent_off = 0;
      m.blob_off16 = (int)(blob_off[b] / 16);
      m.nseg = nseg; m.self_slot = s_self; m.wrows = s_total;
      for (int q = 0; q < MAXSEG; ++q) { m.seg_lo[q] = q < nseg ? s_lo[q] : 0; m.seg_len[q] = q < nseg ? s_len[q] : 0; }
      meta[b] = m;
      if (nseg > 0) atomicAdd(nwin, 1);
    }
    if (nseg == 0) continue;
    // the record: [ values nnzp | 1/diag rowsp | local columns nnzp | row offsets roffp ]
    const int nnzp = (cnt + 7) / 8 * 8;
    const int roffp = (nrows + 1 + 7) / 8 * 8;
    const int rowsp = dinv ? (nrows + 7) / 8 * 8 : 0;
    unsigned char* rec = blob + blob_off[b];
    T* v = reinterpret_cast<T*>(rec);
    T* dv = v + nnzp;
    unsigned short* lc = reinterpret_cast<unsigned short*>(dv + rowsp);
    unsigned short* ro = lc + nnzp;
    for (int i = tid; i < rowsp; i += WB_T) dv[i] = i < nrows ? dinv[r0 + i] : T(0);
    for (int i = tid; i < nnzp; i += WB_T) {
      T val = T(0);
      unsigned short l = 0;
      if (i < cnt) {
        val = vals[s + i];
        const int c = colidx[s + i];
        int k = 0;
        while (k + 1 < nseg && c >= s_lo[k + 1]) ++k;
        l = (unsigned short)(s_off[k] + (c - s_lo[k]));
      }
      v[i] = val;
      lc[i] = l;
    }
    for (int i = tid; i < roffp; i += WB_T) ro[i] = i <= nrows ? (unsigned short)(rowptr[r0 + i] - s) : (unsigned short)0;
  }
}

}  // namespace

template <typename T>
int build_windowed(cudaStream_t s, const int* d_rowptr, const int* d_colidx, const T* d_vals, int64_t nrows,
                   int64_t ncols_pad, int wcap, const T* d_dinv, DWin& out, std::string& err) {
  static_assert(sizeof(BlockMeta) == 96, "descriptor layout");
  out = DWin{};
  int* d_bstart = nullptr;
  int nb = 0;
  int rc = row_blocks(s, d_rowptr, nrows, RB, NNZ_CAP, &d_bstart, &nb, err);
  if (rc) return rc;
  struct Guard { int* p; ~Guard() { cudaFree(p); } } guard{d_bstart};
  if (nb <= 0) return 0;
  Scratch<long long> size, off;
  Scratch<int> nwin;
  CKD(size.alloc((size_t)nb + 1, s));
  CKD(off.alloc((size_t)nb + 1, s));
  CKD(nwin.alloc(1, s));
  CKD(cudaMemsetAsync(nwin.p, 0, sizeof(int), s));
  k_record_sizes<<<grid_for(nb + 1), TPB, 0, s>>>(nb, d_bstart, d_rowptr, (int)sizeof(T), d_dinv ? 1 : 0, size.p);
  CKD(cudaGetLastError());
  rc = exclusive_scan(s, size.p, off.p, (int64_t)nb + 1, err);
  if (rc) return rc;
  long long total = 0;
  CKD(cudaMemcpyAsync(&total, off.p + nb, sizeof(long long), cudaMemcpyDeviceToHost, s));
  CKD(cudaStreamSynchronize(s));
  const size_t blob_bytes = (size_t)total + 64;
  if (blob_bytes / 16 >= (size_t)std::numeric_limits<int>::max()) { err = "windowed records exceed 32 GB"; return -5; }
  BlockMeta* meta = nullptr;
  unsigned char* blob = nullptr;
  CKD(cudaMalloc(&meta, (size_t)nb * sizeof(BlockMeta)));
  cudaError_t e = cudaMalloc(&blob, blob_bytes);
  if (e != cudaSuccess) { cudaFree(meta); err = std::string("CUDA error ") + cudaGetErrorString(e) + " allocating the window records"; return -2; }
  cudaMemsetAsync(blob, 0, blob_bytes, s);
  k_win_build<T><<<std::max(1, std::min(nb, SMS * 16)), WB_T, 0, s>>>(nb, d_bstart, d_rowptr, d_colidx, d_vals, d_dinv,
                                                                      (long long)ncols_pad, wcap, off.p, meta, blob, nwin.p);
  int hw = 0;
  e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpyAsync(&hw, nwin.p, sizeof(int), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) {
    cudaFree(meta); cudaFree(blob);
    err = std::string("CUDA error ") + cudaGetErrorString(e) + " building the window records";
    return -2;
  }
  out.nblocks = nb;
  out.windowed_blocks = hw;
  if ((int64_t)hw * 2 < (int64_t)nb) {   // mostly scattered: the operator keeps the plain kernel
    cudaFree(meta);
    cudaFree(blob);
    return 0;
  }
  out.meta = meta;
  out.blob = blob;
  return 0;
}

// ---------------------------------------------------------------------------------------------
// stencil (DIA) detection + fill
// ---------------------------------------------------------------------------------------------
namespace {

template <typename T>
__global__ void k_dia_fill(int n, int nr, size_t ld, const int* __restrict__ ptr, const int* __restrict__ idx,
                           const T* __restrict__ val, T* __restrict__ dia, int* __restrict__ bad) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    T d[9];
#pragma unroll
    for (int s = 0; s < 9; ++s) d[s] = T(0);
    int miss = 0;
    for (int j = ptr[i]; j < ptr[i + 1]; ++j) {
      const int off = idx[j] - i;
      int s = -1;
      if (off >= -1 && off <= 1) s = 4 + off;
      else if (off >= nr - 1 && off <= nr + 1) s = 7 + (off - nr);
      else if (-off >= nr - 1 && -off <= nr + 1) s = 1 + (off + nr);
      if (s < 0) { miss = 1; continue; }
      // the neighbour must lie in the same or an adjacent raster column: a row offset that leaves
      // [0, nr) is a wrapped neighbour (NODATA before it shifted the numbering), not a stencil entry
      const int r = i % nr + s % 3 - 1;
      if (r < 0 || r >= nr) { miss = 1; continue; }
      const T v = val[j];
#pragma unroll
      for (int q = 0; q < 9; ++q) if (q == s) d[q] += v;
    }
#pragma unroll
    for (int s = 0; s < 9; ++s) dia[(size_t)s * ld + i] = d[s];
    if (miss) atomicOr(bad, 1);
  }
}

template <typename T> struct Bits;
template <> struct Bits<float> { using U = unsigned int; };
template <> struct Bits<double> { using U = unsigned long long; };

// bad = 1 unless every lower slot s < 4 of row i has the bit pattern of upper slot 8 - s of row i + off(s),
// or +0 where that row lies outside [0, n)
template <typename T>
__global__ void k_dia_sym_check(int n, int nr, size_t ld, const T* __restrict__ dia, int* __restrict__ bad) {
  using U = typename Bits<T>::U;
  const U* d = reinterpret_cast<const U*>(dia);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int miss = 0;
#pragma unroll
    for (int s = 0; s < 4; ++s) {
      const long long j = (long long)i + (s / 3 - 1) * (long long)nr + (s % 3 - 1);
      const U lo = d[(size_t)s * ld + i];
      miss |= (j >= 0 && j < n) ? lo != d[(size_t)(8 - s) * ld + j] : lo != U(0);
    }
    if (miss) atomicOr(bad, 1);
  }
}

}  // namespace

template <typename T>
int halve_dia(cudaStream_t s, T** d_dia, int64_t n, int nr, size_t ld, int* half, std::string& err) {
  *half = 0;
  Scratch<int> bad;
  CKD(bad.alloc(1, s));
  CKD(cudaMemsetAsync(bad.p, 0, sizeof(int), s));
  k_dia_sym_check<T><<<grid_for(n), TPB, 0, s>>>((int)n, nr, ld, *d_dia, bad.p);
  int hb = 1;
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpyAsync(&hb, bad.p, sizeof(int), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) {
    err = std::string("CUDA error ") + cudaGetErrorString(e) + " checking the stencil's symmetry";
    return -2;
  }
  if (hb) return 0;
  T* up = nullptr;
  CKD(cudaMalloc(&up, 5 * ld * sizeof(T)));
  e = cudaMemcpyAsync(up, *d_dia + 4 * ld, 5 * ld * sizeof(T), cudaMemcpyDeviceToDevice, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) {
    cudaFree(up);
    err = std::string("CUDA error ") + cudaGetErrorString(e) + " compacting the stencil";
    return -2;
  }
  cudaFree(*d_dia);
  *d_dia = up;
  *half = 1;
  return 0;
}

template <typename T>
int build_dia(cudaStream_t s, const int* d_rowptr, const int* d_colidx, const T* d_vals, int64_t n, T** d_dia, int* nr,
              size_t* ld, std::string& err) {
  *d_dia = nullptr;
  *nr = 0;
  *ld = 0;
  if (n < 16) return 0;
  // Invariant of the form: every entry (i, i + dc nr + dr) has (i % nr) + dr in [0, nr), i.e. row i is
  // raster cell (i % nr, i / nr) and its neighbours are cells of the 3 x 3 block around it.  The
  // tile-based kernels (k_stencil_prolong_jacobi reads the 9 neighbours from a shared-memory tile by
  // raster position) rely on it; an operator with a wrapped entry keeps the CSR / windowed path.
  // stride candidate from row 0: its first column beyond 1 (row 0 of a raster has neighbours 1, nr, nr + 1)
  int rp[2] = {0, 0};
  CKD(cudaMemcpyAsync(rp, d_rowptr, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
  CKD(cudaStreamSynchronize(s));
  const int len = rp[1] - rp[0];
  if (len < 2 || len > 9) return 0;
  int cols[9];
  CKD(cudaMemcpyAsync(cols, d_colidx + rp[0], (size_t)len * sizeof(int), cudaMemcpyDeviceToHost, s));
  CKD(cudaStreamSynchronize(s));
  int stride = 0;
  for (int q = 0; q < len; ++q)
    if (cols[q] > 1 && (stride == 0 || cols[q] < stride)) stride = cols[q];
  if (stride < 3 || stride >= n) return 0;
  const size_t l = ((size_t)n + 3) / 4 * 4;
  T* dia = nullptr;
  Scratch<int> bad;
  CKD(bad.alloc(1, s));
  CKD(cudaMemsetAsync(bad.p, 0, sizeof(int), s));
  CKD(cudaMalloc(&dia, 9 * l * sizeof(T)));
  cudaMemsetAsync(dia, 0, 9 * l * sizeof(T), s);
  k_dia_fill<T><<<grid_for(n), TPB, 0, s>>>((int)n, stride, l, d_rowptr, d_colidx, d_vals, dia, bad.p);
  int hb = 1;
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpyAsync(&hb, bad.p, sizeof(int), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess) {
    cudaFree(dia);
    err = std::string("CUDA error ") + cudaGetErrorString(e) + " building the stencil form";
    return -2;
  }
  if (hb) { cudaFree(dia); return 0; }
  *d_dia = dia;
  *nr = stride;
  *ld = l;
  return 0;
}

// ---------------------------------------------------------------------------------------------
// raster assembly with short-circuit polygons
// ---------------------------------------------------------------------------------------------
namespace {

__device__ __forceinline__ double stencil_weight(double a, double b, bool diagonal, bool avg_res) {
  const double s2 = 1.4142135623730951;                    // src/raster/pairwise.jl:364-367
  if (avg_res) return diagonal ? 1.0 / (s2 * (1.0 / a + 1.0 / b) / 2.0) : 1.0 / ((1.0 / a + 1.0 / b) / 2.0);
  return diagonal ? (a + b) / (2.0 * s2) : (a + b) / 2.0;
}

__global__ void k_poly_valid(int64_t ncell, const double* __restrict__ g, int* __restrict__ valid) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i <= ncell; i += (int64_t)gridDim.x * blockDim.x)
    valid[i] = (i < ncell && g[i] > 0.0) ? 1 : 0;
}

__global__ void k_poly_rep(int64_t ncell, const int* __restrict__ poly, const int* __restrict__ valid,
                           int* __restrict__ rep) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ncell; i += (int64_t)gridDim.x * blockDim.x)
    if (poly[i] > 0 && valid[i]) atomicMin(&rep[poly[i]], (int)i);      // first valid cell in memory order
}

// label = own rank among the valid cells (1-based), or the representative's for polygon cells
__global__ void k_poly_label(int64_t ncell, const int* __restrict__ poly, const int* __restrict__ valid,
                             const int* __restrict__ vrank, const int* __restrict__ rep, int* __restrict__ label,
                             int* __restrict__ used) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ncell; i += (int64_t)gridDim.x * blockDim.x) {
    int l = valid[i] ? vrank[i] + 1 : 0;
    if (poly && poly[i] > 0) {
      const int r = rep[poly[i]];
      if (r != 0x7fffffff) l = vrank[r] + 1;
    }
    label[i] = l;
    if (l) used[l] = 1;
  }
}

__global__ void k_poly_node(int64_t ncell, const int* __restrict__ label, const int* __restrict__ newid,
                            int* __restrict__ node) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ncell; i += (int64_t)gridDim.x * blockDim.x)
    node[i] = label[i] ? newid[label[i]] + 1 : 0;
}

// pass 0: items per cell (1 diagonal placeholder + 2 per adjacency to another node) ; pass 1: emit
template <int PASS>
__global__ void k_poly_items(int nrows, int ncols, int four, int avg_res, const double* __restrict__ g,
                             const int* __restrict__ node, long long* __restrict__ cnt, const long long* __restrict__ off,
                             int cb, unsigned long long* __restrict__ keys, double* __restrict__ vals) {
  const int64_t ncell = (int64_t)nrows * ncols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ncell + (PASS == 0 ? 1 : 0);
       i += (int64_t)gridDim.x * blockDim.x) {
    if (i == ncell) { cnt[i] = 0; continue; }
    const int a = node[i];
    long long k = 0;
    if (a) {
      const int r = (int)(i % nrows), c = (int)(i / nrows);
      const double gi = g[i] > 0.0 ? g[i] : 0.0;
      long long o = PASS ? off[i] : 0;
      const unsigned long long hi = (unsigned long long)(a - 1) << cb;
      if (PASS) { keys[o] = hi | (unsigned)(a - 1); vals[o] = 0.0; ++o; }   // every node has a diagonal entry
      k = 1;
      for (int q = 0; q < 9; ++q) {
        if (q == 4) continue;
        const int dr = q % 3 - 1, dc = q / 3 - 1;
        const bool diagonal = dr != 0 && dc != 0;
        if (four && diagonal) continue;
        const int rr = r + dr, cc = c + dc;
        if (rr < 0 || rr >= nrows || cc < 0 || cc >= ncols) continue;
        const int64_t j = (int64_t)cc * nrows + rr;
        const int b = node[j];
        if (!b || b == a) continue;                          // inside one node: dropped by laplacian!
        if (PASS) {
          const double gj = g[j] > 0.0 ? g[j] : 0.0;
          const double w = stencil_weight(gi, gj, diagonal, avg_res != 0);
          keys[o] = hi | (unsigned)(b - 1); vals[o] = -w; ++o;
          keys[o] = hi | (unsigned)(a - 1); vals[o] = w; ++o;
        }
        k += 2;
      }
    }
    if (!PASS) cnt[i] = k;
  }
}

}  // namespace

int assemble_raster_polygons(cudaStream_t s, int64_t nrows, int64_t ncols, const double* d_g, const int* d_poly,
                             int max_poly, int four, int avg_res, DCsr& out, int** d_nodemap, std::string& err) {
  int dev = 0;
  cudaGetDevice(&dev);
  ensure_pool(dev);
  out = DCsr{};
  *d_nodemap = nullptr;
  const int64_t ncell = nrows * ncols;
  const int g = grid_for(ncell + 1);
  Scratch<int> valid, vrank, rep, label, used, newid;
  CKD(valid.alloc((size_t)ncell + 1, s));
  CKD(vrank.alloc((size_t)ncell + 1, s));
  CKD(label.alloc((size_t)ncell, s));
  k_poly_valid<<<g, TPB, 0, s>>>(ncell, d_g, valid.p);
  CKD(cudaGetLastError());
  int rc = exclusive_scan(s, valid.p, vrank.p, ncell + 1, err);
  if (rc) return rc;
  int nvalid = 0;
  CKD(cudaMemcpyAsync(&nvalid, vrank.p + ncell, sizeof(int), cudaMemcpyDeviceToHost, s));
  CKD(cudaStreamSynchronize(s));
  if (nvalid <= 0) { err = "raster has no cell with conductance > 0"; return -1; }
  if (d_poly) {
    CKD(rep.alloc((size_t)max_poly + 1, s));
    k_fill_int<<<grid_for(max_poly + 1), TPB, 0, s>>>(rep.p, (int64_t)max_poly + 1, 0x7fffffff);   // "no valid cell"
    k_poly_rep<<<g, TPB, 0, s>>>(ncell, d_poly, valid.p, rep.p);
  }
  CKD(used.alloc((size_t)nvalid + 2, s));
  CKD(newid.alloc((size_t)nvalid + 2, s));
  k_zero_int<<<grid_for(nvalid + 2), TPB, 0, s>>>(used.p, nvalid + 2);
  k_poly_label<<<g, TPB, 0, s>>>(ncell, d_poly, valid.p, vrank.p, rep.p, label.p, used.p);
  CKD(cudaGetLastError());
  rc = exclusive_scan(s, used.p, newid.p, (int64_t)nvalid + 2, err);
  if (rc) return rc;
  int nnode = 0;
  CKD(cudaMemcpyAsync(&nnode, newid.p + nvalid + 1, sizeof(int), cudaMemcpyDeviceToHost, s));
  CKD(cudaStreamSynchronize(s));
  int* node = nullptr;
  CKD(cudaMalloc(&node, (size_t)ncell * sizeof(int)));
  k_poly_node<<<g, TPB, 0, s>>>(ncell, label.p, newid.p, node);
  valid.release(); vrank.release(); label.release(); used.release(); newid.release(); rep.release();
  // items -> sort -> CSR
  Scratch<long long> cnt, off;
  cudaError_t e = cnt.alloc((size_t)ncell + 1, s);
  if (e == cudaSuccess) e = off.alloc((size_t)ncell + 1, s);
  if (e != cudaSuccess) { cudaFree(node); CKD(e); }
  const int cb = bits_for(nnode);
  k_poly_items<0><<<g, TPB, 0, s>>>((int)nrows, (int)ncols, four, avg_res, d_g, node, cnt.p, nullptr, cb, nullptr, nullptr);
  rc = exclusive_scan(s, cnt.p, off.p, ncell + 1, err);
  long long m = 0;
  if (!rc) {
    e = cudaMemcpyAsync(&m, off.p + ncell, sizeof(long long), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { err = std::string("CUDA error ") + cudaGetErrorString(e); rc = -2; }
  }
  if (!rc && m >= (long long)std::numeric_limits<int>::max()) { err = "raster too large for int32 entry counts"; rc = -5; }
  if (rc) { cudaFree(node); return rc; }
  cnt.release();
  Scratch<unsigned long long> k0, k1;
  Scratch<double> v0, v1;
  e = k0.alloc((size_t)m, s);
  if (e == cudaSuccess) e = k1.alloc((size_t)m, s);
  if (e == cudaSuccess) e = v0.alloc((size_t)m, s);
  if (e == cudaSuccess) e = v1.alloc((size_t)m, s);
  if (e != cudaSuccess) { cudaFree(node); CKD(e); }
  k_poly_items<1><<<g, TPB, 0, s>>>((int)nrows, (int)ncols, four, avg_res, d_g, node, nullptr, off.p, cb, k0.p, v0.p);
  rc = sort_pairs(s, k0.p, k1.p, v0.p, v1.p, m, 2 * cb, err);
  if (!rc) {
    k0.release();
    v0.release();
    bool over = false;
    rc = compress_to_csr(s, m, k1.p, v1.p, nnode, nnode, cb, false, 0, 0, &over, out, err);
  }
  if (rc) { cudaFree(node); free_csr(out); return rc; }
  CKD(cudaStreamSynchronize(s));
  *d_nodemap = node;
  return 0;
}

namespace {
template <typename T>
__global__ void k_ell4_fill(int n, size_t ld, const int* __restrict__ ptr, const int* __restrict__ idx,
                            const T* __restrict__ val, int* __restrict__ ecol, T* __restrict__ eval, int* __restrict__ bad) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int a = ptr[i], len = ptr[i + 1] - a;
    if (len > 4) atomicOr(bad, 1);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const bool ok = q < len;
      ecol[(size_t)q * ld + i] = ok ? idx[a + q] : 0;
      eval[(size_t)q * ld + i] = ok ? val[a + q] : T(0);
    }
  }
}
}  // namespace

template <typename T>
int build_ell4(cudaStream_t s, const int* d_rowptr, const int* d_colidx, const T* d_vals, int64_t nrows, int** d_col,
               T** d_val, size_t* ld, std::string& err) {
  *d_col = nullptr;
  *d_val = nullptr;
  *ld = 0;
  if (nrows <= 0) return 0;
  const size_t l = ((size_t)nrows + 3) / 4 * 4;
  Scratch<int> bad;
  CKD(bad.alloc(1, s));
  CKD(cudaMemsetAsync(bad.p, 0, sizeof(int), s));
  int* ec = nullptr;
  T* ev = nullptr;
  CKD(cudaMalloc(&ec, 4 * l * sizeof(int)));
  cudaError_t e = cudaMalloc(&ev, 4 * l * sizeof(T));
  if (e != cudaSuccess) { cudaFree(ec); CKD(e); }
  k_ell4_fill<T><<<grid_for(nrows), TPB, 0, s>>>((int)nrows, l, d_rowptr, d_colidx, d_vals, ec, ev, bad.p);
  int hb = 1;
  e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaMemcpyAsync(&hb, bad.p, sizeof(int), cudaMemcpyDeviceToHost, s);
  if (e == cudaSuccess) e = cudaStreamSynchronize(s);
  if (e != cudaSuccess || hb) {
    cudaFree(ec);
    cudaFree(ev);
    if (e != cudaSuccess) { err = std::string("CUDA error ") + cudaGetErrorString(e) + " building the ELL prolongator"; return -2; }
    return 0;
  }
  *d_col = ec;
  *d_val = ev;
  *ld = l;
  return 0;
}

template int build_ell4<float>(cudaStream_t, const int*, const int*, const float*, int64_t, int**, float**, size_t*, std::string&);
template int build_ell4<double>(cudaStream_t, const int*, const int*, const double*, int64_t, int**, double**, size_t*, std::string&);

template int build_dia<float>(cudaStream_t, const int*, const int*, const float*, int64_t, float**, int*, size_t*, std::string&);
template int build_dia<double>(cudaStream_t, const int*, const int*, const double*, int64_t, double**, int*, size_t*, std::string&);
template int halve_dia<float>(cudaStream_t, float**, int64_t, int, size_t, int*, std::string&);
template int halve_dia<double>(cudaStream_t, double**, int64_t, int, size_t, int*, std::string&);

template int build_windowed<float>(cudaStream_t, const int*, const int*, const float*, int64_t, int64_t, int, const float*,
                                   DWin&, std::string&);
template int build_windowed<double>(cudaStream_t, const int*, const int*, const double*, int64_t, int64_t, int,
                                    const double*, DWin&, std::string&);

}  // namespace csb_dev

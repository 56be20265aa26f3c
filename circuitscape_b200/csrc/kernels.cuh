// kernels.cuh -- sm_90a device code for the batched PCG focal-pair solver.
//
// Data layout (DESIGN.md §3): CSR matrix (int32 rowptr/colidx, T values) replicated
// per GPU; every solver vector is a *panel*: n_pad x KT row-major (KT in {1,2,4,8}
// right-hand sides interleaved per node) so one SpMM gather of a neighbour reads
// KT*sizeof(T) contiguous bytes and the 12 B/nnz matrix stream is paid once per KT
// right-hand sides.  n_pad = n rounded up to 4 rows, so the element-wise kernels can use
// 16-byte vectors without tails; pad rows are zero except in X and P of a panel that
// starts from implicit zeros (cs_b200.cu panel_ends), where they are never read into a
// result: the stencil kernels stage rows >= n as zeros, every other reader of X stops at row n.
// All reductions are deterministic: warp tree -> per-CTA partial in a fixed slot ->
// combined in a fixed order by the last CTA to finish (ticket counter), which also
// derives the CG scalars on the device -- no host round trip, no float atomics.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace csb {

constexpr int NT = 256;          // threads per CTA for every kernel
constexpr int NWARP = NT / 32;
constexpr int NNZ_CAP = 2304;    // nnz staged in shared memory per row block (256 rows x 9)
constexpr int MAXKT = 8;

// Per-panel control block in device memory.
struct PanelCtl {
  double rho[MAXKT];      // r.z of the current iterate
  double pap[MAXKT];      // p.Ap
  double alpha[MAXKT];
  double beta[MAXKT];
  double tol[MAXKT];      // stop when sqrt(rho) <= tol   (atol + rtol*sqrt(rho0))
  double rho0[MAXKT];
  double resid[MAXKT];    // ||b - A x||^2 (true residual)
  double bnorm[MAXKT];    // ||b||^2
  double xsrc[MAXKT];     // x[src]  (shift);  R = xdst - xsrc
  double xdst[MAXKT];
  double maxpos[MAXKT];   // branch-current maxima (out.jl:281-287)
  double maxneg[MAXKT];
  double weight[MAXKT];   // cumulative-map multiplicity of the pair
  long long src[MAXKT];
  long long dst[MAXKT];
  int active[MAXKT];      // 1 while the column is iterating
  int iters[MAXKT];
  int iter;               // iterations done on this panel
  int itmax;
  int nactive;
  unsigned int ticket;    // last-CTA-done counter (self-resetting)
  int init;               // AMG path: 1 while the first z = M^-1 r is being formed
  double rtol, atol;      // stop-test parameters (AMG path reads them on the device)
  // stagnation guard (reduced-precision storage can plateau above rtol): a column whose
  // rho has not improved by 10 % for `stall_limit` iterations is frozen; the true-residual
  // gate then decides, exactly as it does after itmax in the reference (core.jl:639-641)
  double best[MAXKT];
  int stall[MAXKT];
  int stall_limit;
  int stalled[MAXKT];
  // fused CG step (k_stencil_cg): alpha of p_j in slot j mod 3 (j >= -1; slot 2 = 0 stands for the zero
  // p_{-1}).  A step reads the two slots of the deferred x updates and writes the third, so its CTAs never
  // read a slot its last CTA rewrites.
  double alpha_ring[3][MAXKT];
};

// ---------------------------------------------------------------------------
// streaming loads: matrix data is read once per kernel -> keep it out of L1 so L1
// stays available for the X-panel gathers.
// ---------------------------------------------------------------------------
__device__ __forceinline__ int ld_stream(const int* p) {
  int v;
  asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ float ld_stream(const float* p) {
  float v;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ double ld_stream(const double* p) {
  double v;
  asm volatile("ld.global.nc.L1::no_allocate.f64 %0, [%1];" : "=d"(v) : "l"(p));
  return v;
}

template <int KT> struct Log2 { static constexpr int v = 1 + Log2<KT / 2>::v; };
template <> struct Log2<1> { static constexpr int v = 0; };

template <typename T> struct Vec;
template <> struct Vec<double> { using type = double2; static constexpr int N = 2; };
template <> struct Vec<float> { using type = float4; static constexpr int N = 4; };

template <typename T> __device__ __forceinline__ void vload(const T* p, T (&v)[Vec<T>::N]) {
  using V = typename Vec<T>::type;
  const V t = *reinterpret_cast<const V*>(p);
  const T* q = reinterpret_cast<const T*>(&t);
#pragma unroll
  for (int i = 0; i < Vec<T>::N; ++i) v[i] = q[i];
}
template <typename T> __device__ __forceinline__ void vstore(T* p, const T (&v)[Vec<T>::N]) {
  using V = typename Vec<T>::type;
  V t;
  T* q = reinterpret_cast<T*>(&t);
#pragma unroll
  for (int i = 0; i < Vec<T>::N; ++i) q[i] = v[i];
  *reinterpret_cast<V*>(p) = t;
}

// ---------------------------------------------------------------------------
// Deterministic grid reduction of per-column quantities.
// Thread `tid` holds val[q][i], q < NV, i < VEC, where slot i belongs to panel
// column (tid*VEC + i) % KT (true for the element-wise kernels whose element index
// is e = (global_thread*VEC + i) + k*stride with stride % KT == 0, and for SpMM with
// VEC = 1, column = tid % KT).
// Steps: fold equal-column slots -> warp xor-tree over lanes of the same column
// class -> fixed-order sum over the 8 warps -> partials[blockIdx][q][c] -> the last
// CTA (ticket) combines all CTAs in a fixed order into out[q*KT + c] (shared).
// Returns true for every thread of the last CTA.
// ---------------------------------------------------------------------------
template <int KT, int VEC, int NV, bool IS_MAX, int NTH = NT>
__device__ __forceinline__ bool grid_reduce(double (&val)[NV][VEC], double* partials,
                                            unsigned int* ticket, double* s_warp /*NWARP*NV*KT*/,
                                            double* s_tree /*NTH*/, double* out /*NV*KT*/) {
  constexpr int NWARP = NTH / 32;
  constexpr int NT = NTH;
  constexpr int S = VEC < KT ? VEC : KT;  // distinct columns held per thread
  constexpr int G = KT / S;               // lane classes
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int q = 0; q < NV; ++q) {
#pragma unroll
    for (int i = S; i < VEC; ++i)
      val[q][i % S] = IS_MAX ? fmax(val[q][i % S], val[q][i]) : val[q][i % S] + val[q][i];
#pragma unroll
    for (int i = 0; i < S; ++i) {
#pragma unroll
      for (int off = 16; off >= G; off >>= 1) {
        const double o = __shfl_xor_sync(0xffffffffu, val[q][i], off);
        val[q][i] = IS_MAX ? fmax(val[q][i], o) : val[q][i] + o;
      }
    }
  }
  __syncthreads();  // s_warp may still be read by a previous use
  if (lane < G) {
#pragma unroll
    for (int q = 0; q < NV; ++q)
#pragma unroll
      for (int i = 0; i < S; ++i) s_warp[(warp * NV + q) * KT + lane * S + i] = val[q][i];
  }
  __syncthreads();
  if (tid < NV * KT) {
    double acc = s_warp[tid];
    for (int w = 1; w < NWARP; ++w) {
      const double v = s_warp[w * NV * KT + tid];
      acc = IS_MAX ? fmax(acc, v) : acc + v;
    }
    partials[(size_t)blockIdx.x * (NV * KT) + tid] = acc;
  }
  __shared__ bool is_last;
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const unsigned int t = atomicAdd(ticket, 1u);
    is_last = (t == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return false;
  __threadfence();
  constexpr int NOUT = NV * KT;                 // <= 16
  constexpr int LANES = NT / NOUT > 32 ? 32 : NT / NOUT;
  const int o = tid / LANES, l = tid % LANES;
  double acc = IS_MAX ? -1.0e300 : 0.0;
  if (o < NOUT) {
    for (int b = l; b < (int)gridDim.x; b += LANES) {
      const double v = __ldcg(&partials[(size_t)b * NOUT + o]);
      acc = IS_MAX ? fmax(acc, v) : acc + v;
    }
  }
  s_tree[tid] = acc;
  __syncthreads();
#pragma unroll
  for (int s = LANES / 2; s > 0; s >>= 1) {
    if (o < NOUT && l < s) {
      const double a = s_tree[tid], b2 = s_tree[tid + s];
      s_tree[tid] = IS_MAX ? fmax(a, b2) : a + b2;
    }
    __syncthreads();
  }
  if (o < NOUT && l == 0) out[o] = s_tree[tid];
  if (tid == 0) *ticket = 0u;  // self-reset for the next kernel on this stream
  __syncthreads();
  return true;
}

// CG bookkeeping after z = M^-1 r and rho_new[c] = r.z are known (general preconditioner).
// First call of a solve (ctl->init): thresholds and activity; later: beta, stop test, freeze.
template <int KT>
__device__ __forceinline__ void cg_after_precond(PanelCtl* ctl, const double* rho_new) {
  const int c = threadIdx.x;
  const int init = ctl->init;
  const int it = ctl->iter + 1;
  __syncthreads();
  if (c < KT) {
    const double rn = fabs(rho_new[c]);
    if (init) {
      const double tol = ctl->atol + ctl->rtol * sqrt(rn);
      ctl->rho[c] = rn;
      ctl->rho0[c] = rn;
      ctl->tol[c] = tol;
      ctl->active[c] = (rn > 0.0 && sqrt(rn) > tol && ctl->itmax > 0) ? 1 : 0;
      ctl->iters[c] = 0;
      ctl->alpha[c] = 0.0;
      ctl->alpha_ring[0][c] = ctl->alpha_ring[1][c] = ctl->alpha_ring[2][c] = 0.0;
      ctl->beta[c] = 0.0;
      ctl->best[c] = rn;
      ctl->stall[c] = 0;
      ctl->stalled[c] = 0;
    } else if (ctl->active[c]) {
      const double ro = ctl->rho[c];
      ctl->beta[c] = ro > 0.0 ? rn / ro : 0.0;
      ctl->rho[c] = rn;
      ctl->iters[c] = it;
      if (rn < 0.81 * ctl->best[c]) { ctl->best[c] = rn; ctl->stall[c] = 0; }
      else if (++ctl->stall[c] >= ctl->stall_limit && ctl->stall_limit > 0) { ctl->stalled[c] = 1; ctl->active[c] = 0; }
      if (!(sqrt(rn) > ctl->tol[c]) || it >= ctl->itmax) ctl->active[c] = 0;
    } else {
      ctl->beta[c] = 0.0;
    }
  }
  __syncthreads();
  if (c == 0) {
    int na = 0;
    for (int k = 0; k < KT; ++k) na += ctl->active[k];
    ctl->nactive = na;
    ctl->iter = init ? 0 : it;
    ctl->init = 0;
  }
}

#define CSB_REDUCE_SMEM(NV, KT)                         \
  __shared__ double s_warp[NWARP * (NV) * (KT)];        \
  __shared__ double s_tree[NT];                         \
  __shared__ double s_out[(NV) * (KT)];
#define CSB_REDUCE_SMEM_W(NV, KT)                       \
  __shared__ double s_warp[(WTT / 32) * (NV) * (KT)];   \
  __shared__ double s_tree[WTT];                        \
  __shared__ double s_out[(NV) * (KT)];

// ---------------------------------------------------------------------------
// SpMM  Y = op(A X)  on an n x KT panel, CSR "row-block streaming":
//   a CTA takes a block of consecutive rows whose nnz fit NNZ_CAP, streams that
//   contiguous slice of vals/colidx into shared memory with coalesced loads, then
//   LPR lanes per (row, c) walk the row out of shared memory and gather X[col][c]
//   (KT lanes read KT*sizeof(T) contiguous bytes; for the raster stencil the columns
//   of neighbouring rows are neighbouring -> sectors are shared across the warp).
// The same kernel serves the operator of every multigrid level, the prolongators
// and the restrictions; the epilogue (MODE) fuses what follows the product:
//   SP_PLAIN       Y = A X
//   SP_CG          Y = A X ; dot(X, Y) per column ; last CTA: alpha = rho / pAp
//   SP_RESNORM     Y = B - A X ; ||Y||^2, ||B||^2 per column      (true-residual gate)
//   SP_RES         Y = B - A X
//   SP_JACOBI      Y = X + omega Dinv (B - A X)                    (damped-Jacobi sweep)
//   SP_JACOBI_DOT  same ; dot(B, Y) per column ; last CTA: CG beta / stop test
//                  (B = r, Y = z = M^-1 r: the last kernel of the V-cycle)
//   SP_ADD         Y += A X                                        (prolongate + correct)
// A row longer than NNZ_CAP (polygon hub / power-law node) is its own block and is
// reduced by the whole CTA.
// ---------------------------------------------------------------------------
enum { SP_PLAIN = 0, SP_CG = 1, SP_RESNORM = 2, SP_RES = 3, SP_JACOBI = 4, SP_JACOBI_DOT = 5, SP_ADD = 6,
       SP_RES0 = 7 /* stencil form only: Y = B - A (omega D^-1 B), the residual after the zero-guess Jacobi sweep */ };

template <typename T> struct CsrDev {
  const int* rowptr;
  const int* colidx;
  const T* vals;
  const int* bstart;   // row-block starts (nblocks + 1)
  int nblocks;
  int nrows;
};

template <typename T> struct SpmmEpi {
  const T* B;
  const T* dinv;
  T omega;
  PanelCtl* ctl;
  double* partials;
  int pair_b;          // k_stencil_pipe SP_RESNORM: b is ctl's pairs rule (pair_rhs_val), B not read, Y not stored
};

// entry (row, c) of a pairs panel's right-hand side: -1 at src, +1 at dst where both are nodes and differ
// (core.jl:224-226, 459-460); what k_pair_rhs leaves in a zeroed B.  Host-callable for the CPU check of
// k_panel_start (tests/panel_start_harness.cu).
template <typename T>
__host__ __device__ __forceinline__ T pair_rhs_val(const PanelCtl* ctl, long long row, int c) {
  const long long s = ctl->src[c], d = ctl->dst[c];
  if (s < 0 || d < 0 || s == d) return T(0);
  return row == d ? T(1) : row == s ? T(-1) : T(0);
}

// element e of a KT-wide pairs panel (row e / KT, column e % KT), as k_panel_start forms it
template <typename T, int KT>
__host__ __device__ __forceinline__ T pair_rhs_at(const PanelCtl* ctl, size_t e) {
  return pair_rhs_val<T>(ctl, (long long)(e / KT), (int)(e % KT));
}

template <typename T, int MODE>
__device__ __forceinline__ void spmm_epilogue(int row, size_t o, T acc, const T* __restrict__ X,
                                              T* __restrict__ Y, const SpmmEpi<T>& ep, double& dot0,
                                              double& dot1) {
  if (MODE == SP_PLAIN) {
    Y[o] = acc;
  } else if (MODE == SP_CG) {
    Y[o] = acc;
    dot0 += (double)acc * (double)X[o];
  } else if (MODE == SP_RESNORM) {
    const T bb = ep.B[o];
    const T rr = bb - acc;
    Y[o] = rr;
    dot0 += (double)rr * (double)rr;
    dot1 += (double)bb * (double)bb;
  } else if (MODE == SP_RES) {
    Y[o] = ep.B[o] - acc;
  } else if (MODE == SP_JACOBI || MODE == SP_JACOBI_DOT) {
    const T bb = ep.B[o];
    const T yn = X[o] + ep.omega * ep.dinv[row] * (bb - acc);
    Y[o] = yn;
    if (MODE == SP_JACOBI_DOT) dot0 += (double)bb * (double)yn;
  } else {
    Y[o] += acc;
  }
}

template <typename T, int KT, int MODE, int LPR>
__global__ void __launch_bounds__(NT)
k_spmm(const CsrDev<T> A, const T* __restrict__ X, T* __restrict__ Y, const SpmmEpi<T> ep) {
  __shared__ T s_val[NNZ_CAP];
  __shared__ int s_col[NNZ_CAP];
  __shared__ double s_long[NT];
  const int tid = threadIdx.x;
  const int c = tid % KT;
  const int lr = (tid / KT) % LPR;          // lane within the row
  constexpr int RPP = NT / (KT * LPR);      // rows per pass
  double dot0 = 0.0, dot1 = 0.0;

  for (int blk = blockIdx.x; blk < A.nblocks; blk += gridDim.x) {
    const int r0 = A.bstart[blk], r1 = A.bstart[blk + 1];
    const int s = A.rowptr[r0], e = A.rowptr[r1];
    const int cnt = e - s;
    __syncthreads();
    if (cnt <= NNZ_CAP) {
      constexpr int U = NNZ_CAP / NT;   // 9 matrix entries per thread per row block
      if constexpr (KT == 1 && LPR == 1) {
        // single right-hand side ("stream-gather"): thread i streams entry i of the block
        // (coalesced vals/colidx), gathers x[col] and parks the PRODUCT in shared memory;
        // all U entries' loads are issued before any use (U*2 streaming + U gather loads
        // in flight per thread); then one thread per row sums its products.
        T v[U];
        int ci[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int i = tid + u * NT;
          if (i < cnt) {
            v[u] = ld_stream(A.vals + s + i);
            ci[u] = ld_stream(A.colidx + s + i);
          } else {
            v[u] = T(0);
            ci[u] = 0;
          }
        }
        T xv[U];
#pragma unroll
        for (int u = 0; u < U; ++u) xv[u] = X[ci[u]];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int i = tid + u * NT;
          if (i < cnt) s_val[i] = v[u] * xv[u];
        }
        __syncthreads();
        const int row = r0 + tid;
        if (row < r1) {
          const int a = A.rowptr[row] - s, b = A.rowptr[row + 1] - s;
          T acc = T(0);
          for (int j = a; j < b; ++j) acc += s_val[j];
          spmm_epilogue<T, MODE>(row, (size_t)row, acc, X, Y, ep, dot0, dot1);
        }
      } else {
        {
          T v[U];
          int ci[U];
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int i = tid + u * NT;
            if (i < cnt) {
              v[u] = ld_stream(A.vals + s + i);
              ci[u] = ld_stream(A.colidx + s + i);
            }
          }
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const int i = tid + u * NT;
            if (i < cnt) {
              s_val[i] = v[u];
              s_col[i] = ci[u];
            }
          }
        }
        __syncthreads();
        const int nr = r1 - r0;
        for (int base = 0; base < nr; base += RPP) {      // uniform trip count: shuffles below
          const int rl = base + tid / (KT * LPR);
          const bool valid = rl < nr;
          const int row = r0 + rl;
          T acc = T(0);
          if (valid) {
            const int a = A.rowptr[row] - s, b = A.rowptr[row + 1] - s;
#pragma unroll 3
            for (int j = a + lr; j < b; j += LPR) acc += s_val[j] * X[(size_t)s_col[j] * KT + c];
          }
#pragma unroll
          for (int off = KT; off < KT * LPR; off <<= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
          if (valid && lr == 0) spmm_epilogue<T, MODE>(row, (size_t)row * KT + c, acc, X, Y, ep, dot0, dot1);
        }
      }
    } else {
      const int row = r0;  // long row: r1 == r0 + 1
      double acc = 0.0;
      constexpr int GRP = NT / KT;
      for (int base = 0; base < cnt; base += NNZ_CAP) {
        const int m = min(NNZ_CAP, cnt - base);
        __syncthreads();
        for (int i = tid; i < m; i += NT) {
          s_val[i] = ld_stream(A.vals + s + base + i);
          s_col[i] = ld_stream(A.colidx + s + base + i);
        }
        __syncthreads();
        for (int j = tid / KT; j < m; j += GRP)
          acc += (double)s_val[j] * (double)X[(size_t)s_col[j] * KT + c];
      }
      __syncthreads();
      s_long[tid] = acc;
      __syncthreads();
      if (tid < KT) {
        double t = 0.0;
        for (int g = 0; g < GRP; ++g) t += s_long[g * KT + tid];
        spmm_epilogue<T, MODE>(row, (size_t)row * KT + tid, (T)t, X, Y, ep, dot0, dot1);
      }
    }
  }
  if (MODE == SP_CG) {
    CSB_REDUCE_SMEM(1, KT)
    double v[1][1] = {{dot0}};
    if (grid_reduce<KT, 1, 1, false>(v, ep.partials, &ep.ctl->ticket, s_warp, s_tree, s_out)) {
      if (tid < KT) {
        const double pap = s_out[tid];
        ep.ctl->pap[tid] = pap;
        ep.ctl->alpha[tid] = (ep.ctl->active[tid] && pap > 0.0) ? ep.ctl->rho[tid] / pap : 0.0;
      }
    }
  } else if (MODE == SP_RESNORM) {
    CSB_REDUCE_SMEM(2, KT)
    double v[2][1] = {{dot0}, {dot1}};
    if (grid_reduce<KT, 1, 2, false>(v, ep.partials, &ep.ctl->ticket, s_warp, s_tree, s_out)) {
      if (tid < KT) {
        ep.ctl->resid[tid] = s_out[tid];
        ep.ctl->bnorm[tid] = s_out[KT + tid];
      }
    }
  } else if (MODE == SP_JACOBI_DOT) {
    CSB_REDUCE_SMEM(1, KT)
    double v[1][1] = {{dot0}};
    if (grid_reduce<KT, 1, 1, false>(v, ep.partials, &ep.ctl->ticket, s_warp, s_tree, s_out))
      cg_after_precond<KT>(ep.ctl, s_out);
  }
}

// ---------------------------------------------------------------------------
// TMA-staged SpMM on the windowed row-block form (win_host.hpp).
//
// Persistent CTAs (one per SM, WT threads) walk the row blocks with a two-stage
// shared-memory ring.  For block i+1 ONE elected thread arms an mbarrier with the
// byte count and issues cp.async.bulk copies (the TMA engine; no registers, no LSU
// instructions) of: the X-panel segments the block's columns fall into, the block's
// B rows when the epilogue needs them, its slice of values, the 16-bit window-local
// column indices and the row offsets -- while all WT threads compute block i out of
// shared memory only.  Global memory sees nothing but large sequential bulk reads
// and the coalesced Y stores.  Blocks flagged nseg == 0 (hub rows, scattered columns)
// use direct gathers on the plain CSR inside the same kernel.
// ---------------------------------------------------------------------------
constexpr int W_RB = 128;               // == csb_win::RB
constexpr int W_NNZ = 1152;             // == csb_win::NNZ_CAP
constexpr int W_WCAP = 512;             // == csb_win::WCAP
constexpr int W_WCAP_WIDE = 1024;       // == csb_win::WCAP_WIDE
constexpr int W_MAXSEG = 8;
constexpr int W_SMEM_BUDGET = 214 * 1024;   // dynamic shared memory the ring may use

struct WinMeta {                        // == csb_win::BlockMeta
  int row0, nrows, nnz, ent_off, blob_off16, nseg, self_slot, wrows;
  int seg_lo[W_MAXSEG];
  int seg_len[W_MAXSEG];
};

template <typename T> struct WinCsr {
  const WinMeta* meta;
  const unsigned char* blob;   // per block: [values | (1/diag) | 16-bit local columns | 16-bit row offsets]
  int has_dinv;                // records of square operators carry 1/diag of their rows
  // plain CSR for the direct-gather blocks
  const int* rowptr;
  const int* colidx;
  const T* vals;
  int nblocks;
};

__device__ __forceinline__ unsigned smem_u32(const void* p) {
  return (unsigned)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes,
                                         unsigned long long* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(unsigned long long* bar, unsigned parity) {
  unsigned ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}

template <typename T, int KT, int MODE, bool WIDE = false> struct WinSmem {
  // SP_ADD stages the rows of Y it updates through the B slot (ep.B = Y): no synchronous
  // global load is left in any epilogue
  static constexpr bool NEEDB = (MODE == SP_RESNORM || MODE == SP_RES || MODE == SP_JACOBI ||
                                 MODE == SP_JACOBI_DOT || MODE == SP_ADD);
  static constexpr int al(int x) { return (x + 127) / 128 * 128; }
  static constexpr int XW = al((WIDE ? W_WCAP_WIDE : W_WCAP) * KT * (int)sizeof(T));
  static constexpr int BW = NEEDB ? al((W_RB + 8) * KT * (int)sizeof(T)) : 0;
  static constexpr int VW = al(W_NNZ * ((int)sizeof(T) + 2) + (W_RB + 8) * (2 + (int)sizeof(T)));   // the block's record
  static constexpr int OFF_X = 0;
  static constexpr int OFF_B = OFF_X + XW;
  static constexpr int OFF_V = OFF_B + BW;
  static constexpr int STAGE = OFF_V + VW;
  static constexpr int NSTAGE = (W_SMEM_BUDGET / STAGE) >= 6 ? 6 : (W_SMEM_BUDGET / STAGE);   // >= 3 for every T, KT
  static constexpr int TOTAL = NSTAGE * STAGE;
};

// Warp-specialised: warps 0..15 (WC threads) consume, warp 16 produces.
// The producer walks the CTA's contiguous range of row blocks: its lanes fetch the
// block's 96-byte descriptor with ONE coalesced load, lane 0 posts a 16-byte header
// (row0, nrows, nseg, self slot) into the stage and either arms full[stage] with the
// byte count and issues the bulk copies, or (direct-gather block) just arrives.
// Consumers wait full[stage], compute from shared memory, and each consumer warp
// arrives on empty[stage]; the producer waits empty[stage] before refilling it.
constexpr int WC = 512;                 // consumer threads
constexpr int WTT = WC + 32;            // + producer warp

__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void consumer_sync() {   // named barrier 1: consumers only
  asm volatile("bar.sync 1, %0;" ::"r"(WC) : "memory");
}

// N contiguous values through the widest aligned vector access (<= 16 B); p is aligned to
// min(16, N*sizeof(T)) bytes by construction (rows of KT values, column groups of CPT).
// NC: through the read-only path, for data no thread of the kernel writes that the compiler cannot prove so.
template <typename T, int N, bool NC = false>
__device__ __forceinline__ void ldvec(const T* p, T (&v)[N]) {
  constexpr int BYTES = N * (int)sizeof(T);
  if constexpr (BYTES >= 16) {
    constexpr int PER = 16 / (int)sizeof(T);
#pragma unroll
    for (int k = 0; k < N / PER; ++k) {
      const uint4* a = reinterpret_cast<const uint4*>(p + k * PER);
      const uint4 t = NC ? __ldg(a) : *a;
      const T* q = reinterpret_cast<const T*>(&t);
#pragma unroll
      for (int i = 0; i < PER; ++i) v[k * PER + i] = q[i];
    }
  } else if constexpr (BYTES == 8) {
    const uint2* a = reinterpret_cast<const uint2*>(p);
    const uint2 t = NC ? __ldg(a) : *a;
    const T* q = reinterpret_cast<const T*>(&t);
#pragma unroll
    for (int i = 0; i < N; ++i) v[i] = q[i];
  } else {
    v[0] = NC ? __ldg(p) : p[0];
  }
}
template <typename T, int N>
__device__ __forceinline__ void stvec(T* p, const T (&v)[N]) {
  constexpr int BYTES = N * (int)sizeof(T);
  if constexpr (BYTES >= 16) {
    constexpr int PER = 16 / (int)sizeof(T);
#pragma unroll
    for (int k = 0; k < N / PER; ++k) {
      uint4 t;
      T* q = reinterpret_cast<T*>(&t);
#pragma unroll
      for (int i = 0; i < PER; ++i) q[i] = v[k * PER + i];
      *reinterpret_cast<uint4*>(p + k * PER) = t;
    }
  } else if constexpr (BYTES == 8) {
    uint2 t;
    T* q = reinterpret_cast<T*>(&t);
#pragma unroll
    for (int i = 0; i < N; ++i) q[i] = v[i];
    *reinterpret_cast<uint2*>(p) = t;
  } else {
    p[0] = v[0];
  }
}

// Work decomposition of the windowed kernel.  A ring stage holds SB consecutive row
// blocks ("super-block"); consumer group g = tid / (WC/SB) owns sub-block g.  Within a
// group a row is served by CG column groups (CPT = one 16-byte vector of the panel row
// each -> conflict-free LDS.128 across the lanes of a row) times LPR lanes that split
// the row's entries.  Sizes are chosen so that a full 128-row block occupies every
// lane of its group once (narrow rows) and each lane has >= BATCH independent
// load chains in flight.
template <typename T, int KT, bool WIDE> struct WinMap {
  static constexpr int V16 = 16 / (int)sizeof(T);
  static constexpr int CPT = KT < V16 ? KT : V16;       // panel columns per thread
  static constexpr int CG = KT / CPT;                   // column groups per row
  static constexpr int SB = CG >= 4 ? 1 : (CG == 2 ? 1 : (KT == 1 ? 4 : 2));   // blocks per stage
  static constexpr int GT = WC / SB;                    // threads per consumer group
  static constexpr int LPR0 = (GT / W_RB) / CG < 1 ? 1 : (GT / W_RB) / CG;
  static constexpr int LPR = WIDE ? (LPR0 * 4 * CG > 32 ? 32 / CG : LPR0 * 4) : LPR0;
  static constexpr int LPRW = CG * LPR;                 // lanes per row
  static constexpr int RPP = GT / LPRW;                 // rows per pass of a group
  static constexpr int BATCH = WIDE ? 3 : (9 + LPR - 1) / LPR;   // entries per lane per batch
};

template <typename T, int KT, int MODE, bool WIDE> struct WinSmem2 {
  using S1 = WinSmem<T, KT, MODE, WIDE>;
  static constexpr int SB = WinMap<T, KT, WIDE>::SB;
  static constexpr int STAGE = S1::STAGE * SB;
  static constexpr int NSTAGE = (W_SMEM_BUDGET / STAGE) >= 6 ? 6 : (W_SMEM_BUDGET / STAGE);
  static constexpr int TOTAL = NSTAGE * STAGE;
};

template <typename T, int KT, int MODE, bool WIDE>
__global__ void __launch_bounds__(WTT, 1)
k_spmm_win(const WinCsr<T> A, const T* __restrict__ X, T* __restrict__ Y, const SpmmEpi<T> ep) {
  using SM = WinSmem<T, KT, MODE, WIDE>;
  using S2 = WinSmem2<T, KT, MODE, WIDE>;
  using MP = WinMap<T, KT, WIDE>;
  constexpr int NS = S2::NSTAGE;
  constexpr int SB = MP::SB, CPT = MP::CPT, CG = MP::CG, LPR = MP::LPR, LPRW = MP::LPRW;
  constexpr int GT = MP::GT, RPP = MP::RPP, BATCH = MP::BATCH;
  static_assert(NS >= 2, "ring needs two stages");
  extern __shared__ __align__(128) unsigned char dsm[];
  __shared__ unsigned long long full[NS], empty[NS];
  __shared__ int4 hdr[NS][SB];
  __shared__ double s_long[WC];
  const int tid = threadIdx.x;
  const bool producer = tid >= WC;
  double dot0[CPT], dot1[CPT];
#pragma unroll
  for (int i = 0; i < CPT; ++i) dot0[i] = dot1[i] = 0.0;

  if (tid == 0) {
#pragma unroll
    for (int i = 0; i < NS; ++i) {
      mbar_init(&full[i], SB);          // one arrival per sub-block
      mbar_init(&empty[i], WC / 32);    // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // super-blocks are dealt round-robin: at any time the CTAs work on a front of
  // gridDim.x * SB consecutive row blocks, so the halo strips of X re-read by
  // neighbouring blocks are still in L2.
  const int nsuper = (A.nblocks + SB - 1) / SB;

  if (producer) {
    const int lane = tid & 31;
    const int* mw = reinterpret_cast<const int*>(A.meta);
    constexpr int MWORDS = (int)(sizeof(WinMeta) / 4);   // 24
    // Descriptor prefetch: slots q = 0,1,2,... enumerate (stage iteration, sub-block) pairs of
    // this CTA; the 96-byte descriptors of the next PD slots are already in flight (one
    // coalesced load each) while the current PD slots are being issued.
    constexpr int PD = 4;
    const int nmine = nsuper > (int)blockIdx.x ? (nsuper - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    const int nslots = nmine * SB;
    auto slot_block = [&](int q) { return ((int)blockIdx.x + (q / SB) * (int)gridDim.x) * SB + (q % SB); };
    auto fetch = [&](int q) {
      const int blk = q < nslots ? slot_block(q) : A.nblocks;
      return (blk < A.nblocks && lane < MWORDS) ? mw[(size_t)blk * MWORDS + lane] : 0;
    };
    int wcur[PD], wnxt[PD];
#pragma unroll
    for (int u = 0; u < PD; ++u) wcur[u] = fetch(u);
    for (int q0 = 0; q0 < nslots; q0 += PD) {
#pragma unroll
      for (int u = 0; u < PD; ++u) wnxt[u] = fetch(q0 + PD + u);
#pragma unroll
      for (int u = 0; u < PD; ++u) {
        const int q = q0 + u;
        if (q >= nslots) break;
        const int it = q / SB, g = q % SB;
        const int st = it % NS;
        const int blk = slot_block(q);
        if (g == 0 && it >= NS) {
          const unsigned par = ((it / NS) - 1) & 1u;
          while (!mbar_try_wait(&empty[st], par)) {}
        }
        if (blk >= A.nblocks) {               // tail of the last super-block
          if (lane == 0) { hdr[st][g] = make_int4(0, 0, -1, 0); mbar_arrive(&full[st]); }
          continue;
        }
        const int w = wcur[u];
        // meta words: 0 row0, 1 nrows, 2 nnz, 3 ent_off, 4 roff_off, 5 nseg, 6 self_slot, 7 wrows,
        //             8.. seg_lo, 16.. seg_len
        const int row0 = __shfl_sync(0xffffffffu, w, 0), nrows = __shfl_sync(0xffffffffu, w, 1);
        const int nnz = __shfl_sync(0xffffffffu, w, 2);
        const int blob16 = __shfl_sync(0xffffffffu, w, 4), nseg = __shfl_sync(0xffffffffu, w, 5);
        const int self = __shfl_sync(0xffffffffu, w, 6), wrows = __shfl_sync(0xffffffffu, w, 7);
        const int my_lo = __shfl_sync(0xffffffffu, w, 8 + (lane & 7));
        const int my_len = __shfl_sync(0xffffffffu, w, 16 + (lane & 7));
        int slot = (lane < nseg) ? my_len : 0;    // exclusive prefix of segment lengths
#pragma unroll
        for (int off = 1; off < 8; off <<= 1) {
          const int v = __shfl_up_sync(0xffffffffu, slot, off);
          if ((lane & 7) >= off) slot += v;
        }
        slot -= (lane < nseg) ? my_len : 0;
        unsigned char* base = dsm + st * S2::STAGE + g * SM::STAGE;
        const int nnzp = (nnz + 7) / 8 * 8;
        if (lane == 0) hdr[st][g] = make_int4(row0, nrows | (nseg << 16), self, nnzp);
        if (nseg == 0) {
          if (lane == 0) mbar_arrive(&full[st]);
          continue;
        }
        const int roffp = (nrows + 1 + 7) / 8 * 8;
        const int b_lo = row0 & ~3;
        const int b_len = ((row0 + nrows + 3) & ~3) - b_lo;
        const int rowsp = A.has_dinv ? (nrows + 7) / 8 * 8 : 0;
        const unsigned blob_bytes = (unsigned)(nnzp * ((int)sizeof(T) + 2) + roffp * 2 + rowsp * (int)sizeof(T));
        if (lane == 0) {
          unsigned bytes = (unsigned)(wrows * KT * (int)sizeof(T)) + blob_bytes;
          if (SM::NEEDB) bytes += (unsigned)(b_len * KT * (int)sizeof(T));
          mbar_expect_tx(&full[st], bytes);
        }
        __syncwarp();
        // lanes 0..nseg-1: one X segment each; lane 8: B rows; lane 9: the matrix blob
        if (lane < nseg)
          bulk_g2s(base + SM::OFF_X + (size_t)slot * KT * sizeof(T), X + (size_t)my_lo * KT,
                   (unsigned)(my_len * KT * (int)sizeof(T)), &full[st]);
        if (SM::NEEDB && lane == 8)
          bulk_g2s(base + SM::OFF_B, ep.B + (size_t)b_lo * KT, (unsigned)(b_len * KT * (int)sizeof(T)), &full[st]);
        if (lane == 9) bulk_g2s(base + SM::OFF_V, A.blob + (size_t)blob16 * 16, blob_bytes, &full[st]);
      }
#pragma unroll
      for (int u = 0; u < PD; ++u) wcur[u] = wnxt[u];
    }
  } else {
    const int g = tid / GT;                        // consumer group = sub-block
    const int gt = tid % GT;                       // thread within the group
    const int cg = gt % CG;                        // column group of this thread
    const int lr = (gt / CG) % LPR;                // lane within the row's entries
    const int c0 = cg * CPT;
    int it = 0;
    for (int sbi = blockIdx.x; sbi < nsuper; sbi += gridDim.x, ++it) {
      const int st = it % NS;
      while (!mbar_try_wait(&full[st], (unsigned)((it / NS) & 1))) {}
      const int4 h = hdr[st][g];
      const int row0 = h.x, nr = h.y & 0xffff, nseg = h.y >> 16, self = h.z, nnzp = h.w;
      if (nseg > 0) {
        const unsigned char* base = dsm + st * S2::STAGE + g * SM::STAGE;
        const T* xw = reinterpret_cast<const T*>(base + SM::OFF_X);
        const T* bw = reinterpret_cast<const T*>(base + SM::OFF_B);
        const T* vw = reinterpret_cast<const T*>(base + SM::OFF_V);
        const T* dw = vw + nnzp;                                  // 1/diag of the block's rows
        const unsigned short* lw = reinterpret_cast<const unsigned short*>(dw + (A.has_dinv ? (nr + 7) / 8 * 8 : 0));
        const unsigned short* rw = lw + nnzp;
        const int b_lo = row0 & ~3;
        for (int basei = 0; basei < nr; basei += RPP) {
          const int rl = basei + gt / LPRW;
          const bool valid = rl < nr;
          T acc[CPT];
#pragma unroll
          for (int i = 0; i < CPT; ++i) acc[i] = T(0);
          if (valid) {
            const int a = rw[rl], b = rw[rl + 1];
            for (int j0 = a + lr; j0 < b; j0 += LPR * BATCH) {
              // BATCH independent chains: values + local columns, then the X vectors, then FMAs
              T v[BATCH];
              int sl[BATCH];
#pragma unroll
              for (int u = 0; u < BATCH; ++u) {
                const int j = j0 + u * LPR;
                const bool ok = j < b;
                v[u] = ok ? vw[j] : T(0);
                sl[u] = ok ? (int)lw[j] : 0;
              }
              T xv[BATCH][CPT];
#pragma unroll
              for (int u = 0; u < BATCH; ++u) ldvec<T, CPT>(xw + sl[u] * KT + c0, xv[u]);
#pragma unroll
              for (int u = 0; u < BATCH; ++u)
#pragma unroll
                for (int i = 0; i < CPT; ++i) acc[i] += v[u] * xv[u][i];
            }
          }
#pragma unroll
          for (int off = CG; off < LPRW; off <<= 1)
#pragma unroll
            for (int i = 0; i < CPT; ++i) acc[i] += __shfl_xor_sync(0xffffffffu, acc[i], off);
          if (valid && lr == 0) {
            const int row = row0 + rl;
            const size_t o = (size_t)row * KT + c0;
            T out[CPT], bb[CPT], xo[CPT];
            constexpr bool NEEDX = (MODE == SP_CG || MODE == SP_JACOBI || MODE == SP_JACOBI_DOT);
            if (SM::NEEDB) ldvec<T, CPT>(bw + (row - b_lo) * KT + c0, bb);
            if (NEEDX) {
              if (self >= 0) ldvec<T, CPT>(xw + (self + rl) * KT + c0, xo);
              else ldvec<T, CPT>(X + o, xo);
            }
            T dv = T(0);
            if (MODE == SP_JACOBI || MODE == SP_JACOBI_DOT) dv = ep.omega * (A.has_dinv ? dw[rl] : ep.dinv[row]);
#pragma unroll
            for (int i = 0; i < CPT; ++i) {
              if (MODE == SP_PLAIN) {
                out[i] = acc[i];
              } else if (MODE == SP_ADD) {
                out[i] = bb[i] + acc[i];
              } else if (MODE == SP_CG) {
                out[i] = acc[i];
                dot0[i] += (double)acc[i] * (double)xo[i];
              } else if (MODE == SP_RESNORM) {
                const T rr = bb[i] - acc[i];
                out[i] = rr;
                dot0[i] += (double)rr * (double)rr;
                dot1[i] += (double)bb[i] * (double)bb[i];
              } else if (MODE == SP_RES) {
                out[i] = bb[i] - acc[i];
              } else {
                const T yn = xo[i] + dv * (bb[i] - acc[i]);
                out[i] = yn;
                if (MODE == SP_JACOBI_DOT) dot0[i] += (double)bb[i] * (double)yn;
              }
            }
            stvec<T, CPT>(Y + o, out);
          }
        }
      } else if (nr > 1 || (nr == 1 && (A.rowptr[row0 + 1] - A.rowptr[row0]) <= W_NNZ)) {
        // scattered block: direct gathers on the plain CSR, same (row, column-group) ownership
        for (int basei = 0; basei < nr; basei += GT / CG) {
          const int rl = basei + gt / CG;
          if (rl < nr) {
            const int row = row0 + rl;
            T acc[CPT];
#pragma unroll
            for (int i = 0; i < CPT; ++i) acc[i] = T(0);
            for (int j = A.rowptr[row]; j < A.rowptr[row + 1]; ++j) {
              const T v = A.vals[j];
              T xv[CPT];
              ldvec<T, CPT>(X + (size_t)A.colidx[j] * KT + c0, xv);
#pragma unroll
              for (int i = 0; i < CPT; ++i) acc[i] += v * xv[i];
            }
#pragma unroll
            for (int i = 0; i < CPT; ++i)
              spmm_epilogue<T, MODE>(row, (size_t)row * KT + c0 + i, acc[i], X, Y, ep, dot0[i], dot1[i]);
          }
        }
      } else if (nr == 1) {
        // long row (its own block): the group's GT threads stride over it; thread q < CG of the
        // group finalises its own CPT columns (same ownership as everywhere else)
        const int row = row0;
        const int c = gt % KT;
        const int a = A.rowptr[row], b = A.rowptr[row + 1];
        double acc = 0.0;
        constexpr int GRP = GT / KT;
        for (int j = a + gt / KT; j < b; j += GRP)
          acc += (double)A.vals[j] * (double)X[(size_t)A.colidx[j] * KT + c];
        s_long[tid] = acc;
      }
      // long rows need a group-wide exchange; every consumer takes the same barrier sequence
      // (sub-blocks of one stage may differ, so the test is on "any long row in this stage")
      bool any_long = false;
#pragma unroll
      for (int q = 0; q < SB; ++q) {
        const int4 hq = hdr[st][q];
        any_long |= (hq.y == 1 && (A.rowptr[hq.x + 1] - A.rowptr[hq.x]) > W_NNZ);   // nseg 0, one row
      }
      if (any_long) {
        consumer_sync();
        const bool mine = nseg == 0 && nr == 1 && (A.rowptr[row0 + 1] - A.rowptr[row0]) > W_NNZ;
        if (mine && gt < CG) {
          constexpr int GRP = GT / KT;
#pragma unroll
          for (int i = 0; i < CPT; ++i) {
            const int col = gt * CPT + i;
            double t = 0.0;
            // not unrolled: a full unroll of the GRP-term chain (GRP = 64 .. 512) times the CPT columns
            // held the shared-memory operands of all of them in registers and spilled to local memory
#pragma unroll 1
            for (int q = 0; q < GRP; ++q) t += s_long[g * GT + q * KT + col];
            spmm_epilogue<T, MODE>(row0, (size_t)row0 * KT + col, (T)t, X, Y, ep, dot0[i], dot1[i]);
          }
        }
        consumer_sync();
      }
      __syncwarp();
      if ((tid & 31) == 0) mbar_arrive(&empty[st]);
    }
  }
  if (MODE == SP_CG) {
    CSB_REDUCE_SMEM_W(1, KT)
    double v[1][CPT];
#pragma unroll
    for (int i = 0; i < CPT; ++i) v[0][i] = dot0[i];
    if (grid_reduce<KT, CPT, 1, false, WTT>(v, ep.partials, &ep.ctl->ticket, s_warp, s_tree, s_out)) {
      if (tid < KT) {
        const double pap = s_out[tid];
        ep.ctl->pap[tid] = pap;
        ep.ctl->alpha[tid] = (ep.ctl->active[tid] && pap > 0.0) ? ep.ctl->rho[tid] / pap : 0.0;
      }
    }
  } else if (MODE == SP_RESNORM) {
    CSB_REDUCE_SMEM_W(2, KT)
    double v[2][CPT];
#pragma unroll
    for (int i = 0; i < CPT; ++i) { v[0][i] = dot0[i]; v[1][i] = dot1[i]; }
    if (grid_reduce<KT, CPT, 2, false, WTT>(v, ep.partials, &ep.ctl->ticket, s_warp, s_tree, s_out)) {
      if (tid < KT) {
        ep.ctl->resid[tid] = s_out[tid];
        ep.ctl->bnorm[tid] = s_out[KT + tid];
      }
    }
  } else if (MODE == SP_JACOBI_DOT) {
    CSB_REDUCE_SMEM_W(1, KT)
    double v[1][CPT];
#pragma unroll
    for (int i = 0; i < CPT; ++i) v[0][i] = dot0[i];
    if (grid_reduce<KT, CPT, 1, false, WTT>(v, ep.partials, &ep.ctl->ticket, s_warp, s_tree, s_out))
      cg_after_precond<KT>(ep.ctl, s_out);
  }
}

// ---------------------------------------------------------------------------
// Stencil (DIA) SpMM: Y = op(A X) for an operator whose every stored entry (i, j) has
// j - i in {0, +-1, +-nr, +-(nr -+ 1)} for one stride nr -- the 5-/9-point raster stencil of the
// reference with its column-major node numbering (src/raster/pairwise.jl:316-367) whenever
// every cell of the raster is a node, and the Galerkin operators of the regular coarse grids
// below it.  Found at setup (setup_device.cu build_dia); the operator is then stored as 9
// diagonals, slot-major (vals[s * ld + i], s = 3 * (dc + 1) + (dr + 1)): no column stream, no
// row offsets -- 9 s_v bytes per row instead of 9 (s_v + 4) + 4 of CSR (SURVEY.md 8f rank 2).
//
// A CTA owns a tile of RPP consecutive rows of one raster column x TC consecutive raster
// columns and sweeps the columns left to right; thread (row, column group) issues its 9
// coalesced value loads and 9 panel-row gathers (one 16-byte vector each) before the first FMA.
// The +-1 neighbours sit in the lines the warp's own rows fetch, the +-nr strips of column c are
// the centre strips of columns c -+ 1 of the same tile (L1) or of the neighbouring tile, which
// the round-robin tile order keeps in flight at the same time (L2).  Same epilogues / same
// deterministic reductions as k_spmm / k_spmm_win.
// ---------------------------------------------------------------------------
// Half form (half = 1): an operator whose lower slot s < 4 of every row i holds, bit for bit, the upper slot
// 8 - s of row i + off(s), off(s) = (s / 3 - 1) nr + s % 3 - 1 (and +0 where that row lies outside [0, n)), is
// stored as slots 4 ... 8 only (setup_device.hpp halve_dia): 5 values per row instead of 9.  The kernels take
// a lower slot from the neighbour row's upper slot, which is the same number in the same slot of the sums.
template <typename T> struct DiaDev {
  const T* vals;   // 9 diagonals (half: slots 4 ... 8), ld apart
  size_t ld;
  int n;
  int nr;          // stride between raster columns
  int half;
  // the stored run of slot s (s >= 4 when half)
  __device__ __forceinline__ const T* run(int s) const { return vals + (size_t)(half ? s - 4 : s) * ld; }
  // entry (row, row + off(s)); half: a lower slot from the neighbour row, 0 outside [0, n)
  __device__ __forceinline__ T at(int s, int row) const {
    if (!half || s >= 4) return __ldg(run(s) + row);
    const long long j = (long long)row + (s / 3 - 1) * (long long)nr + (s % 3 - 1);
    return j >= 0 && j < n ? __ldg(run(8 - s) + j) : T(0);
  }
};

constexpr int ST_TC = 16;   // raster columns per tile

// Three CTAs per SM (80 registers): all 18 loads of a row are in flight before the first FMA.  Carried
// over from the tuning on the previous GPU target, where the variants that issue the loads in smaller
// batches (64 registers for a fourth CTA, a sliding 3 x 3 register window) were slower; not re-measured
// on the H100.
template <typename T, int KT, int MODE>
__global__ void __launch_bounds__(NT, 3)
k_stencil(const DiaDev<T> A, const T* __restrict__ X, T* __restrict__ Y, const SpmmEpi<T> ep) {
  constexpr int V16 = 16 / (int)sizeof(T);
  constexpr int CPT = KT < V16 ? KT : V16;      // panel columns per thread (one 16-byte vector)
  constexpr int CG = KT / CPT;                  // column groups per row
  constexpr int RPP = NT / CG;                  // rows per pass of the CTA
  const int tid = threadIdx.x;
  const int cg = tid % CG, rl = tid / CG, c0 = cg * CPT;
  const int n = A.n, nr = A.nr;
  const int ncol = (n + nr - 1) / nr;           // raster columns
  const int nrc = (nr + RPP - 1) / RPP;         // row chunks per raster column
  const int ntc = (ncol + ST_TC - 1) / ST_TC;   // column groups
  const long long ntiles = (long long)nrc * ntc;
  double dot0[CPT], dot1[CPT];
#pragma unroll
  for (int i = 0; i < CPT; ++i) dot0[i] = dot1[i] = 0.0;

  for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int tc = (int)(t / nrc), rc = (int)(t % nrc);
    const int r = rc * RPP + rl;                // row within the raster column
    if (r >= nr) continue;
    const int cend = min(ncol, (tc + 1) * ST_TC);
    for (int c = tc * ST_TC; c < cend; ++c) {
      const long long row_l = (long long)c * nr + r;
      if (row_l >= n) break;
      const int row = (int)row_l;
      T v[9];
#pragma unroll
      for (int s = 0; s < 9; ++s) v[s] = __ldcs(A.vals + (size_t)s * A.ld + row);   // streamed once: evict first
      T xv[9][CPT];
      T wj[9];
#pragma unroll
      for (int s = 0; s < 9; ++s) {
        // missing neighbours carry a zero value: any in-range row will do for the gather
        int j = row + (s / 3 - 1) * nr + (s % 3 - 1);
        j = max(0, min(n - 1, j));
        if (MODE == SP_RES0) {       // x_j = omega D^-1_j b_j is never stored: gather b and 1/diag instead
          ldvec<T, CPT>(ep.B + (size_t)j * KT + c0, xv[s]);
          wj[s] = ep.omega * ep.dinv[j];
        } else {
          ldvec<T, CPT>(X + (size_t)j * KT + c0, xv[s]);
        }
      }
      T acc[CPT];
#pragma unroll
      for (int i = 0; i < CPT; ++i) acc[i] = T(0);
#pragma unroll
      for (int s = 0; s < 9; ++s) {
        const T vs = MODE == SP_RES0 ? v[s] * wj[s] : v[s];
#pragma unroll
        for (int i = 0; i < CPT; ++i) acc[i] += vs * xv[s][i];
      }
      const size_t o = (size_t)row * KT + c0;
      T out[CPT], bb[CPT];
      constexpr bool NEEDB = (MODE == SP_RESNORM || MODE == SP_RES || MODE == SP_JACOBI || MODE == SP_JACOBI_DOT);
      if (NEEDB) ldvec<T, CPT>(ep.B + o, bb);
      T dv = T(0);
      if (MODE == SP_JACOBI || MODE == SP_JACOBI_DOT) dv = ep.omega * ep.dinv[row];
#pragma unroll
      for (int i = 0; i < CPT; ++i) {
        const T xo = xv[4][i];
        if (MODE == SP_PLAIN) {
          out[i] = acc[i];
        } else if (MODE == SP_CG) {
          out[i] = acc[i];
          dot0[i] += (double)acc[i] * (double)xo;
        } else if (MODE == SP_RESNORM) {
          const T rr = bb[i] - acc[i];
          out[i] = rr;
          dot0[i] += (double)rr * (double)rr;
          dot1[i] += (double)bb[i] * (double)bb[i];
        } else if (MODE == SP_RES) {
          out[i] = bb[i] - acc[i];
        } else if (MODE == SP_RES0) {
          out[i] = xo - acc[i];                    // xv[4] holds the row's own b
        } else {
          const T yn = xo + dv * (bb[i] - acc[i]);
          out[i] = yn;
          if (MODE == SP_JACOBI_DOT) dot0[i] += (double)bb[i] * (double)yn;
        }
      }
      stvec<T, CPT>(Y + o, out);
    }
  }
  if (MODE == SP_CG) {
    CSB_REDUCE_SMEM(1, KT)
    double v[1][CPT];
#pragma unroll
    for (int i = 0; i < CPT; ++i) v[0][i] = dot0[i];
    if (grid_reduce<KT, CPT, 1, false>(v, ep.partials, &ep.ctl->ticket, s_warp, s_tree, s_out)) {
      if (tid < KT) {
        const double pap = s_out[tid];
        ep.ctl->pap[tid] = pap;
        ep.ctl->alpha[tid] = (ep.ctl->active[tid] && pap > 0.0) ? ep.ctl->rho[tid] / pap : 0.0;
      }
    }
  } else if (MODE == SP_RESNORM) {
    CSB_REDUCE_SMEM(2, KT)
    double v[2][CPT];
#pragma unroll
    for (int i = 0; i < CPT; ++i) { v[0][i] = dot0[i]; v[1][i] = dot1[i]; }
    if (grid_reduce<KT, CPT, 2, false>(v, ep.partials, &ep.ctl->ticket, s_warp, s_tree, s_out)) {
      if (tid < KT) {
        ep.ctl->resid[tid] = s_out[tid];
        ep.ctl->bnorm[tid] = s_out[KT + tid];
      }
    }
  } else if (MODE == SP_JACOBI_DOT) {
    CSB_REDUCE_SMEM(1, KT)
    double v[1][CPT];
#pragma unroll
    for (int i = 0; i < CPT; ++i) v[0][i] = dot0[i];
    if (grid_reduce<KT, CPT, 1, false>(v, ep.partials, &ep.ctl->ticket, s_warp, s_tree, s_out))
      cg_after_precond<KT>(ep.ctl, s_out);
  }
}

// ---------------------------------------------------------------------------
// Fused CG step of the AMG-PCG loop on a stencil-form finest level, iteration it = ctl->iter:
//   p_it = z + beta p_{it-1}   formed for the 9 gathered neighbours and for the own row, which goes to Pd
//   Y    = A p_it ; p.Ap per column ; last CTA: alpha_it exactly as k_stencil<SP_CG>, also into alpha_ring
//   x    the deferred solution updates, two at a time: on odd it, x = (x + alpha_{it-2} p_{it-2}) + alpha_{it-1}
//        p_{it-1}, with p_{it-2} read from the own row of Pd before p_it overwrites it
// p of even iterations lives in Pb[0], of odd ones in Pb[1]: the step reads p_{it-1} at neighbour rows while
// it writes p_it, so the two cannot share a buffer, and the buffer is picked from ctl->iter on the device
// (the loop body is captured once).  Tile order, grid and per-thread dot accumulation are those of
// k_stencil<SP_CG>, and every p and x value is formed with the expressions of k_cg_update_xp2: the partials,
// alpha and the iterates are bit-identical to the SpMM + update pair this replaces.  k_cg_x_tail applies
// the updates still pending when the loop ends.  It moves Z, p_{it-1}, the diagonals in and AP, p_it out
// every step, and X in/out and p_{it-2} in every other step, against the pair's Z, P, X in and X, P out
// plus the SpMM's diagonals, P in and AP out.
// ---------------------------------------------------------------------------
// CTAs per SM of k_stencil_cg: two (128 registers), all the z and p gathers of a row in flight.  At three (80
// registers) the T = double variants are spill-free but ptxas issues the gathers in smaller batches: on an
// H100 80GB HBM3 (700 W), fp64 k = 8 with the fp32 z on the 3163^2 raster, one step took 1.96 ms against
// 1.70 ms at two.  The fp32 k = 4 and 8 variants spill at three.
constexpr int CGF_MINB = 2;

template <typename T, int KT, typename TV>
__device__ __forceinline__ void stencil_cg_body(const DiaDev<T>& A, const TV* __restrict__ Z, const T* __restrict__ Pold,
                                                T* __restrict__ Pd, T* __restrict__ X, T* __restrict__ Y,
                                                PanelCtl* ctl, double* partials, int it) {
  constexpr int V16 = 16 / (int)sizeof(T);
  constexpr int CPT = KT < V16 ? KT : V16;      // panel columns per thread (one 16-byte vector)
  constexpr int CG = KT / CPT;                  // column groups per row
  constexpr int RPP = NT / CG;                  // rows per pass of the CTA
  const int tid = threadIdx.x;
  const int cg = tid % CG, rl = tid / CG, c0 = cg * CPT;
  const int n = A.n, nr = A.nr;
  const int ncol = (n + nr - 1) / nr;
  const int nrc = (nr + RPP - 1) / RPP;
  const int ntc = (ncol + ST_TC - 1) / ST_TC;
  const long long ntiles = (long long)nrc * ntc;
  const bool pair = it & 1;
  T be[CPT], a1[CPT], a2[CPT];                  // beta_it ; alpha_{it-1}, alpha_{it-2}
#pragma unroll
  for (int i = 0; i < CPT; ++i) {
    be[i] = (T)ctl->beta[c0 + i];
    a1[i] = (T)ctl->alpha_ring[(it + 2) % 3][c0 + i];
    a2[i] = (T)ctl->alpha_ring[(it + 1) % 3][c0 + i];
  }
  double dot0[CPT];
#pragma unroll
  for (int i = 0; i < CPT; ++i) dot0[i] = 0.0;

  for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
    const int tc = (int)(t / nrc), rc = (int)(t % nrc);
    const int r = rc * RPP + rl;
    if (r >= nr) continue;
    const int cend = min(ncol, (tc + 1) * ST_TC);
    for (int c = tc * ST_TC; c < cend; ++c) {
      const long long row_l = (long long)c * nr + r;
      if (row_l >= n) break;
      const int row = (int)row_l;
      T v[9];
#pragma unroll
      for (int s = 0; s < 9; ++s) v[s] = __ldcs(A.vals + (size_t)s * A.ld + row);
      TV zv[9][CPT];
      T pv[9][CPT];
#pragma unroll
      for (int s = 0; s < 9; ++s) {
        int j = row + (s / 3 - 1) * nr + (s % 3 - 1);
        j = max(0, min(n - 1, j));
        ldvec<TV, CPT>(Z + (size_t)j * KT + c0, zv[s]);
        ldvec<T, CPT, true>(Pold + (size_t)j * KT + c0, pv[s]);   // Pold != Pd: nothing writes it here
      }
      const size_t o = (size_t)row * KT + c0;
      T xo[CPT], pd[CPT], po[CPT];
      if (pair) {
        ldvec<T, CPT>(X + o, xo);
        ldvec<T, CPT>(Pd + o, pd);
      }
#pragma unroll
      for (int i = 0; i < CPT; ++i) po[i] = pv[4][i];
#pragma unroll
      for (int s = 0; s < 9; ++s)
#pragma unroll
        for (int i = 0; i < CPT; ++i) pv[s][i] = (T)zv[s][i] + be[i] * pv[s][i];
      T acc[CPT];
#pragma unroll
      for (int i = 0; i < CPT; ++i) acc[i] = T(0);
#pragma unroll
      for (int s = 0; s < 9; ++s)
#pragma unroll
        for (int i = 0; i < CPT; ++i) acc[i] += v[s] * pv[s][i];
#pragma unroll
      for (int i = 0; i < CPT; ++i) dot0[i] += (double)acc[i] * (double)pv[4][i];
      stvec<T, CPT>(Y + o, acc);
      stvec<T, CPT>(Pd + o, pv[4]);
      if (pair) {
#pragma unroll
        for (int i = 0; i < CPT; ++i) {
          xo[i] += a2[i] * pd[i];
          xo[i] += a1[i] * po[i];
        }
        stvec<T, CPT>(X + o, xo);
      }
    }
  }
  CSB_REDUCE_SMEM(1, KT)
  double v[1][CPT];
#pragma unroll
  for (int i = 0; i < CPT; ++i) v[0][i] = dot0[i];
  if (grid_reduce<KT, CPT, 1, false>(v, partials, &ctl->ticket, s_warp, s_tree, s_out)) {
    if (tid < KT) {
      const double pap = s_out[tid];
      const double al = (ctl->active[tid] && pap > 0.0) ? ctl->rho[tid] / pap : 0.0;
      ctl->pap[tid] = pap;
      ctl->alpha[tid] = al;
      ctl->alpha_ring[it % 3][tid] = al;
    }
  }
}

template <typename T, int KT, typename TV>
__global__ void __launch_bounds__(NT, CGF_MINB)
k_stencil_cg(const DiaDev<T> A, const TV* __restrict__ Z, T* Pb0, T* Pb1, T* __restrict__ X, T* __restrict__ Y,
             PanelCtl* ctl, double* partials) {
  const int it = ctl->iter;
  stencil_cg_body<T, KT, TV>(A, Z, (it & 1) ? Pb0 : Pb1, (it & 1) ? Pb1 : Pb0, X, Y, ctl, partials, it);
}

// ---------------------------------------------------------------------------
// Pipelined stencil sweeps (k_stencil_pipe, k_stencil_cg_pipe).  Tiles, tile walk, grid, thread map, each thread's
// order of (tile, column) steps, the 9-slot FMA order and every epilogue are those of k_stencil / k_stencil_cg, so
// the outputs and the per-CTA partial sums are bit-identical to theirs.  What changes is how operands arrive: a
// CTA's tiles form one flat sequence of load steps -- tile (tc, rc) loads the raster columns 16 tc - 1 ... ce
// (ce = the tile's last column + 1) -- and every load step is filled by cp.async S steps ahead of its use, across
// tile boundaries.  The step that loads column c + 1 computes column c.  Two rings in dynamic shared memory:
//   panel ring (S + 3 slots): rows [c nr + r0 - 1, c nr + r0 + RPP] of each gathered panel, one contiguous range:
//     the +-1 neighbours of a row are rows of the same slot, the +-nr ones the same rows of the slots of c -+ 1
//   own ring (S + 1 slots): the 9 diagonal runs of the RPP rows of column c and the own-row streams the step reads
// HALF (a half-form operator): the panel slot also holds the 5 upper-slot runs of its RPP + 2 rows and the own slot no
// diagonals; a lower slot s is upper slot 8 - s at the panel row the gather of slot s reads (st_half_val).
// A slot is rewritten three (panel) or one (own) step after its last read, behind the step's barrier.  Rows
// outside [0, n) are zero-filled by the copy (src-size 0): such a neighbour has a zero diagonal, and 0 x 0 adds
// nothing to a sum, as 0 x (the clamped row) does in the register kernels.  Every thread takes part in every copy
// and barrier; rows past nr or n only mask their compute and stores.
// Depth S: the largest (<= ST_SMAX) whose rings fit the shared memory of MINB CTAs per SM.  On an H100 80GB HBM3
// (700 W), 3163^2 raster, k = 8: the fused CG step (fp64, fp32 z; S = 2 at 3 CTAs/SM, 80 registers) 1.425 ms per
// step against 1.656 ms for k_stencil_cg, the fp32 level-0 residual (S = 4 at 3 CTAs/SM) 383 us against 418 us.
// Other S x CTAs/SM points were not measured.
// ---------------------------------------------------------------------------
constexpr int ST_SMAX = 4;
constexpr int st_a16(int b) { return (b + 15) & ~15; }

// EXTRA: dynamic shared memory the kernel keeps beside the two rings
template <int PANEL, int OWN, int MINB, int EXTRA = 0> struct StDepth {
  static constexpr int BUDGET = 228 * 1024 / MINB - 1024 - 3 * 1024 - EXTRA;   // less the per-CTA reserve, static buffers
  static constexpr int FIT = (BUDGET - 3 * PANEL - OWN) / (PANEL + OWN);
  static constexpr int S = FIT < 1 ? 1 : (FIT > ST_SMAX ? ST_SMAX : FIT);
  static constexpr int BYTES = (S + 3) * PANEL + (S + 1) * OWN + EXTRA;
};

template <int B>
__device__ __forceinline__ void cp_async_zfill(void* dst, const void* src, bool ok) {
  const int sz = ok ? B : 0;
  if constexpr (B == 16)
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(dst)), "l"(src), "r"(sz) : "memory");
  else
    asm volatile("cp.async.ca.shared.global [%0], [%1], %2, %3;" ::"r"(smem_u32(dst)), "l"(src), "n"(B), "r"(sz)
                 : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// rows [g0, g0 + NROWS) of a panel of W values per row, zero outside [0, n); chunks of min(16, row) bytes.
// !live: all zero, src not read (a panel known to hold zeros)
template <typename U, int W, int NROWS>
__device__ __forceinline__ void cp_rows(U* dst, const U* src, long long g0, int n, bool live = true) {
  constexpr int RB = W * (int)sizeof(U);
  constexpr int CH = RB < 16 ? RB : 16;
  constexpr int CPR = RB / CH;
  constexpr int NCH = NROWS * CPR;
#pragma unroll 1
  for (int q0 = 0; q0 < NCH; q0 += NT) {
    const int q = q0 + (int)threadIdx.x;
    if (NCH % NT == 0 || q < NCH) {
      const long long g = g0 + q / CPR;
      const bool ok = live && g >= 0 && g < n;
      cp_async_zfill<CH>(reinterpret_cast<char*>(dst) + q * CH,
                         reinterpret_cast<const char*>(src + (ok ? g : 0) * W) + (q % CPR) * CH, ok);
    }
  }
}

// the 9 diagonal runs of rows [row0, row0 + RPP), slot-major, zero past n
template <typename T, int RPP>
__device__ __forceinline__ void cp_diag(T* dst, const DiaDev<T>& A, long long row0) {
  constexpr int NCH = 9 * RPP;
#pragma unroll 1
  for (int q0 = 0; q0 < NCH; q0 += NT) {
    const int q = q0 + (int)threadIdx.x;
    if (NCH % NT == 0 || q < NCH) {
      const long long g = row0 + q % RPP;
      const bool ok = g < A.n;
      cp_async_zfill<(int)sizeof(T)>(dst + q, A.run(q / RPP) + (ok ? g : 0), ok);
    }
  }
}

// half form: the upper-slot runs 4 + [u0, u1) of the RPP + 2 rows [g0, g0 + RPP + 2) of a panel slot, slot-major
// (RPP + 2 apart), zero outside [0, n) -- the +0 that halve_dia demands of a lower slot whose mirror row is missing
template <typename T, int RPP>
__device__ __forceinline__ void cp_diag_half(T* dst, const DiaDev<T>& A, long long g0, int u0, int u1) {
  constexpr int RW = RPP + 2;
  const int nch = (u1 - u0) * RW;
#pragma unroll 1
  for (int q = (int)threadIdx.x; q < nch; q += NT) {
    const int u = u0 + q / RW, rr = q % RW;
    const long long g = g0 + rr;
    const bool ok = g >= 0 && g < A.n;
    cp_async_zfill<(int)sizeof(T)>(dst + u * RW + rr, A.run(4 + u) + (ok ? g : 0), ok);
  }
}

// one load step of a CTA's sequence: tile t, raster column c in [cs - 1, ce]
struct StStep {
  long long t;
  int cs, ce, c, r0;
  __device__ __forceinline__ void start(long long t_, int nrc, int ncol, int rpp) {
    t = t_;
    r0 = (int)(t % nrc) * rpp;
    cs = (int)(t / nrc) * ST_TC;
    ce = min(ncol, cs + ST_TC);
    c = cs - 1;
  }
  __device__ __forceinline__ void next(int nrc, int ncol, int rpp) {
    if (++c > ce) start(t + gridDim.x, nrc, ncol, rpp);
  }
  // half form: the upper-slot runs 4 + [u0, u1) this step loads -- all 5 where column c is computed (cs <= c < ce),
  // 6 ... 8 (the lower slots 0 ... 2 of column c + 1) where it is only the left neighbour of one (c = cs - 1)
  __device__ __forceinline__ void half_runs(int& u0, int& u1) const {
    u0 = c >= cs ? 0 : 2;
    u1 = c < ce ? 5 : 2;
  }
};

// half form: slot s9 of the row at panel row rl + 1 of column c, out of the upper-slot runs of the panel slots of
// columns c - 1, c (ds[0], ds[1]; RPP + 2 apart): a lower slot is upper slot 8 - s9 of the row the panel gather
// of slot s9 reads, at panel row rl + s9 % 3 of column c + s9 / 3 - 1
template <typename T, int RPP>
__device__ __forceinline__ T st_half_val(const T* const (&ds)[3], int s9, int rl) {
  return s9 < 4 ? ds[s9 / 3][(4 - s9) * (RPP + 2) + rl + s9 % 3] : ds[1][(s9 - 4) * (RPP + 2) + rl + 1];
}

// acc = the sum over the 9 slots, in slot order, of coef(s9) * val(s9): one row of a stencil product, the
// accumulation every pipelined stencil kernel shares so that they form the same row bit for bit
template <typename T, int CPT, class Val, class Coef>
__device__ __forceinline__ void stencil_row(T (&acc)[CPT], Val&& val, Coef&& coef) {
#pragma unroll
  for (int i = 0; i < CPT; ++i) acc[i] = T(0);
#pragma unroll
  for (int s9 = 0; s9 < 9; ++s9) {
    T v[CPT];
    val(s9, v);
    const T a = coef(s9);
#pragma unroll
    for (int i = 0; i < CPT; ++i) acc[i] += a * v[i];
  }
}

// issue(step, panel slot, own slot) fills the slots of a load step; compute(step, panel slot, own slot) runs on the
// step that loaded column step.c, for column step.c - 1, reading panel slots (slot - 2, slot - 1, slot) mod S + 3
template <int S, int RPP, class Issue, class Compute>
__device__ __forceinline__ void stencil_pipe(int n, int nr, Issue&& issue, Compute&& compute) {
  constexpr int RP = S + 3, RO = S + 1;
  const int ncol = (n + nr - 1) / nr;
  const int nrc = (nr + RPP - 1) / RPP;
  const long long ntiles = (long long)nrc * ((ncol + ST_TC - 1) / ST_TC);
  StStep ld, st;
  ld.start(blockIdx.x, nrc, ncol, RPP);
  st = ld;
  int lp = 0, lo = 0, sp = 0, so = 0;
#pragma unroll 1
  for (int k = 0; k < S; ++k) {
    if (ld.t < ntiles) issue(ld, lp, lo);
    cp_async_commit();
    ld.next(nrc, ncol, RPP);
    lp = lp + 1 == RP ? 0 : lp + 1;
    lo = lo + 1 == RO ? 0 : lo + 1;
  }
#pragma unroll 1
  while (st.t < ntiles) {
    cp_async_wait<S - 1>();
    __syncthreads();                 // this step's slots are filled; every reader of the slots refilled below is done
    if (ld.t < ntiles) issue(ld, lp, lo);
    cp_async_commit();
    ld.next(nrc, ncol, RPP);
    lp = lp + 1 == RP ? 0 : lp + 1;
    lo = lo + 1 == RO ? 0 : lo + 1;
    if (st.c > st.cs) compute(st, sp, so);
    st.next(nrc, ncol, RPP);
    sp = sp + 1 == RP ? 0 : sp + 1;
    so = so + 1 == RO ? 0 : so + 1;
  }
  cp_async_wait<0>();
}

template <typename T, int KT, int MODE, bool HALF> struct StPipe {
  static constexpr int V16 = 16 / (int)sizeof(T);
  static constexpr int CPT = KT < V16 ? KT : V16;
  static constexpr int RPP = NT / (KT / CPT);
  static constexpr bool NEEDB = (MODE == SP_RESNORM || MODE == SP_RES || MODE == SP_JACOBI || MODE == SP_JACOBI_DOT);
  static constexpr bool NEEDD = (MODE == SP_JACOBI || MODE == SP_JACOBI_DOT);
  // panel slot: X (B for SP_RES0) rows, then for SP_RES0 1/diag rows, then (HALF) the 5 upper-slot runs of the
  // same rows ; own slot: (!HALF) the 9 diagonal runs, B rows, 1/diag
  static constexpr int PX = st_a16((RPP + 2) * KT * (int)sizeof(T));
  static constexpr int PDG = PX + (MODE == SP_RES0 ? st_a16((RPP + 2) * (int)sizeof(T)) : 0);
  static constexpr int PANEL = PDG + (HALF ? st_a16(5 * (RPP + 2) * (int)sizeof(T)) : 0);
  static constexpr int OD = HALF ? 0 : st_a16(9 * RPP * (int)sizeof(T));
  static constexpr int OB = NEEDB ? st_a16(RPP * KT * (int)sizeof(T)) : 0;
  static constexpr int OWN = OD + OB + (NEEDD ? st_a16(RPP * (int)sizeof(T)) : 0);
  using D = StDepth<PANEL, OWN, 3>;
};

// k_stencil, operands through the shared-memory pipeline.  Three CTAs per SM as k_stencil.  HALF: A is in the
// half form (A.half), its diagonals come with the panel rows.
template <typename T, int KT, int MODE, bool HALF>
__global__ void __launch_bounds__(NT, 3)
k_stencil_pipe(const DiaDev<T> A, const T* __restrict__ X, T* __restrict__ Y, const SpmmEpi<T> ep) {
  using SP = StPipe<T, KT, MODE, HALF>;
  constexpr int CPT = SP::CPT, RPP = SP::RPP, S = SP::D::S;
  constexpr int RP = S + 3;
  extern __shared__ __align__(128) unsigned char st_sm[];
  unsigned char* const pring = st_sm;
  unsigned char* const oring = st_sm + RP * SP::PANEL;
  const int tid = threadIdx.x;
  const int cg = tid % (KT / CPT), rl = tid / (KT / CPT), c0 = cg * CPT;
  const int n = A.n, nr = A.nr;
  double dot0[CPT], dot1[CPT];
#pragma unroll
  for (int i = 0; i < CPT; ++i) dot0[i] = dot1[i] = 0.0;

  const T* const G = MODE == SP_RES0 ? ep.B : X;     // the gathered panel
  auto issue = [&](const StStep& s, int lp, int lo) {
    unsigned char* ps = pring + lp * SP::PANEL;
    const long long g0 = (long long)s.c * nr + s.r0 - 1;
    cp_rows<T, KT, RPP + 2>(reinterpret_cast<T*>(ps), G, g0, n);
    if (MODE == SP_RES0) cp_rows<T, 1, RPP + 2>(reinterpret_cast<T*>(ps + SP::PX), ep.dinv, g0, n);
    if (HALF) {
      int u0, u1;
      s.half_runs(u0, u1);
      cp_diag_half<T, RPP>(reinterpret_cast<T*>(ps + SP::PDG), A, g0, u0, u1);
    }
    if (s.c > s.cs) {
      unsigned char* os = oring + lo * SP::OWN;
      const long long row0 = (long long)(s.c - 1) * nr + s.r0;
      if (!HALF) cp_diag<T, RPP>(reinterpret_cast<T*>(os), A, row0);
      if (SP::NEEDB && !(MODE == SP_RESNORM && ep.pair_b))
        cp_rows<T, KT, RPP>(reinterpret_cast<T*>(os + SP::OD), ep.B, row0, n);
      if (SP::NEEDD) cp_rows<T, 1, RPP>(reinterpret_cast<T*>(os + SP::OD + SP::OB), ep.dinv, row0, n);
    }
  };
  auto compute = [&](const StStep& s, int sp, int so) {
    const int c = s.c - 1, r = s.r0 + rl;
    const long long row_l = (long long)c * nr + r;
    if (r >= nr || row_l >= n) return;
    const int row = (int)row_l;
    const T* xs[3];
    const T* ws[3];
    const T* ds[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const int k = sp + d + RP - 2;
      const unsigned char* p = pring + (k >= RP ? k - RP : k) * SP::PANEL;
      xs[d] = reinterpret_cast<const T*>(p);
      ws[d] = reinterpret_cast<const T*>(p + SP::PX);
      ds[d] = reinterpret_cast<const T*>(p + SP::PDG);
    }
    const unsigned char* os = oring + so * SP::OWN;
    const T* dg = reinterpret_cast<const T*>(os);
    T acc[CPT], xo[CPT];
#pragma unroll
    for (int i = 0; i < CPT; ++i) acc[i] = T(0);
#pragma unroll
    for (int s9 = 0; s9 < 9; ++s9) {
      T xv[CPT];
      ldvec<T, CPT>(xs[s9 / 3] + (rl + s9 % 3) * KT + c0, xv);
      if (s9 == 4) {
#pragma unroll
        for (int i = 0; i < CPT; ++i) xo[i] = xv[i];
      }
      const T a9 = HALF ? st_half_val<T, RPP>(ds, s9, rl) : dg[s9 * RPP + rl];
      const T vs = MODE == SP_RES0 ? a9 * (ep.omega * ws[s9 / 3][rl + s9 % 3]) : a9;
#pragma unroll
      for (int i = 0; i < CPT; ++i) acc[i] += vs * xv[i];
    }
    const size_t o = (size_t)row * KT + c0;
    T out[CPT], bb[CPT];
    if (MODE == SP_RESNORM && ep.pair_b) {
#pragma unroll
      for (int i = 0; i < CPT; ++i) bb[i] = pair_rhs_val<T>(ep.ctl, row, c0 + i);
    } else if (SP::NEEDB) {
      ldvec<T, CPT>(reinterpret_cast<const T*>(os + SP::OD) + rl * KT + c0, bb);
    }
    T dv = T(0);
    if (SP::NEEDD) dv = ep.omega * reinterpret_cast<const T*>(os + SP::OD + SP::OB)[rl];
#pragma unroll
    for (int i = 0; i < CPT; ++i) {
      if (MODE == SP_PLAIN) {
        out[i] = acc[i];
      } else if (MODE == SP_CG) {
        out[i] = acc[i];
        dot0[i] += (double)acc[i] * (double)xo[i];
      } else if (MODE == SP_RESNORM) {
        const T rr = bb[i] - acc[i];
        out[i] = rr;
        dot0[i] += (double)rr * (double)rr;
        dot1[i] += (double)bb[i] * (double)bb[i];
      } else if (MODE == SP_RES) {
        out[i] = bb[i] - acc[i];
      } else if (MODE == SP_RES0) {
        out[i] = xo[i] - acc[i];
      } else {
        const T yn = xo[i] + dv * (bb[i] - acc[i]);
        out[i] = yn;
        if (MODE == SP_JACOBI_DOT) dot0[i] += (double)bb[i] * (double)yn;
      }
    }
    if (!(MODE == SP_RESNORM && ep.pair_b)) stvec<T, CPT>(Y + o, out);
  };
  stencil_pipe<S, RPP>(n, nr, issue, compute);

  if (MODE == SP_CG) {
    CSB_REDUCE_SMEM(1, KT)
    double v[1][CPT];
#pragma unroll
    for (int i = 0; i < CPT; ++i) v[0][i] = dot0[i];
    if (grid_reduce<KT, CPT, 1, false>(v, ep.partials, &ep.ctl->ticket, s_warp, s_tree, s_out)) {
      if (tid < KT) {
        const double pap = s_out[tid];
        ep.ctl->pap[tid] = pap;
        ep.ctl->alpha[tid] = (ep.ctl->active[tid] && pap > 0.0) ? ep.ctl->rho[tid] / pap : 0.0;
      }
    }
  } else if (MODE == SP_RESNORM) {
    CSB_REDUCE_SMEM(2, KT)
    double v[2][CPT];
#pragma unroll
    for (int i = 0; i < CPT; ++i) { v[0][i] = dot0[i]; v[1][i] = dot1[i]; }
    if (grid_reduce<KT, CPT, 2, false>(v, ep.partials, &ep.ctl->ticket, s_warp, s_tree, s_out)) {
      if (tid < KT) {
        ep.ctl->resid[tid] = s_out[tid];
        ep.ctl->bnorm[tid] = s_out[KT + tid];
      }
    }
  } else if (MODE == SP_JACOBI_DOT) {
    CSB_REDUCE_SMEM(1, KT)
    double v[1][CPT];
#pragma unroll
    for (int i = 0; i < CPT; ++i) v[0][i] = dot0[i];
    if (grid_reduce<KT, CPT, 1, false>(v, ep.partials, &ep.ctl->ticket, s_warp, s_tree, s_out))
      cg_after_precond<KT>(ep.ctl, s_out);
  }
}

// k_stencil_cg, operands through the shared-memory pipeline: panel slot p_{it-1} and Z rows, own slot the diagonals
// and, on odd iterations, the X and Pd (p_{it-2}) rows.  Without the register arrays of the gathers it runs at
// CGP_MINB CTAs per SM.  !STORE_AP: Y is not written (k_stencil_res_update forms A p again from the stored p).
constexpr int CGP_MINB = 3;

template <typename T, int KT, typename TV, bool HALF> struct StPipeCg {
  static constexpr int V16 = 16 / (int)sizeof(T);
  static constexpr int CPT = KT < V16 ? KT : V16;
  static constexpr int RPP = NT / (KT / CPT);
  static constexpr int PP = st_a16((RPP + 2) * KT * (int)sizeof(T));
  static constexpr int PDG = PP + st_a16((RPP + 2) * KT * (int)sizeof(TV));
  static constexpr int PANEL = PDG + (HALF ? st_a16(5 * (RPP + 2) * (int)sizeof(T)) : 0);
  static constexpr int OD = HALF ? 0 : st_a16(9 * RPP * (int)sizeof(T));
  static constexpr int OX = st_a16(RPP * KT * (int)sizeof(T));
  static constexpr int OWN = OD + 2 * OX;
  using D = StDepth<PANEL, OWN, CGP_MINB>;
};

template <typename T, int KT, typename TV, bool HALF, bool STORE_AP>
__global__ void __launch_bounds__(NT, CGP_MINB)
k_stencil_cg_pipe(const DiaDev<T> A, const TV* __restrict__ Z, T* Pb0, T* Pb1, T* __restrict__ X, T* __restrict__ Y,
                  PanelCtl* ctl, double* partials) {
  using SP = StPipeCg<T, KT, TV, HALF>;
  constexpr int CPT = SP::CPT, RPP = SP::RPP, S = SP::D::S;
  constexpr int RP = S + 3;
  extern __shared__ __align__(128) unsigned char st_sm[];
  unsigned char* const pring = st_sm;
  unsigned char* const oring = st_sm + RP * SP::PANEL;
  const int it = ctl->iter;
  const T* const Pold = (it & 1) ? Pb0 : Pb1;      // Pold != Pd: nothing writes it here
  T* const Pd = (it & 1) ? Pb1 : Pb0;
  const int tid = threadIdx.x;
  const int cg = tid % (KT / CPT), rl = tid / (KT / CPT), c0 = cg * CPT;
  const int n = A.n, nr = A.nr;
  const bool pair = it & 1;
  // a panel starts from x = 0, p_{-1} = 0: p_{it-1} at it = 0 and x, p_{it-2} at it = 1 are staged as zeros, not
  // read, so the start of a panel need not fill X and P (panel_ends)
  const bool p_live = it != 0, x_live = it != 1;
  T be[CPT], a1[CPT], a2[CPT];                  // beta_it ; alpha_{it-1}, alpha_{it-2}
#pragma unroll
  for (int i = 0; i < CPT; ++i) {
    be[i] = (T)ctl->beta[c0 + i];
    a1[i] = (T)ctl->alpha_ring[(it + 2) % 3][c0 + i];
    a2[i] = (T)ctl->alpha_ring[(it + 1) % 3][c0 + i];
  }
  double dot0[CPT];
#pragma unroll
  for (int i = 0; i < CPT; ++i) dot0[i] = 0.0;

  auto issue = [&](const StStep& s, int lp, int lo) {
    unsigned char* ps = pring + lp * SP::PANEL;
    const long long g0 = (long long)s.c * nr + s.r0 - 1;
    cp_rows<T, KT, RPP + 2>(reinterpret_cast<T*>(ps), Pold, g0, n, p_live);
    cp_rows<TV, KT, RPP + 2>(reinterpret_cast<TV*>(ps + SP::PP), Z, g0, n);
    if (HALF) {
      int u0, u1;
      s.half_runs(u0, u1);
      cp_diag_half<T, RPP>(reinterpret_cast<T*>(ps + SP::PDG), A, g0, u0, u1);
    }
    if (s.c > s.cs) {
      unsigned char* os = oring + lo * SP::OWN;
      const long long row0 = (long long)(s.c - 1) * nr + s.r0;
      if (!HALF) cp_diag<T, RPP>(reinterpret_cast<T*>(os), A, row0);
      if (pair) {
        cp_rows<T, KT, RPP>(reinterpret_cast<T*>(os + SP::OD), X, row0, n, x_live);
        cp_rows<T, KT, RPP>(reinterpret_cast<T*>(os + SP::OD + SP::OX), Pd, row0, n, x_live);
      }
    }
  };
  auto compute = [&](const StStep& s, int sp, int so) {
    const int c = s.c - 1, r = s.r0 + rl;
    const long long row_l = (long long)c * nr + r;
    if (r >= nr || row_l >= n) return;
    const int row = (int)row_l;
    const T* ps[3];
    const TV* zs[3];
    const T* ds[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const int k = sp + d + RP - 2;
      const unsigned char* p = pring + (k >= RP ? k - RP : k) * SP::PANEL;
      ps[d] = reinterpret_cast<const T*>(p);
      zs[d] = reinterpret_cast<const TV*>(p + SP::PP);
      ds[d] = reinterpret_cast<const T*>(p + SP::PDG);
    }
    const unsigned char* os = oring + so * SP::OWN;
    const T* dg = reinterpret_cast<const T*>(os);
    T acc[CPT], po[CPT], pc[CPT];
    stencil_row<T, CPT>(
        acc,
        [&](int s9, T (&pv)[CPT]) {
          TV zv[CPT];
          ldvec<T, CPT>(ps[s9 / 3] + (rl + s9 % 3) * KT + c0, pv);
          ldvec<TV, CPT>(zs[s9 / 3] + (rl + s9 % 3) * KT + c0, zv);
          if (s9 == 4) {
#pragma unroll
            for (int i = 0; i < CPT; ++i) po[i] = pv[i];
          }
#pragma unroll
          for (int i = 0; i < CPT; ++i) pv[i] = (T)zv[i] + be[i] * pv[i];
          if (s9 == 4) {
#pragma unroll
            for (int i = 0; i < CPT; ++i) pc[i] = pv[i];
          }
        },
        [&](int s9) { return HALF ? st_half_val<T, RPP>(ds, s9, rl) : dg[s9 * RPP + rl]; });
#pragma unroll
    for (int i = 0; i < CPT; ++i) dot0[i] += (double)acc[i] * (double)pc[i];
    const size_t o = (size_t)row * KT + c0;
    if (STORE_AP) stvec<T, CPT>(Y + o, acc);
    stvec<T, CPT>(Pd + o, pc);
    if (pair) {
      T xo[CPT], pd[CPT];
      ldvec<T, CPT>(reinterpret_cast<const T*>(os + SP::OD) + rl * KT + c0, xo);
      ldvec<T, CPT>(reinterpret_cast<const T*>(os + SP::OD + SP::OX) + rl * KT + c0, pd);
#pragma unroll
      for (int i = 0; i < CPT; ++i) {
        xo[i] += a2[i] * pd[i];
        xo[i] += a1[i] * po[i];
      }
      stvec<T, CPT>(X + o, xo);
    }
  };
  stencil_pipe<S, RPP>(n, nr, issue, compute);

  CSB_REDUCE_SMEM(1, KT)
  double v[1][CPT];
#pragma unroll
  for (int i = 0; i < CPT; ++i) v[0][i] = dot0[i];
  if (grid_reduce<KT, CPT, 1, false>(v, partials, &ctl->ticket, s_warp, s_tree, s_out)) {
    if (tid < KT) {
      const double pap = s_out[tid];
      const double al = (ctl->active[tid] && pap > 0.0) ? ctl->rho[tid] / pap : 0.0;
      ctl->pap[tid] = pap;
      ctl->alpha[tid] = al;
      ctl->alpha_ring[it % 3][tid] = al;
    }
  }
}

// ---------------------------------------------------------------------------
// Residual update and finest-level residual sweep of the AMG-PCG iteration, fused, on a half-form stencil finest
// level with an fp32 (TV) V-cycle, iteration it = ctl->iter, right after k_stencil_cg_pipe<..., false> (no A p):
//   Ap  = A p_it                            (p_it: the panel the CG step wrote, Pb0 / Pb1 by it as there)
//   r'  = r - alpha_it Ap ; r32 = (TV) r'   (k_cg_update_r0's expressions)
//   T32 = r32 - A32 (omega D32^-1 r32)      (k_stencil_pipe<SP_RES0>'s expressions on the fp32 level 0)
// A p is formed by stencil_row as the CG step forms it, so it is the same number, and neither A p nor r32 goes
// through global memory.  r of even iterations lives in Rb0, of odd ones in Rb1: a strip reads the halo rows of r
// that neighbouring strips rewrite, so the update cannot be in place.
// Work split as k_stencil_prolong_jacobi: strips of RPS = RH - 2 rows, (strip, raster column) steps strip-major,
// one contiguous run per CTA; thread (rr, g) takes row rr - 1 of the strip (rr = 0, RH - 1: the halo rows) and
// column group g.  A run's segment [cb, ce) of one strip takes the load steps x = cb - 2 ... ce + 2 through the
// cp.async rings of stencil_pipe (one barrier per step):
//   panel slot (S + 3): p rows -2 ... RPS + 1 of column x and their 5 upper-slot runs (x <= ce + 1); the fp32
//                       1/diag of rows -1 ... RPS of column x - 2 (x - 2 in [cb - 1, ce])
//   own slot (S + 1):   r rows -1 ... RPS of column x - 1
// and, once the slots of step x are in, computes A p, r', r32 of the RH rows of column x - 1 (x - 1 in [cb - 1, ce];
// r32 and the fp32 rounding of the row's 5 upper-slot values into rings of 4 columns) and T32 of the strip rows of
// column x - 3 (in [cb, ce)) out of the ring columns x - 4 ... x - 2, which the previous steps wrote.  The fp32
// level-0 operator is the fp64 one rounded, so its diagonals are not read: launch_res_update runs the kernel only
// where the stored fp32 runs equal the rounded fp64 ones bit for bit (k_dia_rounds).  Halo rows and columns are recomputed bit for bit by the
// owner; only the owner stores r', R32 and T32.
// ---------------------------------------------------------------------------
constexpr int RU_MINB = 3;
constexpr int RU_RING = 4;   // r32 columns: x - 4 ... x - 2 read, x - 1 written

template <typename T, typename TV, int KT> struct RuShape {
  static constexpr int V16 = 16 / (int)sizeof(T);
  static constexpr int CPT = KT < V16 ? KT : V16;
  static constexpr int CG = KT / CPT;
  static constexpr int RH = NT / CG;
  static constexpr int RPS = RH - 2;
  static constexpr int PDG = st_a16((RH + 2) * KT * (int)sizeof(T));
  static constexpr int PW32 = PDG + st_a16(5 * (RH + 2) * (int)sizeof(T));
  static constexpr int PANEL = PW32 + st_a16(RH * (int)sizeof(TV));
  static constexpr int OWN = st_a16(RH * KT * (int)sizeof(T));
  static constexpr int RING = RU_RING * RH * KT * (int)sizeof(TV);     // r32 columns
  static constexpr int DRING = RU_RING * 5 * RH * (int)sizeof(TV);     // fp32 upper-slot runs, per column
  using D = StDepth<PANEL, OWN, RU_MINB, RING + DRING>;
};

// one load step: column x of the segment [cb, ce) of strip `strip`; s0 = the segment's first (strip, column) step
struct RuStep {
  int s0, s_end, ncol, strip, cb, ce, x;
  __device__ __forceinline__ void start(int s) {
    s0 = s;
    if (s >= s_end) return;
    strip = s / ncol;
    cb = s % ncol;
    ce = min(ncol, cb + (s_end - s));
    x = cb - 2;
  }
  __device__ __forceinline__ bool valid() const { return s0 < s_end; }
  __device__ __forceinline__ void next() {
    if (++x > ce + 2) start(s0 + (ce - cb));
  }
};

template <typename T, typename TV, int KT>
__global__ void __launch_bounds__(NT, RU_MINB)
k_stencil_res_update(const DiaDev<T> A, const TV* __restrict__ dinv32, TV omega,
                     const T* __restrict__ Pb0, const T* __restrict__ Pb1, T* Rb0, T* Rb1, TV* __restrict__ R32,
                     TV* __restrict__ T32, const PanelCtl* __restrict__ ctl) {
  using SH = RuShape<T, TV, KT>;
  constexpr int CPT = SH::CPT, CG = SH::CG, RH = SH::RH, RPS = SH::RPS, S = SH::D::S;
  constexpr int RP = S + 3, RO = S + 1;
  extern __shared__ __align__(128) unsigned char st_sm[];
  unsigned char* const pring = st_sm;
  unsigned char* const oring = st_sm + RP * SH::PANEL;
  TV* const xring = reinterpret_cast<TV*>(oring + RO * SH::OWN);   // [RU_RING][RH][KT]
  TV* const dring = xring + RU_RING * RH * KT;                       // [RU_RING][5][RH]
  const int it = ctl->iter;
  const T* const Pk = (it & 1) ? Pb1 : Pb0;
  const T* const Rin = (it & 1) ? Rb1 : Rb0;
  T* const Rout = (it & 1) ? Rb0 : Rb1;
  const int tid = threadIdx.x;
  const int g = tid % CG, rr = tid / CG, c0 = g * CPT;
  const bool inner = rr >= 1 && rr <= RPS;
  const int n = A.n, nr = A.nr;
  const int ncol = (n + nr - 1) / nr;
  const int nstrip = (nr + RPS - 1) / RPS;
  // nstep <= nr * ncol < n + nr: int for every operator launch_prolong_jacobi accepts (n + nr < 2^31)
  const int nstep = nstrip * ncol;
  const int per = (nstep + (int)gridDim.x - 1) / (int)gridDim.x;
  const int s_beg = (int)min((long long)nstep, (long long)blockIdx.x * per);
  const int s_end = (int)min((long long)nstep, ((long long)blockIdx.x + 1) * per);
  T al[CPT];
#pragma unroll
  for (int i = 0; i < CPT; ++i) al[i] = (T)ctl->alpha[c0 + i];

  auto issue = [&](const RuStep& s, int lp, int lo) {
    unsigned char* ps = pring + lp * SH::PANEL;
    const long long r0 = (long long)s.strip * RPS;
    if (s.x <= s.ce + 1) {
      const long long g0 = (long long)s.x * nr + r0 - 2;
      cp_rows<T, KT, RH + 2>(reinterpret_cast<T*>(ps), Pk, g0, n);
      cp_diag_half<T, RH>(reinterpret_cast<T*>(ps + SH::PDG), A, g0, 0, 5);
    }
    if (s.x - 2 >= s.cb - 1)
      cp_rows<TV, 1, RH>(reinterpret_cast<TV*>(ps + SH::PW32), dinv32, (long long)(s.x - 2) * nr + r0 - 1, n);
    if (s.x - 1 >= s.cb - 1 && s.x - 1 <= s.ce)
      cp_rows<T, KT, RH>(reinterpret_cast<T*>(oring + lo * SH::OWN), Rin, (long long)(s.x - 1) * nr + r0 - 1, n);
  };
  auto compute = [&](const RuStep& s, int sp, int so, int q) {
    const unsigned char* pk[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const int k = sp + d + RP - 2;
      pk[d] = pring + (k >= RP ? k - RP : k) * SH::PANEL;
    }
    const int r = s.strip * RPS + rr - 1;                  // this thread's row within a raster column
    const int ca = s.x - 1;                                // A p, r', r32 of column ca
    if (ca >= s.cb - 1 && ca <= s.ce) {
      const T* ps[3];
      const T* ds[3];
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        ps[d] = reinterpret_cast<const T*>(pk[d]);
        ds[d] = reinterpret_cast<const T*>(pk[d] + SH::PDG);
      }
      T acc[CPT], rv[CPT];
      TV r32[CPT];
      stencil_row<T, CPT>(
          acc, [&](int s9, T (&pv)[CPT]) { ldvec<T, CPT>(ps[s9 / 3] + (rr + s9 % 3) * KT + c0, pv); },
          [&](int s9) { return st_half_val<T, RH>(ds, s9, rr); });
      ldvec<T, CPT>(reinterpret_cast<const T*>(oring + so * SH::OWN) + rr * KT + c0, rv);
#pragma unroll
      for (int i = 0; i < CPT; ++i) {
        rv[i] -= al[i] * acc[i];
        r32[i] = (TV)rv[i];
      }
      stvec<TV, CPT>(xring + (q * RH + rr) * KT + c0, r32);
      if (g == 0) {
#pragma unroll
        for (int u = 0; u < 5; ++u) dring[(q * 5 + u) * RH + rr] = (TV)ds[1][u * (RH + 2) + rr + 1];
      }
      const long long row = (long long)ca * nr + r;
      if (inner && r < nr && ca >= s.cb && ca < s.ce && row < n) {
        stvec<T, CPT>(Rout + (size_t)row * KT + c0, rv);
        stvec<TV, CPT>(R32 + (size_t)row * KT + c0, r32);
      }
    }
    const int ct = s.x - 3;                                // T32 of column ct
    const long long row = (long long)ct * nr + r;
    if (ct >= s.cb && ct < s.ce && inner && r < nr && row < n) {
      const TV* xs[3];
      const TV* ws[3];
      const TV* ds[3];
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        xs[d] = xring + ((q + 1 + d) & (RU_RING - 1)) * RH * KT;   // columns ct - 1, ct, ct + 1
        ws[d] = reinterpret_cast<const TV*>(pk[d] + SH::PW32);
        ds[d] = dring + ((q + 1 + d) & (RU_RING - 1)) * 5 * RH;
      }
      const int rl = rr - 1;
      TV acc[CPT], xo[CPT], out[CPT];
      stencil_row<TV, CPT>(
          acc,
          [&](int s9, TV (&xv)[CPT]) {
            ldvec<TV, CPT>(xs[s9 / 3] + (rl + s9 % 3) * KT + c0, xv);
            if (s9 == 4) {
#pragma unroll
              for (int i = 0; i < CPT; ++i) xo[i] = xv[i];
            }
          },
          [&](int s9) { return st_half_val<TV, RPS>(ds, s9, rl) * (omega * ws[s9 / 3][rl + s9 % 3]); });
#pragma unroll
      for (int i = 0; i < CPT; ++i) out[i] = xo[i] - acc[i];
      stvec<TV, CPT>(T32 + (size_t)row * KT + c0, out);
    }
  };

  RuStep ld, st;
  ld.s_end = s_end;
  ld.ncol = ncol;
  ld.start(s_beg);
  st = ld;
  int lp = 0, lo = 0, sp = 0, so = 0, q = 0;
#pragma unroll 1
  for (int k = 0; k < S; ++k) {
    if (ld.valid()) issue(ld, lp, lo);
    cp_async_commit();
    if (ld.valid()) ld.next();
    lp = lp + 1 == RP ? 0 : lp + 1;
    lo = lo + 1 == RO ? 0 : lo + 1;
  }
#pragma unroll 1
  while (st.valid()) {
    cp_async_wait<S - 1>();
    __syncthreads();                 // this step's slots are in, the previous step's r32 column is written
    if (ld.valid()) issue(ld, lp, lo);
    cp_async_commit();
    if (ld.valid()) ld.next();
    lp = lp + 1 == RP ? 0 : lp + 1;
    lo = lo + 1 == RO ? 0 : lo + 1;
    compute(st, sp, so, q);
    st.next();
    sp = sp + 1 == RP ? 0 : sp + 1;
    so = so + 1 == RO ? 0 : so + 1;
    q = (q + 1) & (RU_RING - 1);
  }
  cp_async_wait<0>();
}

// differs = 1 unless the 5 upper-slot runs of A32 are those of A rounded to TV, bit for bit
template <typename T, typename TV>
__global__ void k_dia_rounds(const DiaDev<T> A, const DiaDev<TV> A32, int* differs) {
  const long long tot = 5LL * A.n;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < tot; i += (long long)gridDim.x * blockDim.x) {
    const int u = (int)(i / A.n), row = (int)(i % A.n);
    const TV a = (TV)A.run(4 + u)[row], b = A32.run(4 + u)[row];
    static_assert(sizeof(TV) == 4, "fp32 copies");
    unsigned ua, ub;
    memcpy(&ua, &a, 4);
    memcpy(&ub, &b, 4);
    if (ua != ub) *differs = 1;
  }
}

// ---------------------------------------------------------------------------
// Upward leg of the V-cycle on a stencil-form level, fused:  prolongate + correct + post-smooth
//     x1 = x0 + P y          (y: the coarser level's correction, P: ~3 entries per row)
//     z  = x1 + omega D^-1 (b - A x1)        [+ dot(b, z) -> CG beta / stop test on the finest level]
// Streaming form.  The rows of every raster column are cut into strips of PJ_RH - 2 rows; the (strip, raster
// column) steps, strip-major, are dealt to the CTAs in contiguous runs, and a CTA sweeps its run column by
// column.  Thread (rr, g) owns row rr - 1 of the strip (rr = 0 and RH - 1 are the one-row halo) and column
// group g of the panel.  Per column step a thread builds x1 of its row of column c into a four-column ring in
// shared memory, the CTA synchronises once, and the strip's threads apply the 9 diagonals to column c - 1 out
// of the ring.  So each x1 is built once (the halo rows add 2 / (RH - 2) of P / x0 traffic, against 27 % for
// the 128 x 8 tiles with a recomputed halo this replaces), a row's b and 1/diag are read once for both x0 and
// the Jacobi step, and the prolongator row of column c + 1 is in flight while column c is built.  x1 never
// goes to global memory: against the two-kernel form (k_spmm_win SP_ADD then k_stencil SP_JACOBI_DOT) that
// saves the write and both re-reads of the x panel.  Per element the arithmetic is that of the two-kernel
// form: the P terms summed in slot order onto x0, the 9 diagonal terms in slot order.
// ---------------------------------------------------------------------------
constexpr int PJ_RING = 4;   // x1 columns in shared memory: c - 2 (still being read by slow threads), c - 1, c, c + 1
constexpr int PJ_MINB_F32 = 3;   // CTAs per SM of k_stencil_prolong_jacobi (see below)
constexpr int PJ_MINB_F64 = 2;

template <typename T> struct CsrP {
  const int* rowptr;
  const int* colidx;
  const T* vals;
  // ELL-4 copy (slot-major, ld apart; unused slots: column 0, value 0) when no row has more than 4
  // entries -- the prolongator of a regular grid; null otherwise
  const int* ell_col;
  const T* ell_val;
  size_t ell_ld;
};

template <typename T, int KT> struct PjShape {
  static constexpr int V16 = 16 / (int)sizeof(T);
  static constexpr int CPT = KT < V16 ? KT : V16;     // panel columns per thread (one 16-byte vector)
  static constexpr int CG = KT / CPT;                 // column groups per row
  static constexpr int RH = NT / CG;                  // strip rows + the two halo rows
  static constexpr int RPS = RH - 2;                  // rows per strip
  // fp32: the 9 diagonal values of a row wait for the Jacobi step in shared memory (fp64: in registers)
  static constexpr bool VSMEM = sizeof(T) == 4;
  // the x1 ring, per thread the b vector and omega / diag of its row, and (VSMEM) per strip row its 9
  // diagonal values, the last two double-buffered by column parity.  A half-form operator keeps 5 upper-slot
  // values per strip row in three buffers by column (rel % 3): the lower slots of column c - 1 are read from
  // column c - 2's buffer, which the step of column c + 1 must not refill yet; 15 RH <= 18 RH.
  static constexpr int SMEM = (PJ_RING * RH * KT + 2 * NT * CPT + 2 * NT + (VSMEM ? 2 * 9 * RH : 0)) * (int)sizeof(T);
};

// MINB: CTAs per SM the register budget is cut for (launch_prolong_jacobi).  The b.z partial sums are
// double in every instantiation.  What waits for the Jacobi step of the next column step -- the row's b and
// omega / diag, and in fp32 its 9 diagonal values (cp.async) -- waits in shared memory, not in registers:
// that keeps the fp32 variants within the 80 registers of three CTAs per SM without spills.  Measured on an
// H100 80GB HBM3 (700 W), fp32 k = 8 on the 3163^2 raster, with those values still in registers: one PCG
// iteration took 4.30 ms at MINB = 2 (no spills), 4.14 ms at 3 and 4.04 ms at 4, where ptxas spilled 16-48 B
// of the SP_JACOBI_DOT variant.  With the shared-memory slots MINB = 3 is spill-free; MINB = 4 (64 registers)
// still spills.  fp64 needs up to 128 registers (k = 1) and keeps its diagonals in registers: MINB = 2.
template <typename T, int KT, int MODE, int MINB>
__global__ void __launch_bounds__(NT, MINB)
k_stencil_prolong_jacobi(const DiaDev<T> A, const CsrP<T> P, const T* __restrict__ Yc, const T* __restrict__ X0,
                         T* __restrict__ Z, const SpmmEpi<T> ep) {
  static_assert(MODE == SP_JACOBI || MODE == SP_JACOBI_DOT, "post-smoothing modes only");
  using S = PjShape<T, KT>;
  constexpr int CPT = S::CPT, CG = S::CG, RH = S::RH, RPS = S::RPS;
  extern __shared__ __align__(16) unsigned char pj_smem[];
  T* xs = reinterpret_cast<T*>(pj_smem);                 // [PJ_RING][RH][KT]
  T* bsm = xs + PJ_RING * RH * KT;                       // [2][NT][CPT]
  T* wsm = bsm + 2 * NT * CPT;                           // [2][NT]
  T* vsm = wsm + 2 * NT;                                 // [2][9][RH] (VSMEM)
  const int tid = threadIdx.x;
  const int g = tid % CG, rr = tid / CG, c0 = g * CPT;
  const bool inner = rr >= 1 && rr <= RPS;
  const int n = A.n, nr = A.nr;
  const int ncol = (n + nr - 1) / nr;
  const int nstrip = (nr + RPS - 1) / RPS;
  // nstep <= nr * ncol < n + nr: int for every operator launch_prolong_jacobi accepts (n + nr < 2^31)
  const int nstep = nstrip * ncol;
  const int per = (nstep + (int)gridDim.x - 1) / (int)gridDim.x;
  const int s_beg = (int)min((long long)nstep, (long long)blockIdx.x * per);
  const int s_end = (int)min((long long)nstep, ((long long)blockIdx.x + 1) * per);
  const bool ell = P.ell_col != nullptr;
  double dot0[CPT];
#pragma unroll
  for (int i = 0; i < CPT; ++i) dot0[i] = 0.0;

  for (int s0 = s_beg; s0 < s_end;) {
    // one segment: raster columns [cb, ce) of one strip
    const int strip = s0 / ncol, cb = s0 % ncol;
    const int ce = min(ncol, cb + (s_end - s0));
    s0 += ce - cb;
    const int r = strip * RPS + rr - 1;                  // this thread's row within a raster column
    const bool rok = r >= 0 && r < nr;
    auto row_of = [&](int c, int& row) {
      const long long rl = (long long)c * nr + r;
      const bool ok = rok && c >= 0 && c < ncol && rl < n;
      row = ok ? (int)rl : 0;                            // out of the raster: x1 = 0, any row will do for the loads
      return ok;
    };
    auto ell_row = [&](int row, int (&cj)[4], T (&pv)[4]) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        cj[q] = __ldg(P.ell_col + (size_t)q * P.ell_ld + row);
        pv[q] = __ldg(P.ell_val + (size_t)q * P.ell_ld + row);
      }
    };
    int rowc, rowp = 0;
    bool okc = row_of(cb - 1, rowc), okp = false;
    int cj[4] = {0, 0, 0, 0};
    T pv[4] = {T(0), T(0), T(0), T(0)};
    if (ell) ell_row(rowc, cj, pv);
    __syncthreads();                                     // the ring's readers of the previous segment are done
    for (int c = cb - 1; c <= ce; ++c) {
      const int rel = c - (cb - 1);                      // ring slot of column c: rel % PJ_RING
      const bool zdo = inner && c > cb && okp;           // z of column c - 1 (row rowp) after the barrier
      // ---- loads: diagonals of column c - 1, the prolongator row of column c + 1, then b, 1/diag, x0 and the
      //      y gathers of column c
      T v[9];
      if constexpr (S::VSMEM) {
        // straight to shared memory (cp.async), one copy per row by its column group 0
        if (A.half) {
          // the upper-slot runs of column c - 1, every strip row (the halo rows too, for the lower slots of the
          // rows next to them): all 5 where it is computed (c > cb), 6 ... 8 (the lower slots 0 ... 2 of column c)
          // where it is only the left neighbour of one (c = cb); zero for rows outside the raster, as halve_dia
          // demands
          if (g == 0) {
            const int u0 = c > cb ? 0 : 2, u1 = c >= cb ? 5 : 2;
            for (int u = u0; u < u1; ++u)
              cp_async_zfill<(int)sizeof(T)>(vsm + ((rel % 3) * 5 + u) * RH + rr, A.run(4 + u) + rowp, okp);
          }
        } else if (zdo && g == 0) {
#pragma unroll
          for (int s = 0; s < 9; ++s)
            asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(smem_u32(vsm + ((rel & 1) * 9 + s) * RH + rr)),
                         "l"(A.run(s) + rowp), "n"((int)sizeof(T)) : "memory");
        }
      } else {
#pragma unroll
        for (int s = 0; s < 9; ++s)   // streamed once; half: the lower slots straight from the neighbour rows
          v[s] = zdo ? (A.half && s < 4 ? A.at(s, rowp) : __ldcs(A.run(s) + rowp)) : T(0);
      }
      int rown;
      const bool okn = row_of(c + 1, rown);
      int cjn[4] = {0, 0, 0, 0};
      T pvn[4] = {T(0), T(0), T(0), T(0)};
      if (ell && c < ce) ell_row(rown, cjn, pvn);
      T bc[CPT], x1[CPT];
      ldvec<T, CPT>(ep.B + (size_t)rowc * KT + c0, bc);
      const T wc = ep.omega * ep.dinv[rowc];
      if (X0) {
        ldvec<T, CPT>(X0 + (size_t)rowc * KT + c0, x1);
      } else {                                           // x0 = omega D^-1 b, never stored
#pragma unroll
        for (int i = 0; i < CPT; ++i) x1[i] = bc[i] * wc;
      }
      if (ell) {
        T yv[4][CPT];
#pragma unroll
        for (int q = 0; q < 4; ++q) ldvec<T, CPT>(Yc + (size_t)cj[q] * KT + c0, yv[q]);
#pragma unroll
        for (int i = 0; i < CPT; ++i) {
          T a = x1[i];
#pragma unroll
          for (int q = 0; q < 4; ++q) a += pv[q] * yv[q][i];
          x1[i] = okc ? a : T(0);
        }
      } else if (okc) {                                  // plain CSR (rows with more than 4 entries)
        const int a = P.rowptr[rowc], b = P.rowptr[rowc + 1];
        int cq[4];
        T pq[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const bool ok = a + q < b;
          cq[q] = ok ? __ldg(P.colidx + a + q) : 0;
          pq[q] = ok ? __ldg(P.vals + a + q) : T(0);
        }
        T yv[4][CPT];
#pragma unroll
        for (int q = 0; q < 4; ++q) ldvec<T, CPT>(Yc + (size_t)cq[q] * KT + c0, yv[q]);
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
          for (int i = 0; i < CPT; ++i) x1[i] += pq[q] * yv[q][i];
        for (int j = a + 4; j < b; ++j) {
          const T pw = P.vals[j];
          T yw[CPT];
          ldvec<T, CPT>(Yc + (size_t)P.colidx[j] * KT + c0, yw);
#pragma unroll
          for (int i = 0; i < CPT; ++i) x1[i] += pw * yw[i];
        }
      } else {
#pragma unroll
        for (int i = 0; i < CPT; ++i) x1[i] = T(0);
      }
      stvec<T, CPT>(xs + ((size_t)(rel % PJ_RING) * RH + rr) * KT + c0, x1);
      stvec<T, CPT>(bsm + ((rel & 1) * NT + tid) * CPT, bc);     // for the Jacobi step of column c (next step)
      wsm[(rel & 1) * NT + tid] = wc;
      if constexpr (S::VSMEM) asm volatile("cp.async.wait_all;" ::: "memory");
      __syncthreads();
      // ---- z = x1 + omega D^-1 (b - A x1) on column c - 1
      if (zdo) {
        T acc[CPT], xo[CPT];
#pragma unroll
        for (int i = 0; i < CPT; ++i) acc[i] = T(0);
#pragma unroll
        for (int s = 0; s < 9; ++s) {
          // half: a lower slot is upper slot 8 - s of row rr + s % 3 - 1 of column c - 1 + s / 3 - 1
          const T vs = !S::VSMEM ? v[s]
                       : !A.half ? vsm[((rel & 1) * 9 + s) * RH + rr]
                       : s >= 4  ? vsm[((rel % 3) * 5 + s - 4) * RH + rr]
                                 : vsm[(((rel + (s / 3 == 1 ? 0 : 2)) % 3) * 5 + 4 - s) * RH + rr + s % 3 - 1];
          T xv[CPT];
          ldvec<T, CPT>(xs + ((size_t)((rel + s / 3 - 2) % PJ_RING) * RH + (rr + s % 3 - 1)) * KT + c0, xv);
#pragma unroll
          for (int i = 0; i < CPT; ++i) {
            acc[i] += vs * xv[i];
            if (s == 4) xo[i] = xv[i];
          }
        }
        T bp[CPT], out[CPT];                             // b and omega / diag of row rowp, stored one step back
        ldvec<T, CPT>(bsm + ((~rel & 1) * NT + tid) * CPT, bp);
        const T wp = wsm[(~rel & 1) * NT + tid];
#pragma unroll
        for (int i = 0; i < CPT; ++i) {
          const T zn = xo[i] + wp * (bp[i] - acc[i]);
          out[i] = zn;
          if (MODE == SP_JACOBI_DOT) dot0[i] += (double)bp[i] * (double)zn;
        }
        stvec<T, CPT>(Z + (size_t)rowp * KT + c0, out);
      }
      rowp = rowc;
      okp = okc;
      rowc = rown;
      okc = okn;
#pragma unroll
      for (int q = 0; q < 4; ++q) { cj[q] = cjn[q]; pv[q] = pvn[q]; }
    }
  }
  if (MODE == SP_JACOBI_DOT) {
    CSB_REDUCE_SMEM(1, KT)
    double v[1][CPT];
#pragma unroll
    for (int i = 0; i < CPT; ++i) v[0][i] = dot0[i];
    if (grid_reduce<KT, CPT, 1, false>(v, ep.partials, &ep.ctl->ticket, s_warp, s_tree, s_out))
      cg_after_precond<KT>(ep.ctl, s_out);
  }
}

// Build the per-block records of the windowed form on the device: one CTA per block copies
// the values (through the host-built permutation), the 16-bit local columns and the row
// offsets into  blob + blob_off16*16 :  [ values nnzp | lcol nnzp | roff roffp ].
template <typename T>
__global__ void k_pack_blob(int nblocks, const WinMeta* __restrict__ meta, const int* __restrict__ perm,
                            const unsigned short* __restrict__ lcol, const unsigned short* __restrict__ roff,
                            const int* __restrict__ roff_off, const T* __restrict__ vals,
                            const T* __restrict__ dinv /* null: no 1/diag section */,
                            unsigned char* __restrict__ blob) {
  for (int b = blockIdx.x; b < nblocks; b += gridDim.x) {
    const WinMeta m = meta[b];
    if (m.nseg == 0) continue;
    const int nnzp = (m.nnz + 7) / 8 * 8;
    const int roffp = (m.nrows + 1 + 7) / 8 * 8;
    unsigned char* rec = blob + (size_t)m.blob_off16 * 16;
    T* v = reinterpret_cast<T*>(rec);
    const int rowsp = dinv ? (m.nrows + 7) / 8 * 8 : 0;
    T* dv = v + nnzp;
    unsigned short* lc = reinterpret_cast<unsigned short*>(dv + rowsp);
    unsigned short* ro = lc + nnzp;
    for (int i = threadIdx.x; i < rowsp; i += blockDim.x) dv[i] = i < m.nrows ? dinv[m.row0 + i] : T(0);
    for (int i = threadIdx.x; i < nnzp; i += blockDim.x) {
      const int p = perm[(size_t)m.ent_off + i];
      v[i] = p >= 0 ? vals[p] : T(0);
      lc[i] = lcol[(size_t)m.ent_off + i];
    }
    const int r0 = roff_off[b];
    for (int i = threadIdx.x; i < roffp; i += blockDim.x) ro[i] = i <= m.nrows ? roff[(size_t)r0 + i] : (unsigned short)0;
  }
}

// ---------------------------------------------------------------------------
// element-wise panel kernels.  Element e = row*KT + col; thread walks vectors of
// VEC = 16/sizeof(T) elements with a grid stride that is a multiple of KT.
// ---------------------------------------------------------------------------

// init (Jacobi):  X = 0, R = B, P = Dinv R, rho0 = R.Dinv R ; last CTA: tolerances.
template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_cg_init(size_t nelem, const T* __restrict__ B, const T* __restrict__ dinv, T* __restrict__ X,
          T* __restrict__ R, T* __restrict__ P, PanelCtl* ctl, double* partials, double rtol,
          double atol, int itmax) {
  constexpr int VEC = Vec<T>::N;
  constexpr int L = Log2<KT>::v;
  CSB_REDUCE_SMEM(1, KT)
  const size_t stride = (size_t)gridDim.x * NT * VEC;
  double acc[1][VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) acc[0][i] = 0.0;
  for (size_t e = ((size_t)blockIdx.x * NT + threadIdx.x) * VEC; e < nelem; e += stride) {
    T b[VEC], p[VEC], z[VEC];
    vload(B + e, b);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const T d = dinv[(e + i) >> L];
      p[i] = d * b[i];
      acc[0][i] += (double)b[i] * (double)p[i];
      z[i] = T(0);
    }
    vstore(R + e, b);
    vstore(P + e, p);
    vstore(X + e, z);
  }
  if (grid_reduce<KT, VEC, 1, false>(acc, partials, &ctl->ticket, s_warp, s_tree, s_out)) {
    const int c = threadIdx.x;
    if (c < KT) {
      const double rho = s_out[c];
      const double tol = atol + rtol * sqrt(rho);
      ctl->rho[c] = rho;
      ctl->rho0[c] = rho;
      ctl->tol[c] = tol;
      ctl->active[c] = (rho > 0.0 && sqrt(rho) > tol && itmax > 0) ? 1 : 0;
      ctl->iters[c] = 0;
      ctl->alpha[c] = 0.0;
      ctl->beta[c] = 0.0;
      ctl->best[c] = rho;
      ctl->stall[c] = 0;
      ctl->stalled[c] = 0;
    }
    __syncthreads();
    if (c == 0) {
      int na = 0;
      for (int k = 0; k < KT; ++k) na += ctl->active[k];
      ctl->nactive = na;
      ctl->iter = 0;
      ctl->itmax = itmax;
    }
  }
}

// K2:  R -= alpha*AP ;  rho_new = R.Dinv R ;  last CTA: beta, convergence, freeze.
template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_cg_update_r(size_t nelem, const T* __restrict__ AP, const T* __restrict__ dinv,
              T* __restrict__ R, PanelCtl* ctl, double* partials) {
  constexpr int VEC = Vec<T>::N;
  constexpr int L = Log2<KT>::v;
  CSB_REDUCE_SMEM(1, KT)
  const size_t e0 = ((size_t)blockIdx.x * NT + threadIdx.x) * VEC;
  const size_t stride = (size_t)gridDim.x * NT * VEC;
  T al[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) al[i] = (T)ctl->alpha[(e0 + i) % KT];
  double acc[1][VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) acc[0][i] = 0.0;
  for (size_t e = e0; e < nelem; e += stride) {
    T r[VEC], ap[VEC];
    vload(R + e, r);
    vload(AP + e, ap);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      r[i] -= al[i] * ap[i];
      acc[0][i] += (double)r[i] * (double)r[i] * (double)dinv[(e + i) >> L];
    }
    vstore(R + e, r);
  }
  if (grid_reduce<KT, VEC, 1, false>(acc, partials, &ctl->ticket, s_warp, s_tree, s_out)) {
    const int c = threadIdx.x;
    const int it = ctl->iter + 1;
    if (c < KT) {
      if (ctl->active[c]) {
        const double rn = s_out[c];
        const double ro = ctl->rho[c];
        ctl->beta[c] = ro > 0.0 ? rn / ro : 0.0;
        ctl->rho[c] = rn;
        ctl->iters[c] = it;
        if (rn < 0.81 * ctl->best[c]) { ctl->best[c] = rn; ctl->stall[c] = 0; }
        else if (++ctl->stall[c] >= ctl->stall_limit && ctl->stall_limit > 0) { ctl->stalled[c] = 1; ctl->active[c] = 0; }
        if (!(sqrt(rn) > ctl->tol[c]) || it >= ctl->itmax) ctl->active[c] = 0;
      } else {
        ctl->beta[c] = 0.0;
      }
    }
    __syncthreads();
    if (c == 0) {
      int na = 0;
      for (int k = 0; k < KT; ++k) na += ctl->active[k];
      ctl->nactive = na;
      ctl->iter = it;
    }
  }
}

// K3:  X += alpha*P ;  P = Dinv R + beta*P
template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_cg_update_xp(size_t nelem, const T* __restrict__ R, const T* __restrict__ dinv,
               T* __restrict__ X, T* __restrict__ P, const PanelCtl* ctl) {
  constexpr int VEC = Vec<T>::N;
  constexpr int L = Log2<KT>::v;
  const size_t e0 = ((size_t)blockIdx.x * NT + threadIdx.x) * VEC;
  const size_t stride = (size_t)gridDim.x * NT * VEC;
  T al[VEC], be[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    al[i] = (T)ctl->alpha[(e0 + i) % KT];
    be[i] = (T)ctl->beta[(e0 + i) % KT];
  }
  for (size_t e = e0; e < nelem; e += stride) {
    T r[VEC], x[VEC], p[VEC];
    vload(R + e, r);
    vload(X + e, x);
    vload(P + e, p);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      x[i] += al[i] * p[i];
      p[i] = dinv[(e + i) >> L] * r[i] + be[i] * p[i];
    }
    vstore(X + e, x);
    vstore(P + e, p);
  }
}

// AMG-PCG, after the SpMM:  R -= alpha*AP ;  X0 = omega * Dinv * R   (the zero-guess
// pre-smoothing sweep of the finest level is folded in: one pass fewer over R).
// TV = type of the V-cycle panels: with TV = float (mixed precision) the kernel also
// writes the rounded residual R32 the fp32 cycle starts from.
template <typename T, int KT, typename TV>
__global__ void __launch_bounds__(NT)
k_cg_update_r0(size_t nelem, const T* __restrict__ AP, const T* __restrict__ dinv, T omega,
               T* __restrict__ R, TV* __restrict__ X0, TV* __restrict__ R32, const PanelCtl* ctl) {
  constexpr int VEC = Vec<T>::N;
  constexpr int L = Log2<KT>::v;
  const size_t e0 = ((size_t)blockIdx.x * NT + threadIdx.x) * VEC;
  const size_t stride = (size_t)gridDim.x * NT * VEC;
  T al[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) al[i] = (T)ctl->alpha[(e0 + i) % KT];
  for (size_t e = e0; e < nelem; e += stride) {
    T ap[VEC], r[VEC];
    TV x0[VEC], r32[VEC];
    vload(AP + e, ap);
    vload(R + e, r);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      r[i] -= al[i] * ap[i];
      x0[i] = (TV)(omega * dinv[(e + i) >> L] * r[i]);
      r32[i] = (TV)r[i];
    }
    vstore(R + e, r);
    if (X0) stvec<TV, VEC>(X0 + e, x0);        // null: the level-0 kernels form omega D^-1 r on the fly
    if (R32) stvec<TV, VEC>(R32 + e, r32);
  }
}

// AMG-PCG, after the V-cycle:  X += alpha*P (the deferred solution update) ;  P = Z + beta*P
template <typename T, int KT, typename TV>
__global__ void __launch_bounds__(NT)
k_cg_update_xp2(size_t nelem, const TV* __restrict__ Z, T* __restrict__ X, T* __restrict__ P,
                const PanelCtl* ctl) {
  constexpr int VEC = Vec<T>::N;
  const size_t e0 = ((size_t)blockIdx.x * NT + threadIdx.x) * VEC;
  const size_t stride = (size_t)gridDim.x * NT * VEC;
  T al[VEC], be[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    al[i] = (T)ctl->alpha[(e0 + i) % KT];
    be[i] = (T)ctl->beta[(e0 + i) % KT];
  }
  for (size_t e = e0; e < nelem; e += stride) {
    TV z[VEC];
    T p[VEC], x[VEC];
    ldvec<TV, VEC>(Z + e, z);
    vload(P + e, p);
    vload(X + e, x);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      x[i] += al[i] * p[i];
      p[i] = (T)z[i] + be[i] * p[i];
    }
    vstore(X + e, x);
    vstore(P + e, p);
  }
}

// after a loop of K = ctl->iter fused CG steps (k_stencil_cg): the x updates still pending, in order --
// p_{K-1}, preceded by p_{K-2} when K is odd (the last pair went in at step K - 2).  x is the panel's zero start
// while K <= 1 and p_{-1} is zero (K = 0): those are not read, as in the CG step, so X and P need no fill.
template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_cg_x_tail(size_t nelem, const T* __restrict__ Pb0, const T* __restrict__ Pb1, T* __restrict__ X,
            const PanelCtl* ctl) {
  constexpr int VEC = Vec<T>::N;
  const int K = ctl->iter;
  const bool two = K & 1;
  const bool x_live = K > 1, p_live = K > 0;   // x_live: also p_{K-2} is not p_{-1}
  const T* p2 = (K & 1) ? Pb1 : Pb0;         // p_{K-2} (j = -1: the zero p_{-1} with alpha 0)
  const T* p1 = (K & 1) ? Pb0 : Pb1;         // p_{K-1}
  const size_t e0 = ((size_t)blockIdx.x * NT + threadIdx.x) * VEC;
  const size_t stride = (size_t)gridDim.x * NT * VEC;
  T a1[VEC], a2[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    a1[i] = (T)ctl->alpha_ring[(K + 2) % 3][(e0 + i) % KT];
    a2[i] = (T)ctl->alpha_ring[(K + 1) % 3][(e0 + i) % KT];
  }
  for (size_t e = e0; e < nelem; e += stride) {
    T x[VEC], q1[VEC], q2[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) x[i] = q1[i] = q2[i] = T(0);
    if (x_live) vload(X + e, x);
    if (p_live) vload(p1 + e, q1);
    if (two) {
      if (x_live) vload(p2 + e, q2);           // K = 1: p_{-1}
#pragma unroll
      for (int i = 0; i < VEC; ++i) x[i] += a2[i] * q2[i];
    }
#pragma unroll
    for (int i = 0; i < VEC; ++i) x[i] += a1[i] * q1[i];
    vstore(X + e, x);
  }
}

// panel conversion (mixed-precision start-up: R32 = (float) R)
template <typename TI, typename TO>
__global__ void __launch_bounds__(NT)
k_convert(size_t nelem, const TI* __restrict__ in, TO* __restrict__ out) {
  for (size_t e = (size_t)blockIdx.x * NT + threadIdx.x; e < nelem; e += (size_t)gridDim.x * NT)
    out[e] = (TO)in[e];
}

// start of a fused AMG-PCG panel in one pass: r = b into R and, on mixed handles, r32 = (float) r into R32 (R32
// null otherwise).  b: B, or with B null the pairs rule of ctl (pair_rhs_val), so a pairs panel never writes B.
// The values are those of filling B, copying it to R and k_convert.
template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_panel_start(size_t nelem, const T* __restrict__ B, T* __restrict__ R, float* __restrict__ R32,
              const PanelCtl* __restrict__ ctl) {
  constexpr int VEC = Vec<T>::N;
  const size_t stride = (size_t)gridDim.x * NT * VEC;
  for (size_t e = ((size_t)blockIdx.x * NT + threadIdx.x) * VEC; e < nelem; e += stride) {
    T r[VEC];
    if (B) {
      vload(B + e, r);
    } else {
#pragma unroll
      for (int i = 0; i < VEC; ++i) r[i] = pair_rhs_at<T, KT>(ctl, e + i);
    }
    vstore(R + e, r);
    if (R32) {
      if constexpr (VEC == 2)
        *reinterpret_cast<float2*>(R32 + e) = make_float2((float)r[0], (float)r[1]);
      else
        *reinterpret_cast<float4*>(R32 + e) = make_float4((float)r[0], (float)r[1], (float)r[2], (float)r[3]);
    }
  }
}

// first (zero-guess) damped-Jacobi sweep of a level:  X = omega * Dinv * B
template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_jacobi0(size_t nelem, const T* __restrict__ B, const T* __restrict__ dinv, T omega,
          T* __restrict__ X) {
  constexpr int VEC = Vec<T>::N;
  constexpr int L = Log2<KT>::v;
  const size_t stride = (size_t)gridDim.x * NT * VEC;
  for (size_t e = ((size_t)blockIdx.x * NT + threadIdx.x) * VEC; e < nelem; e += stride) {
    T b[VEC], x[VEC];
    vload(B + e, b);
#pragma unroll
    for (int i = 0; i < VEC; ++i) x[i] = omega * dinv[(e + i) >> L] * b[i];
    vstore(X + e, x);
  }
}

// coarsest level:  X = Pinv * B  (dense n x n pseudo-inverse in double).  One thread per
// output (row, column), 4 independent accumulators; launched over ceil(n*KT/NT) CTAs.
template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_coarse_dense(int n, const double* __restrict__ pinv, const T* __restrict__ B, T* __restrict__ X) {
  const int e = blockIdx.x * NT + threadIdx.x;
  if (e >= n * KT) return;
  const int i = e / KT, c = e % KT;
  const double* row = pinv + (size_t)i * n;
  double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
  int j = 0;
  for (; j + 3 < n; j += 4) {
    a0 += row[j] * (double)B[(size_t)j * KT + c];
    a1 += row[j + 1] * (double)B[(size_t)(j + 1) * KT + c];
    a2 += row[j + 2] * (double)B[(size_t)(j + 2) * KT + c];
    a3 += row[j + 3] * (double)B[(size_t)(j + 3) * KT + c];
  }
  for (; j < n; ++j) a0 += row[j] * (double)B[(size_t)j * KT + c];
  X[e] = (T)((a0 + a1) + (a2 + a3));
}

// loop condition of the device-side PCG loop (CUDA-graph WHILE node): keep iterating while
// any column of the panel is active.  Runs as the node before the loop and as the last
// node of the loop body.
__global__ void k_loop_cond(cudaGraphConditionalHandle handle, const PanelCtl* __restrict__ ctl) {
  cudaGraphSetConditional(handle, (ctl->nactive > 0 && ctl->iter < ctl->itmax) ? 1u : 0u);
}

// ---------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------
// Dinv[i] = 1/A_ii (0 for pad rows / missing diagonals)
template <typename T>
__global__ void k_dinv(int n, int n_pad, const int* __restrict__ rowptr,
                       const int* __restrict__ colidx, const T* __restrict__ vals, T* dinv) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_pad; i += gridDim.x * blockDim.x) {
    T d = T(0);
    if (i < n)
      for (int j = rowptr[i]; j < rowptr[i + 1]; ++j)
        if (colidx[j] == i) d += vals[j];
    dinv[i] = d != T(0) ? T(1) / d : T(0);
  }
}

// B panel for focal pairs:  -1 at src, +1 at dst  (core.jl:224-226, 459-460); B pre-zeroed.
template <typename T, int KT>
__global__ void k_pair_rhs(T* B, const PanelCtl* ctl) {
  const int c = threadIdx.x;
  if (c < KT) {
    const long long s = ctl->src[c], d = ctl->dst[c];
    if (s >= 0 && d >= 0 && s != d) {
      B[(size_t)s * KT + c] = T(-1);
      B[(size_t)d * KT + c] = T(1);
    }
  }
}

template <typename T, int KT>
__global__ void k_pair_extract(const T* X, PanelCtl* ctl) {
  const int c = threadIdx.x;
  if (c < KT) {
    const long long s = ctl->src[c], d = ctl->dst[c];
    ctl->xsrc[c] = s >= 0 ? (double)X[(size_t)s * KT + c] : 0.0;
    ctl->xdst[c] = d >= 0 ? (double)X[(size_t)d * KT + c] : 0.0;
  }
}

// sparse right-hand sides of a panel: column c owns entries ent_ptr[c] .. ent_ptr[c+1]-1;
// one thread per column adds its entries in order (deterministic, duplicates add)
template <typename T, int KT>
__global__ void k_sparse_rhs(T* B, const int* __restrict__ ent_ptr, const long long* __restrict__ rows,
                             const double* __restrict__ vals) {
  const int c = threadIdx.x;
  if (c < KT)
    for (int e = ent_ptr[c]; e < ent_ptr[c + 1]; ++e) B[(size_t)rows[e] * KT + c] += (T)vals[e];
}

// out[c][i] = X[probe[i]][c] - xsrc[c]   (voltages at the probe rows after the shift)
template <typename T, int KT>
__global__ void k_probe(const T* __restrict__ X, const PanelCtl* __restrict__ ctl,
                        const long long* __restrict__ probe, int nprobe, T* __restrict__ out) {
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < nprobe * KT; e += gridDim.x * blockDim.x) {
    const int c = e / nprobe, i = e % nprobe;
    out[e] = (T)((double)X[(size_t)probe[i] * KT + c] - ctl->xsrc[c]);
  }
}

// superposition driver: X[:, c] = U[:, cj[c]] - U[:, ci[c]] on a panel (U column-major with
// leading dimension n_pad; column index -1 = the reference node's identically-zero solution)
template <typename T, int KT>
__global__ void k_combine(int n, size_t n_pad, const T* __restrict__ U, const int* __restrict__ ci,
                          const int* __restrict__ cj, T* __restrict__ X) {
  const size_t total = n_pad * KT;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t i = e / KT;
    const int c = (int)(e % KT);
    T v = T(0);
    if (i < (size_t)n) {
      const int a = ci[c], b = cj[c];
      v = (b >= 0 ? U[(size_t)b * n_pad + i] : T(0)) - (a >= 0 ? U[(size_t)a * n_pad + i] : T(0));
    }
    X[e] = v;
  }
}

// staging (column-major n x KT, leading dimension ld) <-> panel (row-major n_pad x KT)
template <typename T, int KT>
__global__ void k_cm_to_panel(int n, size_t ld, const T* __restrict__ cm, T* __restrict__ panel,
                              int ncols) {
  const size_t total = (size_t)n * KT;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total;
       e += (size_t)gridDim.x * blockDim.x) {
    const size_t i = e / KT;
    const int c = (int)(e % KT);
    panel[e] = c < ncols ? cm[(size_t)c * ld + i] : T(0);
  }
}
// out[c*ld + i] = panel[i][c] - shift[c]
template <typename T, int KT>
__global__ void k_panel_to_cm(int n, size_t ld, const T* __restrict__ panel, T* __restrict__ cm,
                              const PanelCtl* ctl, int use_shift) {
  const size_t total = (size_t)n * KT;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total;
       e += (size_t)gridDim.x * blockDim.x) {
    const size_t i = e / KT;
    const int c = (int)(e % KT);
    const T sh = use_shift ? (T)ctl->xsrc[c] : T(0);
    cm[(size_t)c * ld + i] = panel[e] - sh;
  }
}

// ---------------------------------------------------------------------------
// node currents (out.jl:178-290).  With d_ij = |a_ij| (v_i - v_j):
//   maxpos = max over stored i<j of  d_ij ; maxneg = max over i<j of -d_ij
//   inflow_i  = sum_j max(-d_ij,0) over entries with |d_ij/maxpos| >= 1e-8
//   outflow_i = sum_j max( d_ij,0) over entries with |d_ij/maxneg| >= 1e-8
//   node current = inflow > outflow ? inflow : outflow
// which is the row-wise restatement of  B = triu branch currents; B - B'; drop
// negatives; column sums  done once with the `pos` and once with the `neg` signs.
// With finite grounds fg (k_cur_acc[_dia], non-null only for cs_b200_solve_advanced), x_i = fg_i v_i
// adds its ground current to one side before the max (out.jl:193-202): -x_i to inflow when x_i < 0,
// x_i to outflow when x_i > 0.  The 1e-8 cut does not apply to it.
// ---------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ void ground_current(T x, T& inflow, T& outflow) {
  if (x < T(0)) inflow -= x;
  if (x > T(0)) outflow += x;
}

template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_cur_max(int n, const int* __restrict__ rowptr, const int* __restrict__ colidx,
          const T* __restrict__ vals, const T* __restrict__ V, PanelCtl* ctl, double* partials) {
  CSB_REDUCE_SMEM(2, KT)
  const int c = threadIdx.x % KT;
  constexpr int RPP = NT / KT;
  double mp = -1.0e300, mn = -1.0e300;
  for (int row = blockIdx.x * RPP + threadIdx.x / KT; row < n; row += gridDim.x * RPP) {
    const T vi = V[(size_t)row * KT + c];
    for (int j = rowptr[row]; j < rowptr[row + 1]; ++j) {
      const int col = colidx[j];
      if (col > row) {
        const T d = fabs(vals[j]) * (vi - V[(size_t)col * KT + c]);
        mp = fmax(mp, (double)d);
        mn = fmax(mn, (double)(-d));
      }
    }
  }
  double v[2][1] = {{mp}, {mn}};
  if (grid_reduce<KT, 1, 2, true>(v, partials, &ctl->ticket, s_warp, s_tree, s_out)) {
    if (threadIdx.x < KT) {
      ctl->maxpos[threadIdx.x] = s_out[threadIdx.x];
      ctl->maxneg[threadIdx.x] = s_out[KT + threadIdx.x];
    }
  }
}

template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_cur_acc(int n, const int* __restrict__ rowptr, const int* __restrict__ colidx,
          const T* __restrict__ vals, const T* __restrict__ V, const T* __restrict__ fg, const PanelCtl* ctl,
          T* __restrict__ cur_out /*panel or null*/, T* __restrict__ cum, T* __restrict__ mx,
          int accumulate, int log_transform, int ncols) {
  const int c = threadIdx.x % KT;
  constexpr int RPP = NT / KT;
  const T maxpos = (T)ctl->maxpos[c], maxneg = (T)ctl->maxneg[c];
  const double w = ctl->weight[c];
  const int nrow_iter = (n + RPP - 1) / RPP;
  for (int it = blockIdx.x; it < nrow_iter; it += gridDim.x) {
    const int row = it * RPP + threadIdx.x / KT;
    T cur = T(0);
    if (row < n) {
      const T vi = V[(size_t)row * KT + c];
      T inflow = T(0), outflow = T(0);
      for (int j = rowptr[row]; j < rowptr[row + 1]; ++j) {
        const int col = colidx[j];
        if (col == row) continue;
        const T d = fabs(vals[j]) * (vi - V[(size_t)col * KT + c]);
        if (!(fabs(d / maxneg) < T(1e-8)) && d > T(0)) outflow += d;
        if (!(fabs(d / maxpos) < T(1e-8)) && d < T(0)) inflow -= d;
      }
      if (fg) ground_current(fg[row] * vi, inflow, outflow);
      cur = inflow > outflow ? inflow : outflow;
      if (cur_out) cur_out[(size_t)row * KT + c] = cur;
    }
    if (accumulate) {
      // out.jl:305-309 (log transform) then out.jl:100-107 (cum += , max = max)
      T val = cur;
      if (log_transform) val = cur > T(0) ? (T)log10((double)cur) : T(-9999);
      const unsigned mask = 0xffffffffu;
      const int lane = threadIdx.x & 31;
      const int base = lane - c;
      double s = 0.0;
      T m = T(-1.0e30);
#pragma unroll
      for (int cc = 0; cc < KT; ++cc) {
        const T vv = __shfl_sync(mask, val, base + cc);
        const double ww = __shfl_sync(mask, w, base + cc);
        if (cc < ncols && ww != 0.0) {
          s += ww * (double)vv;
          m = vv > m ? vv : m;
        }
      }
      if (c == 0 && row < n) {
        cum[row] = (T)((double)cum[row] + s);
        if (mx) mx[row] = m > mx[row] ? m : mx[row];
      }
    }
  }
}

// the same two passes on the stencil (DIA) form of the operator: 9 coalesced value loads and 9 panel
// gathers per (row, column), no CSR walk (the CSR versions run at ~1/8 of the HBM rate).  Slots
// without a stored entry hold 0 and are skipped, so the candidates of the maxima are the stored ones.
template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_cur_max_dia(const DiaDev<T> A, const T* __restrict__ V, PanelCtl* ctl, double* partials) {
  CSB_REDUCE_SMEM(2, KT)
  const int c = threadIdx.x % KT;
  constexpr int RPP = NT / KT;
  const int n = A.n, nr = A.nr;
  double mp = -1.0e300, mn = -1.0e300;
  for (int row = blockIdx.x * RPP + threadIdx.x / KT; row < n; row += gridDim.x * RPP) {
    T a[4], vj[4];
    const T vi = V[(size_t)row * KT + c];
#pragma unroll
    for (int q = 0; q < 4; ++q) {                       // the four slots with column > row: +1, nr-1, nr, nr+1
      const int s = 5 + q;
      a[q] = __ldg(A.run(s) + row);
      const int j = min(n - 1, row + (s / 3 - 1) * nr + (s % 3 - 1));
      vj[q] = V[(size_t)j * KT + c];
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (a[q] != T(0)) {
        const T d = fabs(a[q]) * (vi - vj[q]);
        mp = fmax(mp, (double)d);
        mn = fmax(mn, (double)(-d));
      }
  }
  double v[2][1] = {{mp}, {mn}};
  if (grid_reduce<KT, 1, 2, true>(v, partials, &ctl->ticket, s_warp, s_tree, s_out)) {
    if (threadIdx.x < KT) {
      ctl->maxpos[threadIdx.x] = s_out[threadIdx.x];
      ctl->maxneg[threadIdx.x] = s_out[KT + threadIdx.x];
    }
  }
}

template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_cur_acc_dia(const DiaDev<T> A, const T* __restrict__ V, const T* __restrict__ fg, const PanelCtl* ctl,
              T* __restrict__ cur_out,
              T* __restrict__ cum, T* __restrict__ mx, int accumulate, int log_transform, int ncols) {
  const int c = threadIdx.x % KT;
  constexpr int RPP = NT / KT;
  const int n = A.n, nr = A.nr;
  const T maxpos = (T)ctl->maxpos[c], maxneg = (T)ctl->maxneg[c];
  const double w = ctl->weight[c];
  const int nrow_iter = (n + RPP - 1) / RPP;
  for (int it = blockIdx.x; it < nrow_iter; it += gridDim.x) {
    const int row = it * RPP + threadIdx.x / KT;
    T cur = T(0);
    if (row < n) {
      T a[9], vj[9];
#pragma unroll
      for (int s = 0; s < 9; ++s) {
        a[s] = A.at(s, row);
        const int j = max(0, min(n - 1, row + (s / 3 - 1) * nr + (s % 3 - 1)));
        vj[s] = V[(size_t)j * KT + c];
      }
      const T vi = vj[4];
      T inflow = T(0), outflow = T(0);
#pragma unroll
      for (int s = 0; s < 9; ++s) {
        if (s == 4) continue;
        const T d = fabs(a[s]) * (vi - vj[s]);
        if (!(fabs(d / maxneg) < T(1e-8)) && d > T(0)) outflow += d;
        if (!(fabs(d / maxpos) < T(1e-8)) && d < T(0)) inflow -= d;
      }
      if (fg) ground_current(fg[row] * vi, inflow, outflow);
      cur = inflow > outflow ? inflow : outflow;
      if (cur_out) cur_out[(size_t)row * KT + c] = cur;
    }
    if (accumulate) {
      T val = cur;
      if (log_transform) val = cur > T(0) ? (T)log10((double)cur) : T(-9999);
      const unsigned mask = 0xffffffffu;
      const int lane = threadIdx.x & 31;
      const int base = lane - c;
      double s = 0.0;
      T m = T(-1.0e30);
#pragma unroll
      for (int cc = 0; cc < KT; ++cc) {
        const T vv = __shfl_sync(mask, val, base + cc);
        const double ww = __shfl_sync(mask, w, base + cc);
        if (cc < ncols && ww != 0.0) {
          s += ww * (double)vv;
          m = vv > m ? vv : m;
        }
      }
      if (c == 0 && row < n) {
        cum[row] = (T)((double)cum[row] + s);
        if (mx) mx[row] = m > mx[row] ? m : mx[row];
      }
    }
  }
}

// ---------------------------------------------------------------------------
// branch currents (out.jl:150-158, 250-290).  The branches of an operator are its stored strictly-lower
// CSR entries (hi, lo < hi), ordered by hi, then lo: the columns of a row ascend, so branch bptr[hi] + t
// is entry rowptr[hi] + t for t < bptr[hi+1] - bptr[hi].  For a symmetric operator this is the order of
// the reference's CSC walk of the upper triangle (_convert_to_3col).
// ---------------------------------------------------------------------------
// cnt[row] = the row's strictly-lower entry count; *bad_row = the smallest row whose columns do not ascend
__global__ void k_branch_count(int n, const int* __restrict__ rowptr, const int* __restrict__ colidx,
                               int* __restrict__ cnt, int* bad_row) {
  for (int row = blockIdx.x * blockDim.x + threadIdx.x; row < n; row += gridDim.x * blockDim.x) {
    int low = 0;
    for (int j = rowptr[row]; j < rowptr[row + 1]; ++j) {
      const int col = colidx[j];
      if (j > rowptr[row] && col <= colidx[j - 1]) atomicMin(bad_row, row);
      low += col < row;
    }
    cnt[row] = low;
  }
}

// the 0-based endpoints of every branch
__global__ void k_branch_ends(int n, const int* __restrict__ rowptr, const int* __restrict__ colidx,
                              const int* __restrict__ bptr, long long* __restrict__ lo, long long* __restrict__ hi) {
  for (int row = blockIdx.x * blockDim.x + threadIdx.x; row < n; row += gridDim.x * blockDim.x)
    for (int e = bptr[row], j = rowptr[row]; e < bptr[row + 1]; ++e, ++j) {
      lo[e] = colidx[j];
      hi[e] = row;
    }
}

// Branch currents of the panel V (n_pad x KT, row-major), with the maxima maxpos that k_cur_max left in
// ctl for the same panel: b = |a_{hi,lo}| (v_lo - v_hi), zeroed when |b / maxpos| < 1e-8 -- the test is
// written as in k_cur_acc, so a NaN keeps its value as in the reference -- and output as |b|.
// out: column-major nb x KT (leading dimension ld), or null.  cum: cum[e] += sum_c w_c |b_c| in fp64 in
// column order over the columns c < ncols with w_c != 0, or null; never log-transformed (out.jl:62-84).
// One thread walks one row's branches for every column, so each branch's sum has a single owner.
template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_branch_cur(int n, const int* __restrict__ rowptr, const int* __restrict__ colidx, const T* __restrict__ vals,
             const int* __restrict__ bptr, const T* __restrict__ V, const PanelCtl* ctl, T* __restrict__ out,
             size_t ld, T* __restrict__ cum, int ncols) {
  T maxpos[KT];
#pragma unroll
  for (int c = 0; c < KT; ++c) maxpos[c] = (T)ctl->maxpos[c];
  for (int row = blockIdx.x * NT + threadIdx.x; row < n; row += gridDim.x * NT) {
    const int e0 = bptr[row], e1 = bptr[row + 1];
    if (e0 == e1) continue;
    T vhi[KT];
#pragma unroll
    for (int c = 0; c < KT; ++c) vhi[c] = V[(size_t)row * KT + c];
    for (int e = e0, j = rowptr[row]; e < e1; ++e, ++j) {
      const int lo = colidx[j];
      const T a = fabs(vals[j]);
      double s = 0.0;
#pragma unroll
      for (int c = 0; c < KT; ++c) {
        const T d = a * (V[(size_t)lo * KT + c] - vhi[c]);
        const T b = !(fabs(d / maxpos[c]) < T(1e-8)) ? fabs(d) : T(0);
        if (out) out[(size_t)c * ld + e] = b;
        if (cum) {
          const double w = ctl->weight[c];
          if (c < ncols && w != 0.0) s += w * (double)b;
        }
      }
      if (cum) cum[e] = (T)((double)cum[e] + s);
    }
  }
}

// advanced mode on a network: vsum[row] += X[row, owner[row] - c0] for the rows the panel's columns own
template <typename T, int KT>
__global__ void k_owner_sum(int n, const T* __restrict__ X, const long long* __restrict__ owner, long long c0,
                            T* __restrict__ vsum) {
  for (int row = blockIdx.x * blockDim.x + threadIdx.x; row < n; row += gridDim.x * blockDim.x) {
    const long long c = owner[row] - c0;
    if (c >= 0 && c < KT) vsum[row] += X[(size_t)row * KT + c];
  }
}

__global__ void k_set_ctl(PanelCtl* ctl, double rtol, double atol, int itmax, int stall_limit) {
  ctl->stall_limit = stall_limit;
  ctl->rtol = rtol;
  ctl->atol = atol;
  ctl->itmax = itmax;
  ctl->init = 1;
  ctl->iter = 0;
}

__global__ void k_set_stall(PanelCtl* ctl, int stall_limit) { ctl->stall_limit = stall_limit; }

template <typename T>
__global__ void k_fill(T* p, size_t n, T v) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x)
    p[i] = v;
}

// L2 flush helper for benchmarks: touch a buffer larger than L2.
__global__ void k_flush(float* p, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (size_t)gridDim.x * blockDim.x)
    p[i] = p[i] * 1.0001f + 1.0f;
}

// ---------------------------------------------------------------------------
// focal-region pairs (cs_b200_solve_region_pairs).  A panel's Dirichlet sets are 2*KT row
// segments of `rows`: segment 2c is set_a of column c (0 V), segment 2c+1 its set_b (1 V);
// seg[] holds the 2*KT+1 offsets.  The segment kernels run one CTA per segment; the sets of
// one column are disjoint, so no two threads write the same element.  cs_b200_solve_grounded
// uses the same table with segment 2c = column c's ground set and segment 2c+1 empty.
// ---------------------------------------------------------------------------
// P[row][s/2] = v for the rows of every segment s (set_b_only = 0) or of the set_b segments only
template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_seg_set(T* __restrict__ P, const int* __restrict__ seg, const int* __restrict__ rows, int set_b_only, T v) {
  const int s = blockIdx.x;
  if (set_b_only && !(s & 1)) return;
  const int c = s >> 1;
  for (int e = seg[s] + threadIdx.x; e < seg[s + 1]; e += NT) P[(size_t)rows[e] * KT + c] = v;
}

// every row of a set takes its merged node's current.  The set is equipotential, so its internal
// edges carry nothing and each of its rows only sends (set_b, the highest voltage) or only receives
// (set_a, the lowest): the merged node's max(inflow, outflow) is the sum of the rows' currents.
// Fixed-order sum: strided per thread, then a shared-memory tree.
template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_seg_current(T* __restrict__ C, const int* __restrict__ seg, const int* __restrict__ rows) {
  __shared__ double s_sum[NT];
  const int s = blockIdx.x, c = s >> 1, tid = threadIdx.x;
  double a = 0.0;
  for (int e = seg[s] + tid; e < seg[s + 1]; e += NT) a += (double)C[(size_t)rows[e] * KT + c];
  s_sum[tid] = a;
  __syncthreads();
  for (int w = NT / 2; w > 0; w >>= 1) {
    if (tid < w) s_sum[tid] += s_sum[tid + w];
    __syncthreads();
  }
  const T tot = (T)s_sum[0];
  for (int e = seg[s] + tid; e < seg[s + 1]; e += NT) C[(size_t)rows[e] * KT + c] = tot;
}

// true-residual gate of a masked panel:  resid[c] = ||Y[:,c]||^2 , bnorm[c] = ||B[:,c]||^2
// (Y = B - A X with the set rows zeroed, B zero there already).  Only the first nvalid = n*KT elements
// count: the SpMM leaves the pad rows of Y as an earlier, wider panel wrote them.
template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_resnorm(size_t nelem, size_t nvalid, const T* __restrict__ Y, const T* __restrict__ B, PanelCtl* ctl,
          double* partials) {
  constexpr int VEC = Vec<T>::N;
  CSB_REDUCE_SMEM(2, KT)
  const size_t stride = (size_t)gridDim.x * NT * VEC;
  double acc[2][VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) acc[0][i] = acc[1][i] = 0.0;
  for (size_t e = ((size_t)blockIdx.x * NT + threadIdx.x) * VEC; e < nelem; e += stride) {
    T y[VEC], b[VEC];
    vload(Y + e, y);
    vload(B + e, b);
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      if (e + i >= nvalid) continue;
      acc[0][i] += (double)y[i] * (double)y[i];
      acc[1][i] += (double)b[i] * (double)b[i];
    }
  }
  if (grid_reduce<KT, VEC, 2, false>(acc, partials, &ctl->ticket, s_warp, s_tree, s_out)) {
    if (threadIdx.x < KT) {
      ctl->resid[threadIdx.x] = s_out[threadIdx.x];
      ctl->bnorm[threadIdx.x] = s_out[KT + threadIdx.x];
    }
  }
}

// flux into set_b of every column:  xdst[c] = u[:,c] . (A u)[:,c]  over the first nvalid = n*KT elements
template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_flux(size_t nelem, size_t nvalid, const T* __restrict__ U, const T* __restrict__ AU, PanelCtl* ctl,
       double* partials) {
  constexpr int VEC = Vec<T>::N;
  CSB_REDUCE_SMEM(1, KT)
  const size_t stride = (size_t)gridDim.x * NT * VEC;
  double acc[1][VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) acc[0][i] = 0.0;
  for (size_t e = ((size_t)blockIdx.x * NT + threadIdx.x) * VEC; e < nelem; e += stride) {
    T u[VEC], y[VEC];
    vload(U + e, u);
    vload(AU + e, y);
#pragma unroll
    for (int i = 0; i < VEC; ++i)
      if (e + i < nvalid) acc[0][i] += (double)u[i] * (double)y[i];
  }
  if (grid_reduce<KT, VEC, 1, false>(acc, partials, &ctl->ticket, s_warp, s_tree, s_out))
    if (threadIdx.x < KT) ctl->xdst[threadIdx.x] = s_out[threadIdx.x];
}

// X[:,c] /= flux[c]  (the reference's 1 A normalisation)
template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_scale_flux(size_t nelem, T* __restrict__ X, const PanelCtl* __restrict__ ctl) {
  for (size_t e = (size_t)blockIdx.x * NT + threadIdx.x; e < nelem; e += (size_t)gridDim.x * NT)
    X[e] = (T)((double)X[e] / ctl->xdst[e % KT]);
}

// cum += sum_c weight[c] f(C[:,c]) and max = max(max, f(C[:,c])) in column order, f = log10 when
// log_transform (out.jl:100-107, 305-309) -- the accumulation of k_cur_acc, run after the set fix-up
template <typename T, int KT>
__global__ void __launch_bounds__(NT)
k_cur_accum(int n, const T* __restrict__ C, const PanelCtl* __restrict__ ctl, T* __restrict__ cum,
            T* __restrict__ mx, int log_transform) {
  for (int row = blockIdx.x * NT + threadIdx.x; row < n; row += gridDim.x * NT) {
    double s = 0.0;
    T m = T(-1.0e30);
#pragma unroll
    for (int c = 0; c < KT; ++c) {
      const double w = ctl->weight[c];
      if (w == 0.0) continue;
      const T cur = C[(size_t)row * KT + c];
      const T val = log_transform ? (cur > T(0) ? (T)log10((double)cur) : T(-9999)) : cur;
      s += w * (double)val;
      m = val > m ? val : m;
    }
    cum[row] = (T)((double)cum[row] + s);
    if (mx) mx[row] = m > mx[row] ? m : mx[row];
  }
}


// ---------------------------------------------------------------------------
// connected components of an operator (cs_b200_components): union-find over the stored off-diagonal
// entries whose value is != 0 (a NaN is an edge), with integer atomics only.  A union always hangs the
// larger root under the smaller, so parent[v] <= v throughout and every root ends as its component's
// smallest row: the labels do not depend on the order in which the hooks race.
// ---------------------------------------------------------------------------
// the root of v, halving the path on the way up (a racing write only ever stores another ancestor of v)
__device__ __forceinline__ int cc_find(int* parent, int v) {
  int p = __ldcg(parent + v);
  while (p != v) {
    const int gp = __ldcg(parent + p);
    if (gp == p) return p;
    parent[v] = gp;
    v = gp;
    p = __ldcg(parent + v);
  }
  return v;
}

__global__ void k_cc_init(int n, int* __restrict__ parent) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) parent[v] = v;
}

// edge-parallel hooking: thread t takes the entries [t * chunk, (t + 1) * chunk), finds the first one's row
// by bisection of rowptr and walks on, so a row of thousands of entries (a merged polygon) is spread over
// many threads
template <typename T>
__global__ void k_cc_hook(int n, int nnz, const int* __restrict__ rowptr, const int* __restrict__ colidx,
                          const T* __restrict__ vals, int* parent, int chunk) {
  for (int64_t j0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * chunk; j0 < nnz;
       j0 += (int64_t)gridDim.x * blockDim.x * chunk) {
    int lo = 0, hi = n;                            // the last row with rowptr[row] <= j0
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (rowptr[mid] <= j0) lo = mid; else hi = mid;
    }
    int row = lo;
    const int j1 = (int)(j0 + chunk < nnz ? j0 + chunk : nnz);
    for (int j = (int)j0; j < j1; ++j) {
      while (rowptr[row + 1] <= j) ++row;
      const int col = colidx[j];
      if (col == row || !(vals[j] != T(0))) continue;
      int a = cc_find(parent, row), b = cc_find(parent, col);
      while (a != b) {
        if (a > b) { const int t = a; a = b; b = t; }
        const int was = atomicCAS(parent + b, b, a);   // hang the larger root under the smaller
        if (was == b) break;
        b = cc_find(parent, was);                      // b was hooked meanwhile: retry from its new root
        a = cc_find(parent, a);
      }
    }
  }
}

// rootof[v] = the root of v, flag[v] = 1 for the roots (what the label scan numbers).  The roots go to their own
// array: a racing path-halving write may still store a non-root ancestor into parent[v] after v's own thread
// has stored the root there
__global__ void k_cc_compress(int n, int* parent, int* __restrict__ rootof, int* __restrict__ flag) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    const int r = cc_find(parent, v);
    rootof[v] = r;
    flag[v] = r == v;
  }
}

// lab[v] = number of roots below v's root, in place over rootof (idx = the exclusive scan of the root flags)
__global__ void k_cc_label(int n, int* __restrict__ lab, const int* __restrict__ idx) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) lab[v] = idx[lab[v]];
}

// ---------------------------------------------------------------------------
// raster advanced mode's column plan (cs_b200_plan_advanced): node values summed in np.add.at's order, the
// conflict policy, component sums and the columns, with integer atomics only
// ---------------------------------------------------------------------------
// key[i] = the 0-based node of row-major cell i = r * ncols + c (n: no node), val[i] = i; cnt[v] counts node v's
// cells; *bad |= 1 for a node map entry outside [0, n]
__global__ void k_adv_cells(int ncell, int nrows, int ncols, int n, const int* __restrict__ nodemap,
                            unsigned* __restrict__ key, int* __restrict__ val, int* __restrict__ cnt, int* bad) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ncell; i += gridDim.x * blockDim.x) {
    const int r = i / ncols, c = i - r * ncols;
    const int v = nodemap[(int64_t)c * nrows + r];
    unsigned k = (unsigned)n;
    if (v < 0 || v > n) atomicOr(bad, 1);
    else if (v > 0) { k = (unsigned)(v - 1); atomicAdd(cnt + k, 1); }
    key[i] = k;
    val[i] = i;
  }
}

// key[r] = lab[r], val[r] = r, cnt[lab[r]] counts each component's rows
__global__ void k_adv_rows(int n, const int* __restrict__ lab, unsigned* __restrict__ key, int* __restrict__ val,
                           int* __restrict__ cnt) {
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
    key[r] = (unsigned)lab[r];
    val[r] = r;
    atomicAdd(cnt + lab[r], 1);
  }
}

// One thread per node: its cells (ptr / cell: row-major indices grouped by node, ascending) summed in that order
// from +0.0, zeros skipped, as np.add.at adds the selected cells; f = the finite part of the summed grounds
// (before the policy, as resolve_conflicts takes it); then the policy and the Inf-ground rule.  flags[0] |= 2 for
// a node without a cell, flags[1] = 1 when some f != 0.
template <typename M, typename T>
__global__ void k_adv_node_values(int n, int nrows, int ncols, const int* __restrict__ ptr,
                                  const int* __restrict__ cell, const M* __restrict__ src,
                                  const M* __restrict__ gnd, int policy, double* __restrict__ s_out,
                                  double* __restrict__ g_out, T* __restrict__ f_out, int* flags) {
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    const int b = ptr[v], e = ptr[v + 1];
    if (b == e) atomicOr(flags, 2);
    double s = 0.0, g = 0.0;
    for (int j = b; j < e; ++j) {
      const int i = cell[j], r = i / ncols;
      const int64_t x = (int64_t)(i - r * ncols) * nrows + r;     // column-major cell
      const double a = (double)src[x], q = (double)gnd[x];
      if (a != 0.0) s += a;
      if (q != 0.0) g += q;
    }
    const double f = isfinite(g) ? g : 0.0;
    f_out[v] = (T)f;
    if (f != 0.0) atomicOr(flags + 1, 1);
    const bool both = s != 0.0 && g != 0.0;
    if (both && (policy == 1 || policy == 3)) s = 0.0;          // rmvsrc, rmvall (sources only)
    else if (both && policy == 2) g = 0.0;                      // rmvgnd
    if (isinf(g) && s > 0.0) g = 0.0;
    s_out[v] = s;
    g_out[v] = g;
  }
}

// Per sorted position j (rows: each component's rows ascending, lab: their labels): each component's counts of
// nonzero source and ground terms, Inf-ground rows and source rows (s != 0, g != Inf), with integer atomics, and
// the flags that select the nonzero terms of the two sums.
__global__ void k_adv_counts(int n, const int* __restrict__ rows, const unsigned* __restrict__ lab,
                             const double* __restrict__ s, const double* __restrict__ g, int* __restrict__ nzs,
                             int* __restrict__ nzg, int* __restrict__ ninf, int* __restrict__ nsrc,
                             unsigned char* __restrict__ fs, unsigned char* __restrict__ fg) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    const int r = rows[j], c = (int)lab[j];
    const double sv = s[r], gv = g[r];
    const bool inf = gv == __longlong_as_double(0x7ff0000000000000LL);
    fs[j] = sv != 0.0;
    fg[j] = gv != 0.0;
    if (sv != 0.0) atomicAdd(nzs + c, 1);
    if (gv != 0.0) atomicAdd(nzg + c, 1);
    if (inf) atomicAdd(ninf + c, 1);
    if (sv != 0.0 && !inf) atomicAdd(nsrc + c, 1);
  }
}

constexpr int ADV_SUM_THREADS = 64;
constexpr int ADV_SUM_DEPTH = 32;   // frames of the pairwise recursion: ranges of <= 2^30 terms need <= 24

// numpy's pairwise_sum (umath/loops_utils.h: fewer than 8 terms added in order from 0; up to 128 terms in 8 strided
// accumulators r0..r7 combined as ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then the remaining n % 8 in
// order; longer ranges split at n / 2 rounded down to a multiple of 8, left + right) over the n terms of one
// component, of which only the nz nonzero ones are given: positions j = pos[0..nz) ascending (base: the
// component's first position), values x[rows[j]].  A +0.0 term leaves every partial sum as it is, so leaving the
// zeros out, and skipping subtrees without a nonzero term, gives the same bits.  The recursion's frames are the
// thread's column of shared memory.
__device__ double adv_pairwise(int n, int base, const int* __restrict__ pos, int nz, const int* __restrict__ rows,
                               const double* __restrict__ x, int* f_lo, int* f_len, double* f_left) {
  const int t = threadIdx.x;
  int k = 0, sp = 0, lo = 0, len = n;
  unsigned right = 0;                                      // bit d: frame d's left half is done
  for (;;) {
    double v = 0.0;
    if (k >= nz || pos[k] - base >= lo + len || len <= 128) {
      if (k < nz && pos[k] - base < lo + len) {            // a leaf with nonzero terms
        const int m = len < 8 ? 0 : len - (len & 7);
        double r0 = 0.0, r1 = 0.0, r2 = 0.0, r3 = 0.0, r4 = 0.0, r5 = 0.0, r6 = 0.0, r7 = 0.0;
        for (; k < nz && pos[k] - base < lo + m; ++k) {
          const double a = x[rows[pos[k]]];
          switch ((pos[k] - base - lo) & 7) {
            case 0: r0 += a; break;
            case 1: r1 += a; break;
            case 2: r2 += a; break;
            case 3: r3 += a; break;
            case 4: r4 += a; break;
            case 5: r5 += a; break;
            case 6: r6 += a; break;
            default: r7 += a; break;
          }
        }
        v = ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7));
        for (; k < nz && pos[k] - base < lo + len; ++k) v += x[rows[pos[k]]];
      }
      for (;;) {                                           // hand v up to the frames above
        if (sp == 0) return v;
        const int d = sp - 1, idx = d * ADV_SUM_THREADS + t;
        if (!((right >> d) & 1u)) {
          f_left[idx] = v;
          right |= 1u << d;
          int h = f_len[idx] / 2;
          h -= h % 8;
          lo = f_lo[idx] + h;
          len = f_len[idx] - h;
          break;
        }
        v = f_left[idx] + v;
        right &= ~(1u << d);
        --sp;
      }
    } else {                                               // split: descend into the left half
      const int idx = sp * ADV_SUM_THREADS + t;
      f_lo[idx] = lo;
      f_len[idx] = len;
      right &= ~(1u << sp);
      ++sp;
      len = len / 2;
      len -= len % 8;
    }
  }
}

// One thread per component: its source and ground sums by adv_pairwise over the compacted nonzero terms
// (zs_pos / zg_pos, CSR zs_ptr / zg_ptr), solved = both != 0 (NaN counts); a solved component with a source row off
// the Inf grounds is a column.  Per component: solved, column, and for a column its Inf-ground and source row
// counts (0 otherwise).
__global__ void __launch_bounds__(ADV_SUM_THREADS)
k_adv_sums(int ncomp, const int* __restrict__ cptr, const int* __restrict__ rows, const double* __restrict__ s,
           const double* __restrict__ g, const int* __restrict__ zs_ptr, const int* __restrict__ zs_pos,
           const int* __restrict__ zg_ptr, const int* __restrict__ zg_pos, const int* __restrict__ ninf,
           const int* __restrict__ nsrc, long long* __restrict__ solved, long long* __restrict__ iscol,
           long long* __restrict__ nset, long long* __restrict__ nsrc_col) {
  __shared__ int f_lo[ADV_SUM_DEPTH * ADV_SUM_THREADS], f_len[ADV_SUM_DEPTH * ADV_SUM_THREADS];
  __shared__ double f_left[ADV_SUM_DEPTH * ADV_SUM_THREADS];
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < ncomp; c += gridDim.x * blockDim.x) {
    const int base = cptr[c], n = cptr[c + 1] - base;
    const double ss = adv_pairwise(n, base, zs_pos + zs_ptr[c], zs_ptr[c + 1] - zs_ptr[c], rows, s, f_lo, f_len, f_left);
    const double gs = adv_pairwise(n, base, zg_pos + zg_ptr[c], zg_ptr[c + 1] - zg_ptr[c], rows, g, f_lo, f_len, f_left);
    const bool sol = ss != 0.0 && gs != 0.0, col = sol && nsrc[c] > 0;
    solved[c] = sol;
    iscol[c] = col;
    nset[c] = col ? ninf[c] : 0;
    nsrc_col[c] = col ? nsrc[c] : 0;
  }
}

// One thread per column component: its label and the ends of its set and source row ranges (colx / setx / srcx:
// the exclusive scans of iscol / nset / nsrc; set_ptr[0] and src_ptr[0] are written by the caller).
__global__ void k_adv_ptrs(int ncomp, const long long* __restrict__ iscol, const long long* __restrict__ colx,
                           const long long* __restrict__ setx, const long long* __restrict__ nset,
                           const long long* __restrict__ srcx, const long long* __restrict__ nsrc,
                           long long* __restrict__ col_comp, long long* __restrict__ set_ptr,
                           long long* __restrict__ src_ptr) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < ncomp; c += gridDim.x * blockDim.x) {
    if (!iscol[c]) continue;
    const long long col = colx[c];
    col_comp[col] = c;
    set_ptr[col + 1] = setx[c] + nset[c];
    src_ptr[col + 1] = srcx[c] + nsrc[c];
  }
}

// Per sorted position j: col_of_row of the rows of column components, and the flags that select each column's
// Inf-ground rows and source rows (in position order: columns in label order, rows ascending).
__global__ void k_adv_mark(int n, const int* __restrict__ rows, const unsigned* __restrict__ lab,
                           const double* __restrict__ s, const double* __restrict__ g,
                           const long long* __restrict__ iscol, const long long* __restrict__ colx,
                           int* __restrict__ col_of_row, unsigned char* __restrict__ fset,
                           unsigned char* __restrict__ fsrc) {
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
    const int r = rows[j], c = (int)lab[j];
    const bool col = iscol[c] != 0;
    const bool inf = g[r] == __longlong_as_double(0x7ff0000000000000LL);
    if (col) col_of_row[r] = (int)colx[c];
    fset[j] = col && inf;
    fsrc[j] = col && s[r] != 0.0 && !inf;
  }
}

// The selected set rows and source rows (int32, in order) into the plan: int64 rows and the sources' node values.
__global__ void k_adv_widen(int nset, const int* __restrict__ sel_set, int nsrc, const int* __restrict__ sel_src,
                            const double* __restrict__ s, long long* __restrict__ set_rows,
                            long long* __restrict__ src_rows, double* __restrict__ src_vals) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nset + nsrc; i += gridDim.x * blockDim.x) {
    if (i < nset) {
      set_rows[i] = sel_set[i];
    } else {
      const int r = sel_src[i - nset];
      src_rows[i - nset] = r;
      src_vals[i - nset] = s[r];
    }
  }
}

}  // namespace csb

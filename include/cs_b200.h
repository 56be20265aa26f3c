/*
 * cs_b200.h -- C ABI of libcsb200.so: an H100-native (sm_90a) replacement for the
 * inner Laplacian-solve loop of Circuitscape.jl (pairwise + advanced mode).
 *
 * This is the drop-in boundary.  The reference (Julia) reaches a solver through
 * three methods that package extensions overload (ext/CircuitscapePardisoExt.jl:31-45,
 * ext/CircuitscapeAppleAccelerateExt.jl:8-22):
 *
 *   construct_cholesky_factor(matrix, solver)          src/core.jl:379,519-523
 *        -> cs_b200_create            (once per connected component)
 *   solve_linear_system(factor, matrix, rhs::Matrix)   src/core.jl:463,646-653
 *        -> cs_b200_solve_rhs         (n x k column-major in, n x k out, true
 *                                      residual gate 1e-4 reported per column)
 *   multiple_solve(solver, matrix, sources::Vector)    src/raster/advanced.jl:307-333
 *        -> cs_b200_create + cs_b200_solve_rhs(k = 1)
 *
 * and the batched driver around them (src/core.jl:312-515: RHS  -1 at src, +1 at
 * dst; shift so v[src] = 0; R = v[dst] - v[src]; per-pair node currents
 * src/out.jl:178-290 accumulated into cumulative / max maps src/out.jl:100-107)
 * is offered as ONE device-resident call so n x k voltages never cross PCIe:
 *
 *        -> cs_b200_solve_pairs / cs_b200_solve_sources  + cs_b200_read_currents
 *
 * All entry points use plain pointers and sizes; every function returns 0 on
 * success or a negative cs_b200_status; cs_b200_last_error() gives the text.
 * Host buffers are copied during the call (the caller keeps ownership; Julia:
 * GC.@preserve).  A handle is NOT re-entrant: one in-flight call per handle.
 * INTEGRATION.md shows the Julia `ccall` glue that binds these symbols.
 */
#ifndef CS_B200_H
#define CS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct cs_b200_handle cs_b200_handle;

enum cs_b200_status {
  CS_B200_OK = 0,
  CS_B200_ERR_ARG = -1,        /* bad argument                                    */
  CS_B200_ERR_CUDA = -2,       /* CUDA runtime error (no GPU, OOM, launch failure) */
  CS_B200_ERR_RESIDUAL = -3,   /* a column failed the true-residual gate (1e-4), the
                                  reference's `error("... exceeds tolerance 1e-4")`,
                                  src/core.jl:641,650                              */
  CS_B200_ERR_MAXITER = -4,    /* itmax reached, or a column's recurrence stagnated (reduced-precision
                                  storage), before rtol: results still written, relres[] says how far */
  CS_B200_ERR_UNSUPPORTED = -5
};

enum cs_b200_dtype { CS_B200_F32 = 0, CS_B200_F64 = 1 };

enum cs_b200_precond {
  CS_B200_PRECOND_JACOBI = 0,  /* D^-1, built on device                            */
  CS_B200_PRECOND_AMG = 1      /* aggregation multigrid V-cycle, Jacobi-smoothed
                                  (the reference's AMG role, src/core.jl:164-167)  */
};

/* Options; zero-initialise then override.  0 means "library default".             */
typedef struct cs_b200_opts {
  int32_t precond;        /* cs_b200_precond                                       */
  int32_t panel_width;    /* RHS columns solved together per panel: 1,2,4,8 (def 8) */
  int32_t check_every;    /* CG iterations between host convergence polls (def 16)  */
  int32_t use_graph;      /* 0/1: whole PCG loop as a device-side WHILE graph (def);
                             2: host-polled graph chunks of check_every iterations;
                             -1: plain launches                                       */
  double atol;            /* absolute term of the stop test; 0 => sqrt(eps(Float64)), the
                             Krylov.jl default in force at src/core.jl:639; <0 => none */
  double resid_gate;      /* true-residual gate (def 1e-4, src/core.jl:641)         */
  int32_t log_transform;  /* current maps accumulate log10(c) (src/out.jl:305-309)  */
  int32_t window;         /* TMA-staged windowed SpMM: 0 auto (operators >= 20000 rows),
                             1 always, -1 never (plain direct-gather kernel)         */
  int32_t mixed;          /* fp64 handles with AMG: run the V-cycle in fp32 (CG vectors,
                             dot products and the residual gate stay fp64): 0 auto (on),
                             -1 off                                                  */
  int32_t setup;          /* where the multigrid hierarchy and the windowed records are built:
                             0 auto (on the device), 1 on the host (amg_host.hpp / win_host.hpp,
                             the round-1 path, kept for A/B checks), 2 on the device           */
  int32_t stencil;        /* stencil (DIA) SpMM for operators whose entries all sit on the 9 raster
                             diagonals (full rasters, regular coarse grids): 0 auto (operators
                             >= 20000 rows), 1 always, -1 never                                */
  int32_t reserved[3];
} cs_b200_opts;

/* Per-call statistics (milliseconds measured with CUDA events on the solve stream). */
typedef struct cs_b200_stats {
  double setup_ms;        /* create: upload + preconditioner build                  */
  double solve_ms;        /* last solve_*: device time incl. H2D/D2H inside the call */
  double kernel_ms;       /* last solve_*: iteration kernels only                   */
  int64_t iterations;     /* last solve_*: sum over columns                         */
  int64_t spmm_launches;  /* last solve_*: SpMM kernel launches                     */
  int64_t kernel_launches;/* last solve_*: all kernel launches                      */
  double h2d_bytes, d2h_bytes;
} cs_b200_stats;

/* Build the device-resident operator for one connected component.
 * CSR of a symmetric matrix (so Julia's SparseMatrixCSC colptr/rowval/nzval can be
 * passed as-is).  index_bits in {32,64}: width of rowptr/colidx entries;
 * index_base in {0,1}; dtype: type of `vals`, of all RHS/solution buffers and of the
 * device arithmetic.  device: CUDA ordinal.  opts may be NULL.                      */
int cs_b200_create(int64_t n, int64_t nnz, const void* rowptr, const void* colidx,
                   const void* vals, int index_bits, int index_base, int dtype,
                   int device, const cs_b200_opts* opts, cs_b200_handle** out);

/* Same, but rowptr/colidx/vals already live on `device` (int32 0-based indices,
 * values of `dtype`).  Used after an NCCL broadcast of the matrix to peer GPUs.    */
int cs_b200_create_from_device(int64_t n, int64_t nnz, const int32_t* d_rowptr,
                               const int32_t* d_colidx, const void* d_vals, int dtype,
                               int device, const cs_b200_opts* opts, cs_b200_handle** out);

/* The step BEFORE the path (SURVEY.md 8f rank 2): assemble the Laplacian of a conductance raster
 * on the device and build the handle on it -- construct_node_map without polygons
 * (src/raster/pairwise.jl:271-281), construct_graph (src/raster/pairwise.jl:317-367) and
 * laplacian! (src/core.jl:608-624) as three kernels around two prefix sums; nothing of size nnz
 * is built on the host or crosses PCIe on the way in.
 * g: host, COLUMN-major nrows x ncols (a Julia Matrix as it lies in memory), element type `dtype`;
 * cells with g <= 0 (0, NODATA -9999, NaN) are not nodes.  Nodes are numbered 0.. in memory
 * order over the valid cells -- the reference's numbering minus one.  avg_res / four_neighbors:
 * connect_using_avg_resistances / connect_four_neighbors_only.  The whole raster becomes ONE
 * operator (block diagonal over its connected components; a solve's sources and ground must
 * lie in one component, as they do in the reference's per-component calls).
 * *n_out / *nnz_out (optional): nodes and stored entries of the assembled matrix.            */
int cs_b200_create_from_raster(int64_t nrows, int64_t ncols, const void* g, int dtype,
                               int four_neighbors, int avg_res, int device,
                               const cs_b200_opts* opts, cs_b200_handle** out,
                               int64_t* n_out, int64_t* nnz_out);

/* Same with SHORT-CIRCUIT POLYGONS (construct_node_map with a polygon map, src/raster/pairwise.jl:283-314):
 * polymap: host, column-major nrows x ncols int32, 0 = no polygon (NULL = none).  Every cell of a polygon,
 * NODATA cells included, takes the node of the polygon's first valid cell; node labels are compacted in
 * order; parallel cell adjacencies between merged nodes add up and adjacencies inside a node vanish
 * (sparse(I,J,V) + laplacian!, src/core.jl:608-624).  nodemap_out (optional): host, column-major
 * nrows x ncols int32, the node id of every cell (1-based like the reference's nodemap, 0 = none) --
 * what the host needs to place focal points, sources and grounds.                                   */
int cs_b200_create_from_raster_poly(int64_t nrows, int64_t ncols, const void* g, const int32_t* polymap,
                                    int dtype, int four_neighbors, int avg_res, int device,
                                    const cs_b200_opts* opts, cs_b200_handle** out, int64_t* n_out,
                                    int64_t* nnz_out, int32_t* nodemap_out);

/* Copy the handle's CSR (0-based, int32 indices, values of the handle's dtype) to host buffers
 * of n+1, nnz and nnz elements; any pointer may be NULL.  Parity / debugging hook.            */
int cs_b200_get_csr(cs_b200_handle* h, int32_t* rowptr, int32_t* colidx, void* vals);

/* Advanced mode on a RESIDENT operator (src/raster/advanced.jl:274-305): the reference rebuilds
 * `G + diag(finite grounds)` with the rows / columns of the Inf grounds deleted for every solve; here
 * the handle keeps the component's Laplacian and this call re-derives the operator on the device:
 *     finite_g  (n values of the handle's dtype, or NULL)   added to the diagonal
 *     dirichlet (n bytes, non-zero = tied to ground, or NULL) row and column replaced by the identity
 *                                                           row -- the deleted row with its 0 V kept in place
 * then 1/diag, the stencil / window records and the multigrid hierarchy are rebuilt from the device-
 * resident CSR (no matrix crosses PCIe; ~0.1 s at 10^6 nodes).  Right-hand sides passed afterwards must
 * be zero at the Dirichlet rows (the reference drops those sources).  Calling it again starts from the
 * pristine values; NULL, NULL restores the original operator.  Needs the device-side setup and a
 * handle that owns its matrix.  The handle keeps finite_g until the next call or cs_b200_destroy: the
 * node currents of cs_b200_solve_advanced add the finite-ground currents from it.                  */
int cs_b200_set_grounds(cs_b200_handle* h, const void* finite_g, const uint8_t* dirichlet);

/* Multigrid hierarchy inspection (parity / debugging hooks; levels exist only with the AMG
 * preconditioner).  which: 0 = operator A_l, 1 = prolongator P_l (level l <- l+1), 2 = restriction
 * R_l = P_l^T.  level_info returns CS_B200_ERR_ARG past the last level (and for P / R on the
 * coarsest); omega = Jacobi damping of the level.  level_csr copies the operator as 0-based CSR
 * with fp64 values (converted when the cycle runs in fp32); any pointer may be NULL.            */
int cs_b200_level_info(cs_b200_handle* h, int level, int which, int64_t* nrows, int64_t* ncols,
                       int64_t* nnz, double* omega, int* windowed);
int cs_b200_level_csr(cs_b200_handle* h, int level, int which, int32_t* rowptr, int32_t* colidx,
                      double* vals);
/* Diagonals stored for the stencil form of operator A_l: 0 (no stencil form), 9, or 5 when the operator is
 * bitwise symmetric and kept as its upper diagonals only (CS_B200_FULL_STENCIL in the environment keeps 9). */
int cs_b200_level_stencil(cs_b200_handle* h, int level, int* slots);

/* n and nnz of the handle's operator. */
int cs_b200_get_dims(const cs_b200_handle* h, int64_t* n, int64_t* nnz);

void cs_b200_destroy(cs_b200_handle* h);

/* Text of the last error on this handle (or of the last failed create if h==NULL). */
const char* cs_b200_last_error(const cs_b200_handle* h);

/* y = A x, `reps` times back to back; *ms_per_rep = mean device time of one SpMV
 * (CUDA events).  x, y: host vectors of n values of the handle's dtype.  Benchmark
 * and parity hook for the headline kernel.                                          */
int cs_b200_spmv(cs_b200_handle* h, const void* x, void* y, int reps, double* ms_per_rep);

/* Y = A X for k in {1,2,4,8} columns through the panel SpMM kernel: x, y host,
 * column-major n x k.  Parity hook for the batched kernel at any size.             */
int cs_b200_spmm(cs_b200_handle* h, int k, const void* x, void* y);

/* Z = M^-1 R for k in {1,2,4,8} columns through ONE application of the multigrid preconditioner --
 * the V-cycle the solver launches for its first z (in fp32 when the cycle is mixed).  r, z: host,
 * column-major n x k of the handle's dtype.  rz (k values, may be NULL): |r.z| per column as the
 * cycle's last kernel reduces it.  CS_B200_ERR_UNSUPPORTED without a hierarchy.  Parity hook.   */
int cs_b200_apply_precond(cs_b200_handle* h, int k, const void* r, void* z, double* rz);

/* Y = A X for a row-major n x k panel resident on the device (k in 1,2,4,8),
 * timing only -- no host traffic.  flush_l2 != 0 writes a >L2 buffer between reps. */
int cs_b200_bench_spmm(cs_b200_handle* h, int k, int reps, int flush_l2, double* ms_per_rep);

/* One fused PCG iteration (SpMM+dot, residual update+dot, direction update) on a
 * device-resident panel of width k, `reps` times; timing only.                      */
int cs_b200_bench_cg_iter(cs_b200_handle* h, int k, int reps, double* ms_per_rep);

/* solve_linear_system(factor, matrix, rhs): A X = B for k right-hand sides.
 * rhs, lhs: host, column-major n x k (Julia Matrix / Vector when k = 1).
 * iters[k], relres[k] (true relative residual ||A x - b|| / ||b||) may be NULL.
 * Returns CS_B200_ERR_RESIDUAL if any column fails the gate (lhs still written).    */
int cs_b200_solve_rhs(cs_b200_handle* h, int64_t k, const void* rhs, void* lhs,
                      double rtol, int64_t itmax, int64_t* iters, double* relres);

/* Batched focal-pair solve, device-resident:
 *   for c in 0..k-1:  A v = e_dst[c] - e_src[c];  v -= v[src[c]];  R[c] = v[dst[c]]
 * src/dst: 0-based rows of this component.  R: k values of dtype.
 * volt: NULL or host column-major n x k (shifted voltages).
 * If accumulate != 0 the node-current vector of every pair (src/out.jl:178-207:
 * max(inflow, outflow) per node with the 1e-8 relative zeroing of src/out.jl:281-287)
 * is added weight[c] times into the handle's cumulative vector and max-ed into its
 * max vector (src/out.jl:100-107); weight == NULL means 1 each.
 * curr: NULL or host column-major n x k of the per-pair node currents.              */
int cs_b200_solve_pairs(cs_b200_handle* h, int64_t k, const int64_t* src, const int64_t* dst,
                        const double* weight, double rtol, int64_t itmax, void* R,
                        void* volt, void* curr, int accumulate, int64_t* iters,
                        double* relres);

/* Branches of the handle's operator (network mode): its stored strictly-lower CSR entries (hi, lo < hi),
 * ordered by hi, then lo -- for a symmetric operator the order in which the reference writes branch
 * currents (src/out.jl:128-148, 250-278).  Built on the device on first use and kept until cs_b200_destroy;
 * a row whose column indices do not ascend is CS_B200_ERR_ARG (the row in cs_b200_last_error).  Returns nb
 * and, for non-NULL lo / hi, the nb 0-based endpoints of every branch.                                   */
int cs_b200_branch_index(cs_b200_handle* h, int64_t* nb, int64_t* lo, int64_t* hi);

/* Connected components of the handle's operator, labelled on the device: an edge is a stored off-diagonal
 * entry whose value is != 0 (a NaN counts, stored zeros and the diagonal do not) -- what
 * eliminate_zeros() + csgraph.connected_components(directed=False) sees.  After cs_b200_set_grounds the
 * pristine values are used, so identity rows do not split components.  Returns ncomp and, for non-NULL
 * comp_of (n int32 on the host), each row's component, numbered in order of each component's smallest row
 * (SciPy's labels exactly).  Union-find with integer atomics: the output does not depend on the order of the
 * races.  Scratch comes from the stream-ordered pool and is released before return.                      */
int cs_b200_components(cs_b200_handle* h, int64_t* ncomp, int32_t* comp_of);

/* Raster advanced mode's columns on a whole-raster handle (src/raster/advanced.jl:81-196), planned on the device.
 * nodemap: the nrows x ncols column-major 1-based node map cs_b200_create_from_raster[_poly] returned for this
 * handle; src / gnd: the advanced-mode maps, column-major, of dtype (CS_B200_F32 / F64): source currents per cell,
 * ground conductances with Inf for a direct ground; policy 0 keepall, 1 rmvsrc, 2 rmvgnd, 3 rmvall.
 *   - node values: each node's nonzero cell values summed in fp64 from +0.0 in row-major cell order (np.add.at's
 *     order), for sources and grounds alike;
 *   - f = isfinite(g) ? g : 0 of those grounds; then the policy (rmvsrc / rmvall zero the sources, rmvgnd the
 *     grounds, where both are nonzero) and every Inf ground under a source > 0 zeroed;
 *   - if some f != 0 the handle takes cs_b200_set_grounds(f, NULL) through the same code (*finite_applied = 1);
 *     otherwise it is untouched (0);
 *   - components: the labels of cs_b200_components; a component is solved iff its source sum and its ground sum
 *     over its rows in ascending order are both != 0 (NaN counts), each sum numpy's pairwise summation of those
 *     n terms (blocks of <= 128 in 8 strided accumulators, halves split at a multiple of 8), the `s[rows].sum()`
 *     of core.raster_advanced bit for bit; *nsolved counts them;
 *   - a solved component with a row where s != 0 and g != Inf is a column, in label order.
 * Returns the column count and the total set / source rows; the plan stays on the device until
 * cs_b200_read_advanced_plan, the next plan or cs_b200_destroy.  CS_B200_ERR_ARG before the handle changes for a
 * NULL pointer, a bad dtype or policy, more than 2^30 cells, a node map entry outside [0, n] or a node without a
 * cell; CS_B200_ERR_UNSUPPORTED, also before any change and with no plan kept, when finite grounds would apply
 * to a handle cs_b200_set_grounds refuses.  Integer atomics only: the outputs repeat bit for bit.              */
int cs_b200_plan_advanced(cs_b200_handle* h, int64_t nrows, int64_t ncols, const int32_t* nodemap,
                          const void* src, const void* gnd, int dtype, int policy,
                          int64_t* ncol, int64_t* nsolved, int64_t* nset_rows, int64_t* nsrc_rows,
                          int* finite_applied);
/* Copies the plan of cs_b200_plan_advanced to host buffers and frees it: col_comp (ncol) each column's component
 * label; set_ptr (ncol + 1) / set_rows (nset_rows) each column's Inf-ground rows, ascending; src_ptr (ncol + 1) /
 * src_rows / src_vals (nsrc_rows) its rows with s != 0 and g != Inf, ascending, with their node source values;
 * col_of_row (n int32) the column of every row, or -1.  CS_B200_ERR_ARG without a plan.                       */
int cs_b200_read_advanced_plan(cs_b200_handle* h, int64_t* col_comp, int64_t* set_ptr, int64_t* set_rows,
                               int64_t* src_ptr, int64_t* src_rows, double* src_vals, int32_t* col_of_row);

/* cs_b200_solve_pairs with branch currents (network pairwise, src/out.jl:150-158, 250-290): arguments and
 * outputs as cs_b200_solve_pairs, plus branch: NULL or host column-major nb x k of the per-pair branch
 * currents |b|, b = |a_{hi,lo}| (v_lo - v_hi) zeroed where |b / max_e b| < 1e-8 (the maximum over the
 * column's branches, as the node currents use it).  With accumulate, each column's branch currents are
 * also added weight[c] times into the handle's cumulative branch vector (cs_b200_read_branch_currents;
 * summed in fp64 in column order, no log transform).  The other entry points never touch that vector.   */
int cs_b200_solve_pairs_branch(cs_b200_handle* h, int64_t k, const int64_t* src, const int64_t* dst,
                               const double* weight, double rtol, int64_t itmax, void* R, void* volt,
                               void* curr, int accumulate, int64_t* iters, double* relres, void* branch);

/* Pairwise driver by SUPERPOSITION -- the reference's Shortcut (src/core.jl:685-739), extended
 * to voltage / current maps.  All pairs among `np` focal nodes of ONE connected component share
 * the operator and are linear in the right-hand side, so np-1 solves
 *     A u_x = e_{nodes[x]} - e_{nodes[0]} ,  u_x -= u_x[nodes[0]]        (x = 1 .. np-1, u_0 = 0)
 * give every pair:  v(i,j) = u_j - u_i , shifted so that v[src] = 0 , R = v[dst].
 * pi / pj: the k pairs as indices into `nodes` (src = nodes[pi[c]], dst = nodes[pj[c]]).
 * R, volt, curr, accumulate, weight: exactly as cs_b200_solve_pairs.  Each combined voltage is
 * put through the true-residual gate against its own right-hand side (relres[k]); point_iters
 * (np-1 values, may be NULL) are the iterations of the point solves.  Needs np-1 device vectors.  */
int cs_b200_solve_pairs_superposed(cs_b200_handle* h, int64_t np, const int64_t* nodes, int64_t k,
                                   const int64_t* pi, const int64_t* pj, const double* weight,
                                   double rtol, int64_t itmax, void* R, void* volt, void* curr,
                                   int accumulate, int64_t* point_iters, double* relres);

/* Pairwise mode with focal regions (src/raster/pairwise.jl:72-135) on ONE resident operator: column c holds
 * set_a[c] at 0 V and set_b[c] at 1 V (Dirichlet), solves the interior, R[c] = 1 / flux into set_b[c],
 * voltages scaled to the reference's 1 A normalisation (0 on set_a, R on set_b).  Sets: CSR over 0-based rows
 * (set_ptr[nsets+1], set_rows), each non-empty, sorted, unique; the two sets of a column disjoint.
 * weight / volt / curr / accumulate / iters / relres as cs_b200_solve_pairs; curr and the accumulated maps
 * give every row of a set its merged-node current.
 * Bad or overlapping sets, out-of-range rows or set indices and k <= 0 give CS_B200_ERR_ARG before any
 * device work; so does a column whose flux comes out <= 0 (a pair with no conducting path).            */
int cs_b200_solve_region_pairs(cs_b200_handle* h, int64_t nsets, const int64_t* set_ptr,
                               const int64_t* set_rows, int64_t k, const int64_t* set_a,
                               const int64_t* set_b, const double* weight, double rtol, int64_t itmax,
                               void* R, void* volt, void* curr, int accumulate,
                               int64_t* iters, double* relres);

/* Advanced-mode columns with direct grounds on ONE resident operator (src/raster/advanced.jl:274-305 with
 * Inf grounds only; the one-to-all loop src/raster/onetoall.jl:106-118).  Column c: the rows of set gset[c]
 * are held at 0 V (each its own node), b = sum_e src_vals[e] e_{src_rows[e]} over src_ptr[c]..src_ptr[c+1]-1,
 * A_c v = b on the rest.  src_volt[c] = v at src_rows[src_ptr[c]].  weight / volt / curr / accumulate /
 * iters / relres as cs_b200_solve_pairs.  Sets as in cs_b200_solve_region_pairs (CSR over 0-based rows,
 * non-empty, sorted, unique); src_ptr[k+1] with src_ptr[0] = 0.  A column without sources, a source on its
 * own ground set, bad sets, rows or set indices, or k <= 0 give CS_B200_ERR_ARG before any device work.
 * Sources in a component that holds none of the column's ground rows make the system inconsistent: the
 * caller must not pass them (the gate reports such a column as CS_B200_ERR_RESIDUAL / _MAXITER).          */
int cs_b200_solve_grounded(cs_b200_handle* h, int64_t nsets, const int64_t* set_ptr, const int64_t* set_rows,
                           int64_t k, const int64_t* gset, const int64_t* src_ptr, const int64_t* src_rows,
                           const double* src_vals, const double* weight, double rtol, int64_t itmax,
                           void* src_volt, void* volt, void* curr, int accumulate, int64_t* iters,
                           double* relres);

/* Raster advanced mode on ONE resident operator (src/raster/advanced.jl:151-305): column c is one connected
 * component's solve on the handle's current operator L0 + diag(finite grounds of cs_b200_set_grounds).  The
 * rows of set gset[c] (the component's Inf grounds) are held at 0 V; gset[c] = -1 means the column has no
 * direct grounds, which needs a handle that carries finite grounds.  Sources, sets, weight / volt / curr /
 * accumulate / iters / relres and the argument checks as cs_b200_solve_grounded (nsets may be 0 when every
 * gset[c] is -1); gset[c] = -1 without finite grounds on the handle is CS_B200_ERR_ARG before any device
 * work.  The node currents add each node's finite-ground current x = fg_i v_i to the inflow (x < 0, as -x)
 * or the outflow (x > 0) before max(inflow, outflow) (src/out.jl:186-207); the 1e-8 cut of the branch
 * currents stays per column and does not apply to it.  The other entry points never add that term.        */
int cs_b200_solve_advanced(cs_b200_handle* h, int64_t nsets, const int64_t* set_ptr, const int64_t* set_rows,
                           int64_t k, const int64_t* gset, const int64_t* src_ptr, const int64_t* src_rows,
                           const double* src_vals, const double* weight, double rtol, int64_t itmax, void* volt,
                           void* curr, int accumulate, int64_t* iters, double* relres);

/* Network advanced mode on ONE whole-graph operator (src/raster/advanced.jl:184-242 for networks): the columns
 * are solved as in cs_b200_solve_advanced (sets, gset with -1 for finite grounds only, sources, rtol, itmax,
 * iters, relres).  owner: n values, owner[row] = the column whose connected component contains row, or -1.
 * Each column's voltages are added into one vector on the rows it owns; volt (n), curr (n) and branch (nb,
 * order of cs_b200_branch_index) -- each may be NULL -- are that vector, its node currents with the
 * finite-ground currents, and its branch currents, all under ONE 1e-8 cut over the whole graph, as the
 * reference takes them of the summed voltages.  The cumulative vectors are not touched.  owner values
 * outside [-1, k), a source or ground-set row of column c not owned by c, and the checks of
 * cs_b200_solve_advanced are CS_B200_ERR_ARG before any device work.                                     */
int cs_b200_solve_advanced_network(cs_b200_handle* h, int64_t nsets, const int64_t* set_ptr,
                                   const int64_t* set_rows, int64_t k, const int64_t* gset, const int64_t* src_ptr,
                                   const int64_t* src_rows, const double* src_vals, const int64_t* owner,
                                   double rtol, int64_t itmax, void* volt, void* curr, void* branch,
                                   int64_t* iters, double* relres);

/* Batched solve with SPARSE right-hand sides, device-resident -- the advanced-mode kernel
 * (src/raster/advanced.jl:274-305) for source/ground sets without finite grounds, and
 * the all-to-one loop built on it (src/raster/onetoall.jl:110-118,146-151):
 *   column c:  b = sum_e vals[e] * e_rows[e]   for e in colptr[c] .. colptr[c+1]-1
 *              A v = b ;  v -= v[ref[c]]
 * A Dirichlet ground at ref[c] with the other entries as current sources is expressed on
 * the singular Laplacian by giving ref[c] the entry  -(sum of the sources)  (current
 * conservation), exactly as the pairwise driver does with  -1 / +1 ; duplicates of a row
 * within a column add.  Nothing of size n crosses PCIe unless volt / curr are requested.
 * probe: nprobe rows whose shifted voltages are returned in probe_volt (host, k x nprobe,
 * row-major, dtype); may be NULL / 0.  volt, curr, accumulate, weight: as in solve_pairs.  */
int cs_b200_solve_sources(cs_b200_handle* h, int64_t k, const int64_t* colptr, const int64_t* rows,
                          const double* vals, const int64_t* ref, const double* weight,
                          double rtol, int64_t itmax, int64_t nprobe, const int64_t* probe,
                          void* probe_volt, void* volt, void* curr, int accumulate,
                          int64_t* iters, double* relres);

/* Omniscape's moving-window solve (compute_omniscape_current, src/utils.jl:145-257) for a batch of
 * nwin windows of nrows x ncols cells, without a handle: one upload, one kernel launch (one CTA per
 * window), one download, whatever nwin is.
 *   g, src, gnd: host, the nwin windows stacked, each column-major (cell r + c * nrows), element type
 *                `dtype`.  Cells with g <= 0 (0, NODATA -9999, NaN) are not nodes; pad windows of
 *                other shapes with g = 0.  Ground values are conductances: Inf = direct ground (0 V),
 *                finite = added to the diagonal.  Conflicts: rmvsrc.  Neighbours: 4 or 8 with the
 *                average-conductance rule.
 *   Every connected component of a window is its own advanced-mode solve (skipped when its sources
 *   or its grounds sum to 0): Jacobi-preconditioned CG in fp64 with the stop rule
 *   sqrt(r'z) <= sqrt(eps) + rtol sqrt(r0'z0), at most itmax iterations, then the true-residual
 *   gate 1e-4 on the reduced system and the node currents of src/out.jl:178-207.
 *   cur:  host, nwin x nrows x ncols fp64 (same layout), node current per cell, 0 off solved components.
 *   volt: NULL or the same for the voltages.
 *   iters[nwin] (CG iterations summed over the window's components), relres[nwin] (largest true
 *   relative residual of its components), first_failed: may be NULL.
 * CS_B200_ERR_RESIDUAL / CS_B200_ERR_MAXITER name the first window that failed the gate / ran into
 * itmax in *first_failed (-1 otherwise) and in cs_b200_last_error(NULL); every output is still
 * written.  Bad shapes, a NULL required pointer or a bad dtype give CS_B200_ERR_ARG.               */
int cs_b200_solve_advanced_batch(int64_t nwin, int64_t nrows, int64_t ncols, const void* g, const void* src,
                                 const void* gnd, int dtype, int four_neighbors, int device, double rtol,
                                 int64_t itmax, void* cur, void* volt, int64_t* iters, double* relres,
                                 int64_t* first_failed);

/* Omniscape's moving-window loop over one landscape: the windows of cs_b200_solve_advanced_batch cut on
 * the device from resident rasters, their currents summed into one landscape map on the device.
 *   g, src: host, nrows x ncols, column-major (cell r + c * nrows, as cs_b200_create_from_raster),
 *           element type `dtype`; uploaded once.
 *   Window w (nwin of them) is the (2 radius + 1)^2 square centred on the target (target_rows[w],
 *   target_cols[w]), 0-based; its cell (i, j) is landscape cell (tr - radius + i, tc - radius + j).  A
 *   cell is a node when that position is inside the landscape, g > 0 there (0, NODATA -9999 and NaN are
 *   not), and, when `circular`, (i - radius)^2 + (j - radius)^2 <= radius^2.  On the nodes the window's
 *   conductance is g, its source (T)(source_scale[w] * src) and its ground ground[w] at the centre cell
 *   only (a conductance: Inf = direct ground); every other cell has g = 0.  Each window is then solved
 *   exactly as one window of cs_b200_solve_advanced_batch (four_neighbors, rtol, itmax, gate).
 *   source_scale: NULL (all 1) or nwin finite values.  ground: NULL (all Inf) or nwin values > 0.
 *   cum:  host, nrows x ncols fp64, column-major: cum[r, c] = sum over w, in window order, of window w's
 *         current at (r - tr + radius, c - tc + radius), from +0.0 -- bit-identical whatever the batch
 *         split and on repeats (fixed order, no floating-point atomics).  Zero when nwin = 0.
 *   iters[nwin], relres[nwin], first_failed: as in cs_b200_solve_advanced_batch; may be NULL.
 * Windows go to the device in batches of consecutive windows, as many as fit max_batch_bytes at the
 * per-window device bytes of cs_b200_solve_advanced_batch (at least one); the rasters and cum stay on
 * the device for the whole call, so host memory is O(landscape + nwin).
 * CS_B200_ERR_RESIDUAL / CS_B200_ERR_MAXITER name the first window (global index) that failed the gate /
 * ran into itmax in *first_failed and in cs_b200_last_error(NULL); every output is still written.
 * CS_B200_ERR_ARG before any device work: a bad shape, more than INT_MAX landscape or window cells, a
 * negative radius, a target outside the landscape, a ground <= 0 or NaN, a scale that is NaN or Inf, a
 * NULL required pointer, max_batch_bytes <= 0, a bad dtype, rtol or itmax.                               */
int cs_b200_solve_moving_windows(int64_t nrows, int64_t ncols, const void* g, const void* src, int dtype,
                                 int64_t nwin, const int64_t* target_rows, const int64_t* target_cols,
                                 int64_t radius, int circular, const double* source_scale, const double* ground,
                                 int four_neighbors, int device, double rtol, int64_t itmax,
                                 int64_t max_batch_bytes, double* cum, int64_t* iters, double* relres,
                                 int64_t* first_failed);

/* A whole Omniscape job over one landscape: block targets, per-window source normalisation, the
 * moving-window solves of cs_b200_solve_moving_windows (disc on, direct ground at the target), and
 * optionally the flow potential and the normalised current map, all on the device.
 *   g, src: host, nrows x ncols, column-major, element type `dtype`: conductance (a cell is a node when
 *           g > 0) and source strength; uploaded once.  half = (block_size - 1) / 2.
 *   1. s'[c] = src[c] where src[c] > source_threshold, src[c] is finite and g[c] > 0; else 0.
 *   2. Candidates: the block centres (half + i block_size, half + j block_size) inside the landscape, j
 *      outer, i inner.  amps = sum of s' over the block clipped to the landscape, fp64 from +0.0, column
 *      outer, row inner.  Targets: the candidates with amps > 0, in candidate order.
 *   3. Window sum S_w = sum of s' over the landscape cells in the disc of `radius` around the target and
 *      outside its block (|dr| > half or |dc| > half), fp64 in a fixed CTA order; scale = S_w > 0 ?
 *      amps / S_w : 0.
 *   4. Conductance window: cs_b200_solve_moving_windows's circular window, sources (T)(scale * s') on
 *      nodes outside the block, 0 inside it, a direct (Inf) ground at the centre.
 *   5. Flow-potential window (flow_potential != 0): the same square and disc with g = 1 on every
 *      landscape cell in the disc (NODATA, 0 and NaN cells included), the same sources, a direct ground
 *      at the centre.
 *   6. cum / fp: every target's window currents summed in target order from +0.0 in fp64 (bit-identical
 *      whatever the batch split); normalized = fp > 0 ? cum / fp : 0; then every cell where g is NaN or
 *      -9999 is -9999 in every returned map.
 *   cum (and fp, normalized when flow_potential): host, nrows x ncols fp64, column-major.
 *   max_targets: capacity of target_rows, target_cols, amps, scale, iters, relres, fp_iters and
 *   fp_relres; at least the number of block centres.  *ntargets receives the number of targets; the
 *   target arrays (0-based rows and columns), amps and scale receive one value per target.
 *   iters, relres (conductance windows), fp_iters, fp_relres (flow-potential windows): may be NULL.
 * Each window is solved exactly as one window of cs_b200_solve_advanced_batch.  Batches hold as many
 * targets as fit max_batch_bytes at the per-window bytes of cs_b200_solve_advanced_batch, both windows of
 * a target counted (at least one target).
 * CS_B200_ERR_RESIDUAL / CS_B200_ERR_MAXITER: *first_failed is the target of the first failing window
 * (targets in order, a target's conductance window before its flow-potential window) and
 * cs_b200_last_error(NULL) names it and its window kind; every output is still written.
 * CS_B200_ERR_ARG before any device work: a bad shape, more than INT_MAX landscape or window cells, a
 * negative radius, an even or < 1 block_size, source_threshold < 0 or NaN, max_targets below the number
 * of block centres, a NULL g, src, cum, ntargets, target_rows, target_cols, amps or scale, a NULL fp or
 * normalized with flow_potential, max_batch_bytes <= 0, a bad dtype, rtol or itmax.                   */
int cs_b200_solve_omniscape(int64_t nrows, int64_t ncols, const void* g, const void* src, int dtype,
                            int64_t radius, int64_t block_size, double source_threshold, int flow_potential,
                            int four_neighbors, int device, double rtol, int64_t itmax, int64_t max_batch_bytes,
                            double* cum, double* fp, double* normalized, int64_t max_targets, int64_t* ntargets,
                            int64_t* target_rows, int64_t* target_cols, double* amps, double* scale,
                            int64_t* iters, double* relres, int64_t* fp_iters, double* fp_relres,
                            int64_t* first_failed);

/* Cumulative / max node-current vectors (n values of dtype each; either may be
 * NULL).  max is initialised to -9999 like src/utils.jl:124.                        */
int cs_b200_read_currents(cs_b200_handle* h, void* cum, void* max);
int cs_b200_reset_currents(cs_b200_handle* h);
/* The cumulative branch vector of cs_b200_solve_pairs_branch (nb values of dtype; zeros before any
 * accumulation).  cs_b200_reset_currents zeroes it with the node vectors.                           */
int cs_b200_read_branch_currents(cs_b200_handle* h, void* cum_branch);
/* Device pointers of the same vectors (for an NCCL reduce across ranks).            */
int cs_b200_currents_device_ptrs(cs_b200_handle* h, void** d_cum, void** d_max);

int cs_b200_get_stats(const cs_b200_handle* h, cs_b200_stats* out);

/* The CUDA stream (cudaStream_t) every kernel of this handle is launched on, so a
 * caller can bracket calls with its own CUDA events.                                */
int cs_b200_stream(cs_b200_handle* h, void** stream);

/* Per-launch timing of the dominant kernel.  enable = 1/0 switches event pairs around
 * every SpMM launch on/off (the CUDA-graph path is bypassed while on) and clears the
 * totals; enable < 0 only reads.  *total_ms / *launches: totals since last enable.  */
int cs_b200_profile_spmm(cs_b200_handle* h, int enable, double* total_ms, int64_t* launches);

/* Algorithmic bytes (nnz (s_v+4) + (n+1) 4 + panel passes, DESIGN.md section 4) summed over
 * the launches timed since profiling was last enabled; read BEFORE disabling.          */
int cs_b200_profile_bytes(cs_b200_handle* h, double* algorithmic_bytes);

/* ---- multi-GPU: pair sharding behind the C ABI (SURVEY.md 8e) -----------------------------
 * One process (or thread) per GPU.  The path shards over independent focal pairs against ONE
 * replicated read-only operator -- the axis the reference threads over (src/core.jl:262-272) --
 * so the only collectives are: the broadcast of the matrix from the root, and at the END of a job
 * the gather of the per-pair resistances and the SUM / MAX reduction of the cumulative / max
 * current vectors (src/out.jl:100-107).  NCCL is loaded at run time (dlopen "libnccl.so.2"); the
 * host language only has to move the 128-byte unique id from rank 0 to the other ranks (MPI
 * broadcast, a socket, a file) -- nothing else crosses the host.                              */
typedef struct cs_b200_comm cs_b200_comm;

/* rank 0: fill id128 (128 bytes) with a fresh NCCL unique id                                 */
int cs_b200_comm_unique_id(void* id128);
/* every rank: join the communicator on `device`                                              */
int cs_b200_comm_init(int device, int rank, int nranks, const void* id128, cs_b200_comm** out);
void cs_b200_comm_destroy(cs_b200_comm* c);
const char* cs_b200_comm_last_error(const cs_b200_comm* c);

/* cs_b200_create on every rank from the matrix held by `root` (arguments as cs_b200_create;
 * rowptr / colidx / vals may be NULL on the other ranks, n / nnz / dtype / index_* must agree):
 * the root uploads and narrows the CSR, one ncclBroadcast replicates it (and the root's
 * aggregation seeds), every rank builds its own preconditioner from the device copy.          */
int cs_b200_create_bcast(cs_b200_comm* c, int root, int64_t n, int64_t nnz, const void* rowptr,
                         const void* colidx, const void* vals, int index_bits, int index_base,
                         int dtype, const cs_b200_opts* opts, cs_b200_handle** out);

/* end of job: cum <- SUM over ranks, max <- MAX over ranks, in place in every rank's handle
 * (ncclAllReduce on the handle's solve stream, right behind the last accumulation kernel)     */
int cs_b200_comm_reduce_currents(cs_b200_comm* c, cs_b200_handle* h);

/* end of job: every rank contributes the resistances of its own pairs (global pair indices
 * my_idx[k_mine], values my_R[k_mine], fp64) and receives all k_total of them in R_all
 * (entries no rank contributed stay -1, the reference's "not solved" marker).                 */
int cs_b200_comm_gather_pairs(cs_b200_comm* c, int64_t k_total, const int64_t* my_idx,
                              int64_t k_mine, const double* my_R, double* R_all);

/* max over ranks of a host double (timings) / sum of int64 counters                           */
int cs_b200_comm_max_double(cs_b200_comm* c, double* v, int count);
int cs_b200_comm_barrier(cs_b200_comm* c);

/* The same totals per kernel class (read before disabling): 18 slots, slot = 2 * epilogue + (fp32 ? 1 : 0)
 * with epilogue 0 plain, 1 CG (p.Ap), 2 residual + norms (gate), 3 residual, 4 Jacobi sweep, 5 Jacobi
 * sweep + r.z, 6 prolong-add, 7 fused prolongation + sweep, 8 fused CG step (p = z + beta p, A p, p.Ap,
 * deferred x update; since ABI 1005, 16 slots before).                                             */
int cs_b200_profile_classes(cs_b200_handle* h, double* ms18, double* bytes18, int64_t* launches18);
/* The same for the first nslots slots (20 exist): slot 18 (19 unused) is the fused residual update + level-0
 * residual sweep of the mixed cycle (r -= alpha A p, r32, the fp32 level-0 residual; kernels.cuh
 * k_stencil_res_update), which the 18-slot call leaves out.                                       */
int cs_b200_profile_classes_n(cs_b200_handle* h, int nslots, double* ms, double* bytes, int64_t* launches);

/* Library/ABI version: major*1000 + minor.                                          */
int cs_b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* CS_B200_H */

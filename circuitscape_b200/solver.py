"""Host-side mirror of the reference's Solver plug-in surface for the CUDA path.

Same names, argument meaning and error behaviour as the methods a Circuitscape.jl
package extension overloads (ext/CircuitscapePardisoExt.jl:31-45,
ext/CircuitscapeAppleAccelerateExt.jl:8-22; generics in src/core.jl:519-523,
646-653 and src/raster/advanced.jl:307-333):

    construct_cholesky_factor(matrix, solver)       -> B200Factor   (hook #1)
    solve_linear_system(factor, matrix, rhs)        -> lhs          (hook #2)
    multiple_solve(solver, matrix, sources)         -> volt         (hook #3)

`B200Factor` is the opaque "factor" object: it owns a `cs_b200_handle*`.  The Julia
glue of INTEGRATION.md is a line-for-line twin of this file using `ccall`.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import scipy.sparse as sp

from . import _lib

# solver-name table (reference: src/consts.jl:12-15 AMG/CHOLMOD/PARDISO/ACCELERATE)
CUDAB200 = ["cuda", "gpu", "b200", "cg+jacobi+cuda", "cg+amg+cuda"]


@dataclass
class CUDASolver:
    """`struct CUDASolver <: Solver; bs::Int end` -- bs = cfg.cholmod_batch_size
    (src/core.jl:57-63, 81-90).  Extra knobs are this path's own."""
    bs: int = 1000
    precision: str = "double"        # cfg.precision  (src/run.jl:29)
    device: int = 0
    rtol: float = 1e-6               # src/core.jl:639
    itmax: int = 100_000             # src/core.jl:639
    precond: str = "amg"             # "amg" (smoothed aggregation V-cycle) | "jacobi"
    panel_width: int = 8
    check_every: int = 16
    use_graph: object = True      # True: device-side WHILE-graph loop; "chunk": host-polled graph chunks; False: plain launches
    window: str = "auto"             # TMA-staged windowed SpMM: auto | on | off
    f32_compute: bool = False        # precision = single: keep fp32 ON THE DEVICE too (see B200Factor)
    mixed: bool = True               # fp64 + AMG: fp32 V-cycle inside fp64 CG
    stencil: str = "auto"            # stencil (DIA) SpMM on full-raster operators: auto | on | off
    setup: str = "auto"              # hierarchy / window records built: auto (device) | device | host
    superpose: bool = False          # pairwise driver: one solve per focal NODE, pairs by superposition
    batch_all_to_one: bool = False   # all-to-one: every iteration a column of ONE batch on one operator
    batch_one_to_all: bool = False   # one-to-all: one solve per iteration on ONE grounded operator
    resident_grounds: bool = False   # advanced mode: keep the component's factor, move the grounds on the
                                     # device (cs_b200_set_grounds) instead of a new handle per solve
    onetoall_raster: bool = False    # one-to-all / all-to-one iterations as columns on one whole-raster
                                     # handle (core.plan_onetoall); takes precedence over batch_*
    branch_on_device: bool = False   # network pairwise: branch currents and their cumulative vector on the
                                     # device (cs_b200_solve_pairs_branch) instead of from per-pair voltages
    pairwise_raster: bool = False    # raster pairwise with distinct point ids: every component's pairs as columns
                                     # on one whole-raster handle, components labelled on the device
                                     # (core._raster_pairs_device) instead of a host graph and a handle per component
    front_end_on_device: bool = False    # raster advanced, one-to-all (onetoall_raster) and focal regions: node
                                         # map, component labels and advanced mode's columns from the whole-raster
                                         # handle (components, plan_advanced) instead of a host graph

    @property
    def dtype(self):
        """element type of the caller-side buffers (cfg.precision, src/run.jl:29)."""
        return np.float32 if self.precision in ("single", "Single") else np.float64

    @property
    def device_dtype(self):
        """element type of the device arithmetic.  With fp32 *storage* of x the true residual
        ||Gv - b|| / ||b|| cannot fall below ~eps32 * ||G|| ||v|| / ||b||, which is already above the
        reference's own 1e-4 gate (src/core.jl:641) at ~4e6 nodes (measured: 1.2e-4 at 1000^2,
        0.5 at 2000^2) -- upstream never exercises Float32 (SURVEY.md section 4).  So single-
        precision jobs are promoted: Float32 in and out at the boundary, fp64 on the device.
        `f32_compute=True` keeps fp32 panels for small problems and for the kernel tests."""
        if self.dtype == np.float32 and not self.f32_compute:
            return np.float64
        return self.dtype


def _opt(a, dtype):
    """None, or `a` as a contiguous array of `dtype` (the optional per-column inputs)."""
    return None if a is None else np.ascontiguousarray(a, dtype=dtype)


def _csr(ragged, dtype):
    """A ragged list of 1-D arrays as CSR: (ptr (len + 1,) int64, the arrays concatenated as `dtype`)."""
    ptr = np.zeros(len(ragged) + 1, dtype=np.int64)
    ptr[1:] = np.cumsum([len(a) for a in ragged])
    vals = np.concatenate([np.asarray(a, dtype=dtype) for a in ragged]) if len(ragged) else np.zeros(0)
    return ptr, np.ascontiguousarray(vals, dtype=dtype)


def _grounded_columns(sets, gset, sources):
    """Columns with Dirichlet sets and sparse sources as the C entries take them: sets as CSR (ptr, rows),
    gset (k,) int64, sources[c] = (rows, values) as CSR (sptr, srows, svals)."""
    ptr, rows = _csr(sets, np.int64)
    gset = np.ascontiguousarray(gset, dtype=np.int64)
    assert len(sources) == len(gset)
    sptr, srows = _csr([r for r, _ in sources], np.int64)
    _, svals = _csr([v for _, v in sources], np.float64)
    assert len(srows) == len(svals) == sptr[-1]
    return ptr, rows, gset, sptr, srows, svals


class SolverResidualError(RuntimeError):
    """The reference's `error("... residual $r exceeds tolerance 1e-4 ...")`
    (src/core.jl:641,650)."""


class B200Factor:
    """Opaque factor: CSR + preconditioner resident on one GPU (cs_b200_create)."""

    def __init__(self, matrix, solver: CUDASolver, log_transform=False):
        self._bind(solver)
        lib = self._lib
        n, nnz, rowptr, colidx, vals, bits = self._host_csr(matrix)
        self.n = n
        opts = self._opts(solver, log_transform)
        rc = lib.cs_b200_create(n, nnz, _lib._ptr(rowptr), _lib._ptr(colidx), _lib._ptr(vals),
                                bits, 0, _lib.dtype_code(self.dtype), solver.device,
                                C.byref(opts), C.byref(self._h))
        _lib.check(lib, None, rc)

    def _host_csr(self, matrix):
        """`matrix` as the host CSR cs_b200_create and cs_b200_create_bcast take: (n, nnz, rowptr, colidx,
        vals, index bits), sorted indices, the index arrays of one integer type, values contiguous in the
        device's element type."""
        m = sp.csr_matrix(matrix)
        m.sort_indices()
        vals = np.ascontiguousarray(m.data, dtype=self.dtype)
        rowptr = np.ascontiguousarray(m.indptr)
        colidx = np.ascontiguousarray(m.indices)
        if colidx.dtype != rowptr.dtype:
            colidx = colidx.astype(rowptr.dtype)
        return m.shape[0], m.nnz, rowptr, colidx, vals, 64 if rowptr.dtype == np.int64 else 32

    def _bind(self, solver):
        """The attributes every factor carries before its handle is created: the library, an empty handle, the
        caller's (io_dtype) and the device's (dtype) element types, the solver."""
        self._lib = _lib.load()
        self._h = C.c_void_p()
        self.io_dtype = np.dtype(solver.dtype)
        self.dtype = np.dtype(solver.device_dtype)
        self.solver = solver

    @staticmethod
    def _opts(solver, log_transform=False):
        opts = _lib.Opts()
        opts.precond = _lib.PRECOND_AMG if solver.precond == "amg" else _lib.PRECOND_JACOBI
        opts.panel_width = solver.panel_width
        opts.check_every = solver.check_every
        opts.use_graph = 2 if solver.use_graph == "chunk" else (1 if solver.use_graph else -1)
        opts.log_transform = 1 if log_transform else 0
        opts.window = {"auto": 0, "on": 1, "off": -1}[solver.window]
        opts.mixed = 0 if solver.mixed else -1
        opts.setup = {"auto": 0, "host": 1, "device": 2}[solver.setup]
        opts.stencil = {"auto": 0, "on": 1, "off": -1}[solver.stencil]
        return opts

    @classmethod
    def from_raster_polygons(cls, conductance, polymap, solver: "CUDASolver", four_neighbors=False, avg_res=False,
                             log_transform=False):
        """Factor of a raster WITH short-circuit polygons, assembled on the device
        (cs_b200_create_from_raster_poly: construct_node_map with a polygon map, construct_graph with
        summed parallel adjacencies, laplacian!).  Returns (factor, nodemap) -- nodemap as the reference's
        (1-based node id per cell, 0 = none).  NODATA cells may be given as 0 or negative values."""
        f = cls.__new__(cls)
        f._bind(solver)
        lib = f._lib
        g = np.asfortranarray(conductance, dtype=f.dtype)
        pm = None if polymap is None else np.asfortranarray(polymap, dtype=np.int32)
        nodemap = np.zeros(g.shape, dtype=np.int32, order="F")
        n, nnz = C.c_int64(), C.c_int64()
        opts = cls._opts(solver, log_transform)
        rc = lib.cs_b200_create_from_raster_poly(g.shape[0], g.shape[1], _lib._ptr(g), _lib._ptr(pm),
                                                 _lib.dtype_code(f.dtype), 1 if four_neighbors else 0,
                                                 1 if avg_res else 0, solver.device, C.byref(opts), C.byref(f._h),
                                                 C.byref(n), C.byref(nnz), _lib._ptr(nodemap))
        _lib.check(lib, None, rc)
        f.n = n.value
        return f, nodemap

    @classmethod
    def from_raster(cls, conductance, solver: "CUDASolver", four_neighbors=False, avg_res=False,
                    log_transform=False):
        """Factor of a whole conductance raster, assembled ON THE DEVICE
        (cs_b200_create_from_raster): construct_node_map without polygons + construct_graph +
        laplacian! (src/raster/pairwise.jl:271-367, src/core.jl:608-624).  `conductance`:
        2-D array, cells <= 0 / NODATA are not nodes; rows of the factor are the reference's
        node numbers minus one (column-major over the valid cells)."""
        f = cls.__new__(cls)
        f._bind(solver)
        lib = f._lib
        g = np.asfortranarray(conductance, dtype=f.dtype)       # Julia's memory order
        n, nnz = C.c_int64(), C.c_int64()
        opts = cls._opts(solver, log_transform)
        rc = lib.cs_b200_create_from_raster(g.shape[0], g.shape[1], _lib._ptr(g), _lib.dtype_code(f.dtype),
                                            1 if four_neighbors else 0, 1 if avg_res else 0, solver.device,
                                            C.byref(opts), C.byref(f._h), C.byref(n), C.byref(nnz))
        _lib.check(lib, None, rc)
        f.n = n.value
        return f

    def get_csr(self):
        """The handle's operator as a SciPy CSR (downloaded; parity / debugging hook)."""
        n, nnz = C.c_int64(), C.c_int64()
        _lib.check(self._lib, self._h, self._lib.cs_b200_get_dims(self._h, C.byref(n), C.byref(nnz)))
        rp = np.empty(n.value + 1, dtype=np.int32)
        ci = np.empty(nnz.value, dtype=np.int32)
        va = np.empty(nnz.value, dtype=self.dtype)
        _lib.check(self._lib, self._h, self._lib.cs_b200_get_csr(self._h, _lib._ptr(rp), _lib._ptr(ci), _lib._ptr(va)))
        return sp.csr_matrix((va, ci, rp), shape=(n.value, n.value))

    def levels(self):
        """The multigrid hierarchy as SciPy matrices (downloaded; parity / debugging hook):
        list of dicts with A, P, R (None on the coarsest level), omega, windowed flags, and A_stencil_slots:
        the diagonals the stencil form of A stores (0: none, 9, or 5 for a bitwise symmetric operator)."""
        out = []
        l = 0
        while True:
            lev = {}
            for name, which in (("A", 0), ("P", 1), ("R", 2)):
                nr, nc, nnz = C.c_int64(), C.c_int64(), C.c_int64()
                om, win = C.c_double(), C.c_int()
                rc = self._lib.cs_b200_level_info(self._h, l, which, C.byref(nr), C.byref(nc), C.byref(nnz),
                                                  C.byref(om), C.byref(win))
                if rc != _lib.OK:
                    lev[name] = None
                    continue
                rp = np.empty(nr.value + 1, dtype=np.int32)
                ci = np.empty(nnz.value, dtype=np.int32)
                va = np.empty(nnz.value, dtype=np.float64)
                _lib.check(self._lib, self._h,
                           self._lib.cs_b200_level_csr(self._h, l, which, _lib._ptr(rp), _lib._ptr(ci), _lib._ptr(va)))
                lev[name] = sp.csr_matrix((va, ci, rp), shape=(nr.value, nc.value))
                lev["omega"] = om.value
                lev[name + "_windowed"] = bool(win.value)        # TMA-window records or stencil form
                lev[name + "_stencil"] = win.value == 2
            if lev["A"] is None:
                break
            slots = C.c_int()
            _lib.check(self._lib, self._h, self._lib.cs_b200_level_stencil(self._h, l, C.byref(slots)))
            lev["A_stencil_slots"] = slots.value                # 0, 9, or 5: symmetric, upper diagonals only
            out.append(lev)
            l += 1
        return out

    def set_grounds(self, finite=None, dirichlet=None):
        """cs_b200_set_grounds: re-derive the operator on the device as  G + diag(finite)  with the rows /
        columns of the `dirichlet` nodes replaced by identity rows (src/raster/advanced.jl:274-305) and
        rebuild the preconditioner; (None, None) restores the pristine operator."""
        g = None if finite is None else np.ascontiguousarray(finite, dtype=self.dtype)
        m = None if dirichlet is None else np.ascontiguousarray(np.asarray(dirichlet) != 0, dtype=np.uint8)
        assert g is None or len(g) == self.n
        assert m is None or len(m) == self.n
        _lib.check(self._lib, self._h, self._lib.cs_b200_set_grounds(self._h, _lib._ptr(g), _lib._ptr(m)))

    def operator_form(self):
        """'stencil' (9 diagonals, k_stencil), 'windowed' (TMA-staged CSR records, k_spmm_win) or
        'csr' (plain row-block kernel) for the finest operator the CG SpMM runs on."""
        win = C.c_int()
        rc = self._lib.cs_b200_level_info(self._h, 0, 0, None, None, None, None, C.byref(win))
        _lib.check(self._lib, self._h, rc)
        return {2: "stencil", 1: "windowed"}.get(win.value, "csr")

    # -- lifetime ---------------------------------------------------------
    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._lib.cs_b200_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # -- calls ------------------------------------------------------------
    def _limits(self, rtol, itmax):
        """rtol and itmax of one call: the solver's unless given."""
        return (self.solver.rtol if rtol is None else rtol, self.solver.itmax if itmax is None else itmax)

    def _columns(self, k, want_volt, want_curr):
        """Per-column outputs of a batched solve: volt, curr (n, k) F-ordered or None, iters, relres."""
        cols = lambda want: np.empty((self.n, k), dtype=self.dtype, order="F") if want else None
        return cols(want_volt), cols(want_curr), np.zeros(k, dtype=np.int64), np.zeros(k, dtype=np.float64)

    def _io(self, a):
        """`a` (or None) in the caller's element type io_dtype."""
        return a.astype(self.io_dtype) if a is not None and self.io_dtype != self.dtype else a

    def stats(self):
        st = _lib.Stats()
        self._lib.cs_b200_get_stats(self._h, C.byref(st))
        return st.as_dict()

    def stream_ptr(self):
        p = C.c_void_p()
        _lib.check(self._lib, self._h, self._lib.cs_b200_stream(self._h, C.byref(p)))
        return p.value or 0

    def profile_spmm(self, enable):
        """enable True/False: start/stop per-launch SpMM timing; returns (ms, launches)
        accumulated since the previous enable."""
        ms, cnt = C.c_double(), C.c_int64()
        _lib.check(self._lib, self._h,
                   self._lib.cs_b200_profile_spmm(self._h, -1 if enable is None else int(bool(enable)),
                                                  C.byref(ms), C.byref(cnt)))
        return ms.value, cnt.value

    def profile_classes(self):
        """per kernel class of the timed finest-level launches: {name: (ms, algorithmic bytes, launches)}"""
        names = ["plain", "cg", "residual_gate", "residual", "jacobi", "jacobi_dot", "prolong_add", "prolong_jacobi_fused",
                 "cg_step_fused", "residual_sweep_fused"]
        ms = np.zeros(2 * len(names))
        by = np.zeros(2 * len(names))
        ln = np.zeros(2 * len(names), dtype=np.int64)
        _lib.check(self._lib, self._h, self._lib.cs_b200_profile_classes_n(self._h, len(ms), _lib._ptr(ms), _lib._ptr(by),
                                                                           _lib._ptr(ln)))
        return {f"{names[i // 2]}_{'f32' if i % 2 else 'f64'}": (float(ms[i]), float(by[i]), int(ln[i]))
                for i in range(2 * len(names)) if ln[i]}

    def profile_bytes(self):
        """algorithmic bytes of the launches timed since profiling was enabled."""
        b = C.c_double()
        _lib.check(self._lib, self._h, self._lib.cs_b200_profile_bytes(self._h, C.byref(b)))
        return b.value

    def spmv(self, x, reps=1):
        x = np.ascontiguousarray(x, dtype=self.dtype)
        y = np.empty_like(x)
        ms = C.c_double()
        rc = self._lib.cs_b200_spmv(self._h, _lib._ptr(x), _lib._ptr(y), reps, C.byref(ms))
        _lib.check(self._lib, self._h, rc)
        return y, ms.value

    def spmm(self, X):
        """Y = A X for X (n, k), k in {1,2,4,8}, through the panel kernel."""
        X = np.asfortranarray(X, dtype=self.dtype)
        Y = np.empty_like(X, order="F")
        rc = self._lib.cs_b200_spmm(self._h, X.shape[1], _lib._ptr(X), _lib._ptr(Y))
        _lib.check(self._lib, self._h, rc)
        return Y

    def apply_precond(self, R):
        """One application of the multigrid preconditioner, Z = M^-1 R, for R (n,) or (n, k),
        k in {1,2,4,8} (cs_b200_apply_precond).  Returns (Z, rz) with rz[c] = |r_c . z_c| as the
        cycle's last kernel reduces it."""
        R = np.asarray(R, dtype=self.dtype)
        vec = R.ndim == 1
        X = np.asfortranarray(R.reshape(self.n, -1))
        Z = np.empty_like(X, order="F")
        rz = np.zeros(X.shape[1])
        rc = self._lib.cs_b200_apply_precond(self._h, X.shape[1], _lib._ptr(X), _lib._ptr(Z), _lib._ptr(rz))
        _lib.check(self._lib, self._h, rc)
        return (Z[:, 0] if vec else Z), rz

    def bench_spmm(self, k, reps=20, flush_l2=False):
        ms = C.c_double()
        rc = self._lib.cs_b200_bench_spmm(self._h, k, reps, 1 if flush_l2 else 0, C.byref(ms))
        _lib.check(self._lib, self._h, rc)
        return ms.value

    def bench_cg_iter(self, k, reps=20):
        ms = C.c_double()
        rc = self._lib.cs_b200_bench_cg_iter(self._h, k, reps, C.byref(ms))
        _lib.check(self._lib, self._h, rc)
        return ms.value

    def solve_rhs(self, rhs, rtol=None, itmax=None, raise_on_residual=True, out=None):
        """rhs: (n,) or (n, k).  Returns (lhs, iters, relres).  `out`: optional
        F-ordered (n, k) result buffer (e.g. pinned host memory)."""
        rhs = np.asarray(rhs, dtype=self.dtype)
        vec = rhs.ndim == 1
        b = np.asfortranarray(rhs.reshape(self.n, -1))
        k = b.shape[1]
        x = out if out is not None else np.empty_like(b, order="F")
        assert x.flags.f_contiguous and x.shape == b.shape and x.dtype == b.dtype
        iters = np.zeros(k, dtype=np.int64)
        relres = np.zeros(k, dtype=np.float64)
        rc = self._lib.cs_b200_solve_rhs(self._h, k, _lib._ptr(b), _lib._ptr(x), *self._limits(rtol, itmax),
                                         _lib._ptr(iters), _lib._ptr(relres))
        self._raise(rc, raise_on_residual)
        if out is None:
            x = self._io(x)
        return (x[:, 0] if vec else x), iters, relres

    def solve_pairs(self, src, dst, weight=None, want_volt=False, want_curr=False,
                    accumulate=False, rtol=None, itmax=None, raise_on_residual=True, want_branch=False):
        """Batched focal-pair solve (src/dst 0-based rows).  Returns dict with
        R (k,), volt (n,k)|None, curr (n,k)|None, iters, relres, branch (nb,k)|None.
        want_branch: per-pair branch currents in the order of branch_index(), and with accumulate their
        cumulative vector on the device (cs_b200_solve_pairs_branch, read_branch_currents)."""
        src = np.ascontiguousarray(src, dtype=np.int64)
        dst = np.ascontiguousarray(dst, dtype=np.int64)
        k = len(src)
        R = np.zeros(k, dtype=self.dtype)
        volt, curr, iters, relres = self._columns(k, want_volt, want_curr)
        args = (self._h, k, _lib._ptr(src), _lib._ptr(dst), _lib._ptr(_opt(weight, np.float64)),
                *self._limits(rtol, itmax), _lib._ptr(R), _lib._ptr(volt), _lib._ptr(curr), 1 if accumulate else 0,
                _lib._ptr(iters), _lib._ptr(relres))
        branch = None
        if want_branch:
            branch = np.empty((self._num_branches(), k), dtype=self.dtype, order="F")
            rc = self._lib.cs_b200_solve_pairs_branch(*args, _lib._ptr(branch))
        else:
            rc = self._lib.cs_b200_solve_pairs(*args)
        self._raise(rc, raise_on_residual)
        return dict(R=self._io(R), volt=self._io(volt), curr=self._io(curr), iters=iters, relres=relres,
                    branch=self._io(branch))

    def _num_branches(self):
        """nb, the number of stored strictly-lower entries of the operator (cs_b200_branch_index)."""
        nb = C.c_int64()
        _lib.check(self._lib, self._h, self._lib.cs_b200_branch_index(self._h, C.byref(nb), None, None))
        return nb.value

    def branch_index(self):
        """The operator's branches (cs_b200_branch_index): (lo, hi), 0-based int64 arrays with lo < hi, one per
        stored strictly-lower entry, ordered by hi, then lo -- the order of every branch output."""
        nb = self._num_branches()
        lo = np.empty(nb, dtype=np.int64)
        hi = np.empty(nb, dtype=np.int64)
        n_ = C.c_int64()
        _lib.check(self._lib, self._h,
                   self._lib.cs_b200_branch_index(self._h, C.byref(n_), _lib._ptr(lo), _lib._ptr(hi)))
        return lo, hi

    def components(self):
        """Connected components of the operator, labelled on the device (cs_b200_components): (ncomp, comp_of)
        with comp_of (n,) int32 numbered in order of each component's smallest row -- SciPy's labels of the
        pristine operator's nonzero off-diagonal pattern."""
        nc = C.c_int64()
        comp_of = np.empty(self.n, dtype=np.int32)
        _lib.check(self._lib, self._h, self._lib.cs_b200_components(self._h, C.byref(nc), _lib._ptr(comp_of)))
        return nc.value, comp_of

    POLICIES = ("keepall", "rmvsrc", "rmvgnd", "rmvall")

    def plan_advanced(self, nodemap, source_map, ground_map, policy):
        """Raster advanced mode's columns planned on the device (cs_b200_plan_advanced + _read_advanced_plan):
        `nodemap` this handle's node map, the advanced-mode maps (float32 when both are, else float64), `policy`
        a name of POLICIES; any other value is keepall, as resolve_conflicts treats it.  Applies the finite grounds to the handle when any is nonzero.  Returns dict with
        nsolved, finite_applied, col_comp (ncol,), set_ptr / src_ptr (ncol + 1,), set_rows, src_rows (int64),
        src_vals (float64) and col_of_row (n,) int32."""
        sm, gm = np.asarray(source_map), np.asarray(ground_map)
        dt = np.float32 if sm.dtype == np.float32 and gm.dtype == np.float32 else np.float64
        nm = np.asfortranarray(nodemap, dtype=np.int32)
        sm, gm = np.asfortranarray(sm, dtype=dt), np.asfortranarray(gm, dtype=dt)
        if sm.shape != nm.shape or gm.shape != nm.shape:
            raise ValueError("the source and ground maps must have the node map's shape")
        ncol, nsolved, nset, nsrc = (C.c_int64() for _ in range(4))
        fin = C.c_int()
        _lib.check(self._lib, self._h, self._lib.cs_b200_plan_advanced(
            self._h, nm.shape[0], nm.shape[1], _lib._ptr(nm), _lib._ptr(sm), _lib._ptr(gm), _lib.dtype_code(dt),
            self.POLICIES.index(policy) if policy in self.POLICIES else 0, C.byref(ncol), C.byref(nsolved), C.byref(nset), C.byref(nsrc),
            C.byref(fin)))
        k = ncol.value
        out = dict(nsolved=nsolved.value, finite_applied=bool(fin.value), col_comp=np.empty(k, dtype=np.int64),
                   set_ptr=np.empty(k + 1, dtype=np.int64), set_rows=np.empty(nset.value, dtype=np.int64),
                   src_ptr=np.empty(k + 1, dtype=np.int64), src_rows=np.empty(nsrc.value, dtype=np.int64),
                   src_vals=np.empty(nsrc.value, dtype=np.float64), col_of_row=np.empty(self.n, dtype=np.int32))
        _lib.check(self._lib, self._h, self._lib.cs_b200_read_advanced_plan(
            self._h, *(_lib._ptr(out[a]) for a in ("col_comp", "set_ptr", "set_rows", "src_ptr", "src_rows",
                                                    "src_vals", "col_of_row"))))
        return out

    def read_branch_currents(self):
        """The cumulative branch vector (nb,) that solve_pairs(want_branch=True, accumulate=True) adds into."""
        cum = np.empty(self._num_branches(), dtype=self.dtype)
        _lib.check(self._lib, self._h, self._lib.cs_b200_read_branch_currents(self._h, _lib._ptr(cum)))
        return cum

    def solve_pairs_superposed(self, nodes, pi, pj, weight=None, want_volt=False, want_curr=False,
                               accumulate=False, rtol=None, itmax=None, raise_on_residual=True):
        """All pairs (nodes[pi[c]], nodes[pj[c]]) of one component from len(nodes)-1 solves
        (cs_b200_solve_pairs_superposed).  Same outputs as solve_pairs; `iters` are the
        iterations of the point solves."""
        nodes = np.ascontiguousarray(nodes, dtype=np.int64)
        pi = np.ascontiguousarray(pi, dtype=np.int64)
        pj = np.ascontiguousarray(pj, dtype=np.int64)
        k = len(pi)
        R = np.zeros(k, dtype=self.dtype)
        volt, curr, _, relres = self._columns(k, want_volt, want_curr)
        iters = np.zeros(max(len(nodes) - 1, 1), dtype=np.int64)
        rc = self._lib.cs_b200_solve_pairs_superposed(
            self._h, len(nodes), _lib._ptr(nodes), k, _lib._ptr(pi), _lib._ptr(pj),
            _lib._ptr(_opt(weight, np.float64)), *self._limits(rtol, itmax), _lib._ptr(R), _lib._ptr(volt),
            _lib._ptr(curr), 1 if accumulate else 0, _lib._ptr(iters), _lib._ptr(relres))
        self._raise(rc, raise_on_residual)
        return dict(R=self._io(R), volt=self._io(volt), curr=self._io(curr), iters=iters, relres=relres)

    def solve_region_pairs(self, sets, set_a, set_b, weight=None, want_volt=False, want_curr=False,
                           accumulate=False, rtol=None, itmax=None, raise_on_residual=True):
        """Focal-region pairs on this operator (cs_b200_solve_region_pairs): column c holds the rows of
        sets[set_a[c]] at 0 V and those of sets[set_b[c]] at 1 V, then scales to the reference's 1 A
        normalisation.  sets: list of 0-based row arrays (sorted, unique, non-empty).  Returns the dict
        of solve_pairs: R = 1 / flux, volt (0 on set_a, R on set_b), curr (every row of a set carries
        its merged node's current)."""
        ptr, rows = _csr(sets, np.int64)
        set_a = np.ascontiguousarray(set_a, dtype=np.int64)
        set_b = np.ascontiguousarray(set_b, dtype=np.int64)
        k = len(set_a)
        R = np.zeros(k, dtype=self.dtype)
        volt, curr, iters, relres = self._columns(k, want_volt, want_curr)
        rc = self._lib.cs_b200_solve_region_pairs(
            self._h, len(sets), _lib._ptr(ptr), _lib._ptr(rows), k, _lib._ptr(set_a), _lib._ptr(set_b),
            _lib._ptr(_opt(weight, np.float64)), *self._limits(rtol, itmax), _lib._ptr(R), _lib._ptr(volt),
            _lib._ptr(curr), 1 if accumulate else 0, _lib._ptr(iters), _lib._ptr(relres))
        self._raise(rc, raise_on_residual)
        return dict(R=self._io(R), volt=self._io(volt), curr=self._io(curr), iters=iters, relres=relres)

    def solve_grounded(self, sets, gset, sources, weight=None, want_volt=False, want_curr=False,
                       accumulate=False, rtol=None, itmax=None, raise_on_residual=True):
        """Advanced-mode columns with direct grounds on this operator (cs_b200_solve_grounded): column c
        holds the rows of sets[gset[c]] at 0 V and injects sources[c] = (rows, values) (0-based rows, none
        on the column's ground set).  sets: list of 0-based row arrays (sorted, unique, non-empty).
        Returns dict with src_volt (v at each column's first source row), volt, curr (every ground row is
        a node of its own), iters, relres."""
        ptr, rows, gset, sptr, srows, svals = _grounded_columns(sets, gset, sources)
        k = len(gset)
        sv = np.zeros(k, dtype=self.dtype)
        volt, curr, iters, relres = self._columns(k, want_volt, want_curr)
        rc = self._lib.cs_b200_solve_grounded(
            self._h, len(sets), _lib._ptr(ptr), _lib._ptr(rows), k, _lib._ptr(gset), _lib._ptr(sptr),
            _lib._ptr(srows), _lib._ptr(svals), _lib._ptr(_opt(weight, np.float64)), *self._limits(rtol, itmax),
            _lib._ptr(sv), _lib._ptr(volt), _lib._ptr(curr), 1 if accumulate else 0, _lib._ptr(iters),
            _lib._ptr(relres))
        self._raise(rc, raise_on_residual)
        return dict(src_volt=self._io(sv), volt=self._io(volt), curr=self._io(curr), iters=iters, relres=relres)

    def solve_advanced(self, sets, gset, sources, weight=None, want_volt=False, want_curr=False,
                       accumulate=False, rtol=None, itmax=None, raise_on_residual=True):
        """Raster advanced-mode columns on this operator and the finite grounds of the last set_grounds
        (cs_b200_solve_advanced): column c holds the rows of sets[gset[c]] at 0 V (gset[c] = -1: no direct
        grounds, which needs finite grounds on the handle) and injects sources[c] = (rows, values) (0-based
        rows, none on the column's ground set).  The node currents include the finite-ground currents.
        Returns dict with volt, curr, iters, relres."""
        ptr, rows, gset, sptr, srows, svals = _grounded_columns(sets, gset, sources)
        k = len(gset)
        volt, curr, iters, relres = self._columns(k, want_volt, want_curr)
        rc = self._lib.cs_b200_solve_advanced(
            self._h, len(sets), _lib._ptr(ptr), _lib._ptr(rows), k, _lib._ptr(gset), _lib._ptr(sptr),
            _lib._ptr(srows), _lib._ptr(svals), _lib._ptr(_opt(weight, np.float64)), *self._limits(rtol, itmax),
            _lib._ptr(volt), _lib._ptr(curr), 1 if accumulate else 0, _lib._ptr(iters), _lib._ptr(relres))
        self._raise(rc, raise_on_residual)
        return dict(volt=self._io(volt), curr=self._io(curr), iters=iters, relres=relres)

    def solve_advanced_network(self, sets, gset, sources, owner, want_volt=False, want_curr=False,
                               want_branch=False, rtol=None, itmax=None, raise_on_residual=True):
        """Network advanced mode on this whole-graph operator (cs_b200_solve_advanced_network): the columns of
        solve_advanced (sets, gset with -1 for finite grounds only, sources), owner (n,) the column whose
        component holds each row, or -1.  The columns' voltages are summed on the rows they own; returns dict
        with volt (n,), curr (n,) (node currents with the finite-ground currents) and branch (nb,) of that one
        vector under one 1e-8 cut over the graph (each None unless wanted), iters, relres."""
        ptr, rows, gset, sptr, srows, svals = _grounded_columns(sets, gset, sources)
        k = len(gset)
        owner = np.ascontiguousarray(owner, dtype=np.int64)
        assert len(owner) == self.n
        vec = lambda want, m: np.empty(m, dtype=self.dtype) if want else None
        volt, curr = vec(want_volt, self.n), vec(want_curr, self.n)
        branch = vec(want_branch, self._num_branches() if want_branch else 0)
        iters, relres = np.zeros(k, dtype=np.int64), np.zeros(k, dtype=np.float64)
        rc = self._lib.cs_b200_solve_advanced_network(
            self._h, len(sets), _lib._ptr(ptr), _lib._ptr(rows), k, _lib._ptr(gset), _lib._ptr(sptr),
            _lib._ptr(srows), _lib._ptr(svals), _lib._ptr(owner), *self._limits(rtol, itmax), _lib._ptr(volt),
            _lib._ptr(curr), _lib._ptr(branch), _lib._ptr(iters), _lib._ptr(relres))
        self._raise(rc, raise_on_residual)
        return dict(volt=self._io(volt), curr=self._io(curr), branch=self._io(branch), iters=iters, relres=relres)

    def solve_sources(self, columns, ref, probe=None, weight=None, want_volt=False, want_curr=False,
                      accumulate=False, rtol=None, itmax=None, raise_on_residual=True):
        """Batched solve with sparse right-hand sides, device-resident
        (cs_b200_solve_sources).  columns: list of (rows, values) per right-hand side
        (0-based rows); ref[c]: row whose voltage is subtracted (the ground).  Returns dict
        with probe_volt (k, len(probe))|None, volt, curr, iters, relres."""
        k = len(columns)
        colptr, rows = _csr([r for r, _ in columns], np.int64)
        _, vals = _csr([v for _, v in columns], np.float64)
        ref = np.ascontiguousarray(ref, dtype=np.int64)
        assert len(ref) == k and len(rows) == len(vals) == colptr[-1]
        pr = _opt(probe, np.int64)
        npr = 0 if pr is None else len(pr)
        pv = np.zeros((k, npr), dtype=self.dtype) if npr else None
        volt, curr, iters, relres = self._columns(k, want_volt, want_curr)
        rc = self._lib.cs_b200_solve_sources(self._h, k, _lib._ptr(colptr), _lib._ptr(rows), _lib._ptr(vals),
                                             _lib._ptr(ref), _lib._ptr(_opt(weight, np.float64)),
                                             *self._limits(rtol, itmax), npr, _lib._ptr(pr), _lib._ptr(pv),
                                             _lib._ptr(volt), _lib._ptr(curr), 1 if accumulate else 0,
                                             _lib._ptr(iters), _lib._ptr(relres))
        self._raise(rc, raise_on_residual)
        return dict(probe_volt=self._io(pv), volt=self._io(volt), curr=self._io(curr), iters=iters, relres=relres)

    def read_currents(self, want_max=True):
        cum = np.empty(self.n, dtype=self.dtype)
        mx = np.empty(self.n, dtype=self.dtype) if want_max else None
        rc = self._lib.cs_b200_read_currents(self._h, _lib._ptr(cum), _lib._ptr(mx))
        _lib.check(self._lib, self._h, rc)
        return cum, mx

    def reset_currents(self):
        _lib.check(self._lib, self._h, self._lib.cs_b200_reset_currents(self._h))

    def currents_device_ptrs(self):
        a, b = C.c_void_p(), C.c_void_p()
        _lib.check(self._lib, self._h, self._lib.cs_b200_currents_device_ptrs(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def _raise(self, rc, raise_on_residual):
        if rc == _lib.OK:
            return
        if rc == _lib.ERR_RESIDUAL:
            if raise_on_residual:
                msg = self._lib.cs_b200_last_error(self._h).decode()
                raise SolverResidualError(msg)
            return
        if rc == _lib.ERR_MAXITER:
            return  # results written; the residual gate decides (reference: itmax then gate)
        _lib.check(self._lib, self._h, rc)


def advanced_batch_bytes(ncell, itemsize, want_volt):
    """Device bytes cs_b200_solve_advanced_batch allocates per window of `ncell` cells: the three
    inputs, the current (and voltage) raster, five fp64 CG vectors and three int32 label arrays.
    cs_b200_solve_moving_windows sizes its batches by the same formula (want_volt False)."""
    return ncell * (3 * itemsize + 8 * (2 if want_volt else 1) + 5 * 8 + 3 * 4) + 32


def solve_advanced_batch(g, src, gnd, four_neighbors, device, rtol, itmax, want_volt=False):
    """One cs_b200_solve_advanced_batch call on stacks of equal-shape windows (nwin, nrows, ncols)
    of one float dtype (float32 or float64).  Returns dict with cur, volt (nwin, nrows, ncols)
    float64 | None, iters, relres (nwin,), rc (OK, ERR_RESIDUAL or ERR_MAXITER), first_failed
    (window index or -1) and msg; other failures raise."""
    lib = _lib.load()
    nwin, nr, nc = g.shape
    dt = _lib.dtype_code(g.dtype)
    # window-major, column-major inside a window: (nwin, ncols, nrows) in C order
    g_, s_, gnd_ = (np.ascontiguousarray(np.asarray(a, dtype=g.dtype).transpose(0, 2, 1)) for a in (g, src, gnd))
    cur = np.empty((nwin, nc, nr), dtype=np.float64)
    volt = np.empty((nwin, nc, nr), dtype=np.float64) if want_volt else None
    iters = np.zeros(nwin, dtype=np.int64)
    relres = np.zeros(nwin, dtype=np.float64)
    bad = C.c_int64(-1)
    rc = lib.cs_b200_solve_advanced_batch(nwin, nr, nc, _lib._ptr(g_), _lib._ptr(s_), _lib._ptr(gnd_), dt,
                                          1 if four_neighbors else 0, device, float(rtol), int(itmax),
                                          _lib._ptr(cur), _lib._ptr(volt), _lib._ptr(iters), _lib._ptr(relres),
                                          C.byref(bad))
    msg = ""
    if rc not in (_lib.OK, _lib.ERR_RESIDUAL, _lib.ERR_MAXITER):
        _lib.check(lib, None, rc)
    if rc != _lib.OK:
        msg = lib.cs_b200_last_error(None).decode()
    return dict(cur=cur.transpose(0, 2, 1), volt=None if volt is None else volt.transpose(0, 2, 1),
                iters=iters, relres=relres, rc=rc, first_failed=int(bad.value), msg=msg)


def solve_moving_windows(g, src, target_rows, target_cols, radius, circular, source_scale, ground, four_neighbors,
                         device, rtol, itmax, max_batch_bytes):
    """One cs_b200_solve_moving_windows call: landscape rasters g / src (nrows, ncols) of one float dtype
    (float32 or float64), targets (nwin,) each, source_scale / ground (nwin,) float64 or None (all 1 / all
    Inf).  Windows are batched under max_batch_bytes at advanced_batch_bytes(ncell, itemsize, False) each.
    Returns dict with cum (nrows, ncols) float64, iters, relres (nwin,), rc (OK, ERR_RESIDUAL or
    ERR_MAXITER), first_failed (global window index or -1) and msg; other failures raise."""
    lib = _lib.load()
    nr, nc = g.shape
    dt = _lib.dtype_code(g.dtype)
    # column-major rasters: (ncols, nrows) in C order
    g_, s_ = (np.ascontiguousarray(np.asarray(a, dtype=g.dtype).T) for a in (g, src))
    tr, tc = (np.ascontiguousarray(t, dtype=np.int64) for t in (target_rows, target_cols))
    nwin = len(tr)
    cum = np.empty((nc, nr), dtype=np.float64)
    iters = np.zeros(nwin, dtype=np.int64)
    relres = np.zeros(nwin, dtype=np.float64)
    bad = C.c_int64(-1)
    rc = lib.cs_b200_solve_moving_windows(nr, nc, _lib._ptr(g_), _lib._ptr(s_), dt, nwin, _lib._ptr(tr),
                                          _lib._ptr(tc), int(radius), 1 if circular else 0,
                                          _lib._ptr(_opt(source_scale, np.float64)), _lib._ptr(_opt(ground, np.float64)),
                                          1 if four_neighbors else 0, device, float(rtol), int(itmax),
                                          int(max_batch_bytes), _lib._ptr(cum), _lib._ptr(iters), _lib._ptr(relres),
                                          C.byref(bad))
    msg = ""
    if rc not in (_lib.OK, _lib.ERR_RESIDUAL, _lib.ERR_MAXITER):
        _lib.check(lib, None, rc)
    if rc != _lib.OK:
        msg = lib.cs_b200_last_error(None).decode()
    return dict(cum=np.ascontiguousarray(cum.T), iters=iters, relres=relres, rc=rc, first_failed=int(bad.value),
                msg=msg)


def omniscape_candidates(nrows, ncols, block_size):
    """Number of Omniscape block centres (block_size // 2 + i * block_size, ...) inside the landscape."""
    h = (block_size - 1) // 2
    return ((nrows - 1 - h) // block_size + 1 if nrows > h else 0) * ((ncols - 1 - h) // block_size + 1
                                                                      if ncols > h else 0)


def solve_omniscape(g, src, radius, block_size, source_threshold, flow_potential, four_neighbors, device, rtol,
                    itmax, max_batch_bytes):
    """One cs_b200_solve_omniscape call: landscape rasters g / src (nrows, ncols) of one float dtype.
    Returns dict with cum, fp, normalized (nrows, ncols) float64 (fp / normalized None without
    flow_potential), targets (nt, 2) int64, amps, scale, iters, relres, fp_iters, fp_relres (nt,), rc (OK,
    ERR_RESIDUAL or ERR_MAXITER), first_failed (target index or -1) and msg; other failures raise."""
    lib = _lib.load()
    nr, nc = g.shape
    dt = _lib.dtype_code(g.dtype)
    g_, s_ = (np.ascontiguousarray(np.asarray(a, dtype=g.dtype).T) for a in (g, src))
    cap = omniscape_candidates(nr, nc, int(block_size))
    cum = np.empty((nc, nr), dtype=np.float64)
    fp, norm = (np.empty((nc, nr), dtype=np.float64) if flow_potential else None for _ in range(2))
    rows, cols, iters, fp_iters = (np.zeros(cap, dtype=np.int64) for _ in range(4))
    amps, scale, relres, fp_relres = (np.zeros(cap, dtype=np.float64) for _ in range(4))
    nt, bad = C.c_int64(0), C.c_int64(-1)
    rc = lib.cs_b200_solve_omniscape(nr, nc, _lib._ptr(g_), _lib._ptr(s_), dt, int(radius), int(block_size),
                                     float(source_threshold), 1 if flow_potential else 0, 1 if four_neighbors else 0,
                                     device, float(rtol), int(itmax), int(max_batch_bytes), _lib._ptr(cum),
                                     _lib._ptr(fp), _lib._ptr(norm), cap, C.byref(nt), _lib._ptr(rows),
                                     _lib._ptr(cols), _lib._ptr(amps), _lib._ptr(scale), _lib._ptr(iters),
                                     _lib._ptr(relres), _lib._ptr(fp_iters), _lib._ptr(fp_relres), C.byref(bad))
    msg = ""
    if rc not in (_lib.OK, _lib.ERR_RESIDUAL, _lib.ERR_MAXITER):
        _lib.check(lib, None, rc)
    if rc != _lib.OK:
        msg = lib.cs_b200_last_error(None).decode()
    n = nt.value
    t = lambda a: None if a is None else np.ascontiguousarray(a.T)
    return dict(cum=t(cum), fp=t(fp), normalized=t(norm), targets=np.stack([rows[:n], cols[:n]], 1),
                amps=amps[:n], scale=scale[:n], iters=iters[:n], relres=relres[:n],
                fp_iters=fp_iters[:n] if flow_potential else None, fp_relres=fp_relres[:n] if flow_potential else None,
                rc=rc, first_failed=int(bad.value), msg=msg)


# ---------------------------------------------------------------------------
# the three plug-in hooks
# ---------------------------------------------------------------------------
def construct_cholesky_factor(matrix, solver: CUDASolver, **kw) -> B200Factor:
    """Hook #1 (src/core.jl:379,519-523): once per connected component."""
    return B200Factor(matrix, solver, **kw)


def construct_raster_factor(cellmap, polymap, solver: CUDASolver, four_neighbors=False, avg_res=False,
                            log_transform=False):
    """The whole-raster operator of a pairwise, focal-region, one-to-all or advanced-mode job and its node map
    (1-based, 0 = none): B200Factor.from_raster_polygons.  Not one of the three hooks: those drivers need
    the handle's column entries (cs_b200_solve_region_pairs / _grounded / _advanced), which the Solver
    interface has no method for."""
    return B200Factor.from_raster_polygons(cellmap, polymap, solver, four_neighbors=four_neighbors,
                                           avg_res=avg_res, log_transform=log_transform)


def solve_linear_system(factor: B200Factor, matrix, rhs):
    """Hook #2 (src/core.jl:463,646-653): n x k -> n x k; raises if any column's
    true relative residual is >= 1e-4, like every reference solver."""
    lhs, _, _ = factor.solve_rhs(rhs)
    return lhs


def multiple_solve(solver: CUDASolver, matrix, sources):
    """Hook #3 (src/raster/advanced.jl:307-333): factor + one solve + the
    reference's `@assert residual < 1e-4`."""
    with construct_cholesky_factor(matrix, solver) as factor:
        volt = solve_linear_system(factor, matrix, np.asarray(sources))
    return volt

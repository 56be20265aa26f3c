"""Device-side setup (circuitscape_b200/csrc/setup_device.cu) against the round-1 host setup
(amg_host.hpp / win_host.hpp) and against SciPy: hierarchy operators, Galerkin identities, window
records on every operator shape, the 1-based Int64 boundary Julia uses, and a non-Python caller.
Needs an H100: `pytest -m gpu`."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

import circuitscape_b200 as cb
from circuitscape_b200 import _lib, graph
from oracle import circuitscape_oracle as co

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def holey(nr, nc, seed, holes=0.05, sigma=1.0):
    rng = np.random.default_rng(seed)
    g = 1.0 / np.exp(rng.normal(0.0, sigma, size=(nr, nc)))
    g[rng.random((nr, nc)) < holes] = 0.0
    nodemap = graph.construct_node_map(g, None)
    G = graph.laplacian(graph.construct_graph(g, nodemap, False, False))
    big = max(graph.connected_components(G), key=len) - 1
    return G[big][:, big].tocsr()


@pytest.mark.parametrize("kind", ["uniform", "holes"])
def test_hierarchy_device_matches_host(kind):
    """Same levels from both builders: shapes, patterns, values (fp64 cycle so nothing is rounded),
    R = P^T exactly, Galerkin coarse operators, Jacobi weights."""
    A = graph.synthetic_raster_laplacian(230, 170, seed=5)[0] if kind == "uniform" else holey(220, 160, 3)
    lv = {}
    for setup in ("host", "device"):
        with cb.B200Factor(A, cb.CUDASolver(setup=setup, mixed=False, window="on")) as f:
            lv[setup] = f.levels()
    H, D = lv["host"], lv["device"]
    assert len(H) == len(D) >= 3
    for l, (h, d) in enumerate(zip(H, D)):
        assert abs(h["omega"] - d["omega"]) <= 1e-12 * h["omega"], l
        for name in ("A", "P", "R"):
            if h[name] is None:
                assert d[name] is None
                continue
            assert h[name].shape == d[name].shape and h[name].nnz == d[name].nnz, (l, name)
            assert np.array_equal(h[name].indptr, d[name].indptr) and np.array_equal(h[name].indices, d[name].indices)
            scale = np.abs(h[name].data).max()
            assert np.abs(h[name].data - d[name].data).max() <= 1e-12 * scale, (l, name)
            assert d[name + "_windowed"] == h[name + "_windowed"], (l, name)
        if d["P"] is not None:
            assert abs(d["R"] - d["P"].T).max() == 0.0
            Ac = (d["R"] @ d["A"] @ d["P"]).tocsr()
            assert abs(Ac - D[l + 1]["A"]).max() <= 1e-12 * abs(Ac).max()
    assert D[-1]["A"].shape[0] <= 200


@pytest.mark.parametrize("mixed", [True, False])
def test_device_setup_same_iterations_and_resistances(mixed):
    A = holey(300, 260, 11, holes=0.08, sigma=1.5)
    nodes = graph.focal_nodes(A.shape[0], 6, seed=7)
    src, dst = graph.all_pairs(nodes)
    res = {}
    for setup in ("host", "device"):
        with cb.B200Factor(A, cb.CUDASolver(setup=setup, mixed=mixed)) as f:
            res[setup] = f.solve_pairs(src, dst, accumulate=True), f.read_currents()[0]
    (oh, ch), (od, cd) = res["host"], res["device"]
    assert np.abs(oh["iters"] - od["iters"]).max() <= 1
    assert np.abs(oh["R"] - od["R"]).max() <= 2e-6 * np.abs(oh["R"]).max()
    assert np.abs(ch - cd).max() <= 1e-5 * np.abs(ch).max()
    Vref = co.solve_pairs_direct(A, src, dst)
    Rref = Vref[dst, np.arange(len(src))]
    assert np.abs(od["R"] - Rref).max() <= 1e-6 * np.abs(Rref).max()


@pytest.mark.parametrize("shape", [(3, 3), (9, 40), (128, 1), (1, 700), (141, 143), (400, 90)])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_windows_built_on_device_spmm(shape, dtype):
    """Row blocks (chunk-local greedy walk) + window records packed on the device, every panel width,
    ragged holes, tiny and degenerate rasters."""
    A = holey(*shape, seed=shape[0] + shape[1], holes=0.12) if min(shape) > 1 else \
        graph.synthetic_raster_laplacian(*shape, seed=2)[0].tocsr()
    n = A.shape[0]
    prec = "single" if dtype == np.float32 else "double"
    rng = np.random.default_rng(4)
    with cb.B200Factor(A, cb.CUDASolver(precision=prec, f32_compute=True, window="on", precond="jacobi",
                                        setup="device")) as f:
        for k in (1, 2, 4, 8):
            X = rng.standard_normal((n, k))
            Y = f.spmm(X)
            ref = A.astype(dtype) @ X.astype(dtype)
            tol = (1e-13 if dtype == np.float64 else 3e-6) * np.abs(A).sum(axis=1).max() * np.abs(X).max()
            assert np.abs(Y - ref).max() <= tol, (k, shape)


def test_transfer_operator_windows_through_the_cycle():
    """P and R (rectangular, wide rows) get device-built windows above 20 000 rows; a wrong record
    would break the symmetry of the cycle: iteration counts must match the plain-kernel cycle."""
    A = graph.synthetic_raster_laplacian(330, 310, seed=8)[0]
    nodes = graph.focal_nodes(A.shape[0], 5, seed=7)
    src, dst = graph.all_pairs(nodes)
    out = {}
    for window in ("auto", "off"):
        with cb.B200Factor(A, cb.CUDASolver(setup="device", window=window)) as f:
            out[window] = f.solve_pairs(src, dst)
            if window == "auto":
                lv = f.levels()
                assert lv[0]["P_windowed"] and lv[0]["R_windowed"] and lv[0]["A_windowed"]
    assert np.array_equal(out["auto"]["iters"], out["off"]["iters"])
    assert np.abs(out["auto"]["R"] - out["off"]["R"]).max() <= 1e-9 * np.abs(out["off"]["R"]).max()


def _grounded_cg(A, src, dst):
    """R of the pairs from SciPy CG on the grounded system (last node removed), Jacobi-preconditioned:
    a reference that needs no factorisation (power-law graphs fill in badly under LU)."""
    import scipy.sparse.linalg as spla
    n = A.shape[0]
    Ag = A[:n - 1][:, :n - 1].tocsr()
    d = Ag.diagonal()
    M = spla.LinearOperator(Ag.shape, matvec=lambda x: x / d)
    out = []
    for s_, d_ in zip(src, dst):
        b = np.zeros(n); b[s_] = -1.0; b[d_] = 1.0
        x, info = spla.cg(Ag, b[:n - 1], rtol=1e-12, atol=0.0, maxiter=5000, M=M)
        assert info == 0
        v = np.append(x, 0.0)
        out.append(v[d_] - v[s_])
    return np.array(out)


def test_power_law_network_device_setup():
    """Hub rows + densifying Galerkin products: the product budget stops coarsening on the device as
    the nnz budget does on the host; whatever hierarchy is left must solve the system."""
    A = graph.power_law_laplacian(40000, m=5, seed=11)
    nodes = graph.focal_nodes(A.shape[0], 5, seed=3)
    src, dst = graph.all_pairs(nodes)
    with cb.B200Factor(A, cb.CUDASolver(setup="device")) as f:
        out = f.solve_pairs(src, dst)
        nlev = len(f.levels())
    Rref = _grounded_cg(A, src, dst)
    assert out["relres"].max() < 1e-4
    assert np.abs(out["R"] - Rref).max() <= 1e-6 * np.abs(Rref).max()
    assert nlev <= 12


@pytest.mark.parametrize("setup", ["device", "host"])
@pytest.mark.parametrize("bits,base", [(64, 1), (32, 1), (64, 0)])
def test_create_with_julia_style_indices(setup, bits, base):
    """cs_b200_create with 1-based Int64 colptr / rowval (a SparseMatrixCSC{Float64,Int64} as the
    `ccall` of INTEGRATION.md passes it) gives the resistances of the 0-based int32 path."""
    A = holey(120, 100, 21).tocsr()
    A.sort_indices()
    n = A.shape[0]
    nodes = graph.focal_nodes(n, 4, seed=7)
    src, dst = graph.all_pairs(nodes)
    solver = cb.CUDASolver(setup=setup)
    with cb.B200Factor(A, solver) as f0:
        R0 = f0.solve_pairs(src, dst)["R"]
    lib = _lib.load()
    it = np.int64 if bits == 64 else np.int32
    rp = (A.indptr.astype(it) + base)
    ci = (A.indices.astype(it) + base)
    va = np.ascontiguousarray(A.data, dtype=np.float64)
    h = C.c_void_p()
    opts = cb.B200Factor._opts(solver)
    rc = lib.cs_b200_create(n, A.nnz, _lib._ptr(rp), _lib._ptr(ci), _lib._ptr(va), bits, base, _lib.F64, 0,
                            C.byref(opts), C.byref(h))
    _lib.check(lib, None, rc)
    try:
        k = len(src)
        s64, d64 = np.ascontiguousarray(src, dtype=np.int64), np.ascontiguousarray(dst, dtype=np.int64)
        R = np.zeros(k)
        iters = np.zeros(k, dtype=np.int64)
        rr = np.zeros(k)
        rc = lib.cs_b200_solve_pairs(h, k, _lib._ptr(s64), _lib._ptr(d64), None, 1e-6, 100000, _lib._ptr(R), None,
                                     None, 0, _lib._ptr(iters), _lib._ptr(rr))
        _lib.check(lib, h, rc)
    finally:
        lib.cs_b200_destroy(h)
    assert np.array_equal(R, R0)
    # a rowptr that does not span [base, nnz + base] is refused, not read out of bounds; a 64-bit end that is
    # nnz + base only once narrowed to 32 bits is refused by both builders too
    for off in ([1, 1 << 32] if bits == 64 else [1]):
        bad = rp.copy(); bad[-1] += off
        h2 = C.c_void_p()
        rc = lib.cs_b200_create(n, A.nnz, _lib._ptr(bad), _lib._ptr(ci), _lib._ptr(va), bits, base, _lib.F64, 0,
                                C.byref(opts), C.byref(h2))
        assert rc == _lib.ERR_ARG and not h2.value
        assert b"does not span" in lib.cs_b200_last_error(None)


def test_from_raster_and_from_device_use_device_setup():
    rng = np.random.default_rng(9)
    g = 1.0 / rng.uniform(1.0, 10.0, size=(260, 240))
    A = graph.stencil_laplacian_from_conductance(g)
    nodes = graph.focal_nodes(A.shape[0], 4, seed=7)
    src, dst = graph.all_pairs(nodes)
    with cb.B200Factor(A, cb.CUDASolver(setup="host")) as f:
        ref = f.solve_pairs(src, dst)
    with cb.B200Factor.from_raster(g, cb.CUDASolver(setup="device")) as f:
        out = f.solve_pairs(src, dst)
        assert len(f.levels()) >= 3
    assert np.abs(out["iters"] - ref["iters"]).max() <= 1
    assert np.abs(out["R"] - ref["R"]).max() <= 2e-6 * np.abs(ref["R"]).max()


def test_c_program_links_and_solves(tmp_path):
    """A plain C caller (tests/c_caller/caller.c): create with 1-based Int64 CSC, solve_rhs on a
    column-major n x 2 matrix, destroy -- the call sequence of the Julia glue without Python."""
    exe = str(tmp_path / "caller")
    libdir = os.path.join(ROOT, "circuitscape_b200", "lib")
    subprocess.check_call(["gcc", "-O2", "-I", os.path.join(ROOT, "include"), "-o", exe,
                           os.path.join(ROOT, "tests", "c_caller", "caller.c"), "-L", libdir, "-lcsb200", "-lm",
                           f"-Wl,-rpath,{libdir}"])
    for args in (["1", "60"], ["170", "150"]):
        r = subprocess.run([exe] + args, capture_output=True, text=True, timeout=120)
        assert r.returncode == 0, (args, r.stdout, r.stderr)
        assert "R0=" in r.stdout


# ---- stencil (DIA) form: SURVEY.md 8f rank 2 ------------------------------------------------------
def _check_stencil_spmm(A, dtype):
    n = A.shape[0]
    prec = "single" if dtype == np.float32 else "double"
    rng = np.random.default_rng(4)
    with cb.B200Factor(A, cb.CUDASolver(precision=prec, f32_compute=True, precond="jacobi", stencil="on")) as f:
        assert f.operator_form() == "stencil"
        for k in (1, 2, 4, 8):
            X = rng.standard_normal((n, k))
            Y = f.spmm(X)
            ref = A.astype(dtype) @ X.astype(dtype)
            tol = (1e-13 if dtype == np.float64 else 3e-6) * np.abs(A).sum(axis=1).max() * np.abs(X).max()
            assert np.abs(Y - ref).max() <= tol, k
        y, _ = f.spmv(X[:, 0])
        assert np.abs(y - A.astype(dtype) @ X[:, 0].astype(dtype)).max() <= tol


@pytest.mark.parametrize("four", [False, True])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_stencil_form_spmm(dtype, four):
    """Full raster (every cell a node): the operator is stored as 9 diagonals and multiplied by
    k_stencil; every panel width against SciPy, first / last raster columns and rows included."""
    A = graph.synthetic_raster_laplacian(233, 171, seed=5, four_neighbors=four)[0].tocsr()
    _check_stencil_spmm(A, dtype)


@pytest.mark.parametrize("four", [False, True])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("shape", [(3, 50), (20, 37), (65, 43), (257, 29), "ragged"])
def test_stencil_form_spmm_tile_edges(shape, dtype, four):
    """The same below 20 000 rows (stencil = on): rasters shorter than one tile (3, 20 rows), not a
    multiple of it (65, 257), and a last raster column that ends early (NODATA below row 120: still a
    stencil form)."""
    if shape == "ragged":
        g = 1.0 / np.random.default_rng(5).uniform(1.0, 10.0, size=(301, 97))
        g[120:, 96] = 0.0
        A = graph.laplacian(graph.construct_graph(g, graph.construct_node_map(g), False, four))
    else:
        A = graph.synthetic_raster_laplacian(*shape, seed=5, four_neighbors=four)[0].tocsr()
    _check_stencil_spmm(A, dtype)


@pytest.mark.parametrize("mixed", [True, False])
def test_stencil_form_solve_matches_csr_kernels(mixed):
    """Same iteration counts and resistances with the stencil kernels (level 0 and the regular coarse
    grids that qualify) as with the windowed / plain CSR kernels; a raster with NODATA holes has no
    stencil form and silently keeps the CSR path."""
    A = graph.synthetic_raster_laplacian(260, 240, seed=9)[0]
    nodes = graph.focal_nodes(A.shape[0], 6, seed=7)
    src, dst = graph.all_pairs(nodes)
    out = {}
    for st in ("auto", "off"):
        with cb.B200Factor(A, cb.CUDASolver(stencil=st, mixed=mixed)) as f:
            out[st] = f.solve_pairs(src, dst, accumulate=True), f.read_currents()[0]
            lv = f.levels()
            assert lv[0]["A_stencil"] == (st == "auto")
    (a, ca), (b, cb_) = out["auto"], out["off"]
    assert np.array_equal(a["iters"], b["iters"])
    assert np.abs(a["R"] - b["R"]).max() <= 1e-9 * np.abs(b["R"]).max()
    assert np.abs(ca - cb_).max() <= 1e-8 * np.abs(cb_).max()
    Vref = co.solve_pairs_direct(A, src[:3], dst[:3])
    assert np.abs(a["R"][:3] - Vref[dst[:3], np.arange(3)]).max() <= 1e-6 * a["R"][:3].max()
    H = holey(200, 180, 5, holes=0.03)
    with cb.B200Factor(H, cb.CUDASolver(stencil="on")) as f:
        assert not f.levels()[0]["A_stencil"]
        nodes = graph.focal_nodes(H.shape[0], 3, seed=7)
        s2, d2 = graph.all_pairs(nodes)
        o = f.solve_pairs(s2, d2)
    V2 = co.solve_pairs_direct(H, s2, d2)
    assert np.abs(o["R"] - V2[d2, np.arange(len(s2))]).max() <= 1e-6 * o["R"].max()

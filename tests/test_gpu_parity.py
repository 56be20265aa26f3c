"""Parity of the CUDA path (through the C ABI) against the CPU oracle and the
reference's golden vectors.  Needs an H100: `pytest -m gpu`.

Tolerances (fp64): effective resistances 1e-6 relative (BASELINE.json north_star),
voltages max|dv|/R <= 1e-5, maps sum(d^2) < 1e-6 (test/test_utils.jl:196).
fp32: resistances 1e-3 relative (the reference codes 1e-4 *absolute* on its tiny
cases, test/test_utils.jl:73,167 -- never exercised upstream)."""
import numpy as np
import pytest
import scipy.sparse as sp

import circuitscape_b200 as cb
from circuitscape_b200 import graph
from oracle import circuitscape_oracle as co

from . import cases

pytestmark = pytest.mark.gpu


def holey_raster(nr, nc, seed, holes=0.05):
    rng = np.random.default_rng(seed)
    g = 1.0 / np.exp(rng.normal(0.0, 1.0, size=(nr, nc)))
    g[rng.random((nr, nc)) < holes] = 0.0
    nodemap = graph.construct_node_map(g, None)
    G = graph.laplacian(graph.construct_graph(g, nodemap, False, False))
    cc = graph.connected_components(G)
    big = max(cc, key=len) - 1
    return G[big][:, big].tocsr()


@pytest.mark.parametrize("dtype,tol", [(np.float64, 1e-13), (np.float32, 2e-6)])
@pytest.mark.parametrize("shape", [(3, 3), (37, 53), (300, 200)])
def test_spmv_matches_scipy(dtype, tol, shape):
    A = holey_raster(*shape, seed=1)
    x = np.random.default_rng(2).standard_normal(A.shape[0])
    with cb.B200Factor(A, cb.CUDASolver(precision="single" if dtype == np.float32 else "double",
                                        f32_compute=True)) as f:
        y, _ = f.spmv(x)
    ref = A.astype(dtype) @ x.astype(dtype)
    assert np.abs(y - ref).max() <= tol * np.abs(A).sum(axis=1).max() * np.abs(x).max()


def test_spmv_long_rows():
    """hub rows longer than the shared-memory row block (polygon / power-law nodes)."""
    rng = np.random.default_rng(3)
    n = 20000
    rows = np.concatenate([np.zeros(9000, dtype=int), np.full(3000, 7), rng.integers(0, n, 40000)])
    cols = np.concatenate([rng.choice(np.arange(1, n), 9000, replace=False),
                           rng.choice(np.arange(8, n), 3000, replace=False), rng.integers(0, n, 40000)])
    keep = rows != cols
    W = sp.coo_matrix((rng.random(keep.sum()) + 0.1, (rows[keep], cols[keep])), shape=(n, n)).tocsr()
    A = graph.laplacian(W + W.T)
    x = rng.standard_normal(n)
    with cb.B200Factor(A, cb.CUDASolver()) as f:
        y, _ = f.spmv(x)
    ref = A @ x
    assert np.abs(y - ref).max() <= 1e-12 * np.abs(ref).max()


@pytest.mark.parametrize("dtype,tol", [(np.float64, 1e-13), (np.float32, 2e-6)])
@pytest.mark.parametrize("window", ["on", "off"])
def test_spmv_window_modes(dtype, tol, window):
    """TMA-staged windowed kernel vs plain direct-gather kernel on the same operator,
    incl. NODATA holes (ragged segments) and a short last block."""
    A = holey_raster(123, 77, seed=4, holes=0.15)
    x = np.random.default_rng(2).standard_normal(A.shape[0])
    prec = "single" if dtype == np.float32 else "double"
    with cb.B200Factor(A, cb.CUDASolver(precision=prec, window=window, f32_compute=True)) as f:
        y, _ = f.spmv(x)
    ref = A.astype(dtype) @ x.astype(dtype)
    assert np.abs(y - ref).max() <= tol * np.abs(A).sum(axis=1).max() * np.abs(x).max()


@pytest.mark.parametrize("window", ["on", "off"])
@pytest.mark.parametrize("precond", ["jacobi", "amg"])
def test_window_modes_solve(window, precond):
    A = holey_raster(90, 70, seed=6)
    nodes = graph.focal_nodes(A.shape[0], 6, seed=7)
    src, dst = graph.all_pairs(nodes)
    Vref = co.solve_pairs_direct(A, src, dst)
    Rref = Vref[dst, np.arange(len(src))]
    with cb.B200Factor(A, cb.CUDASolver(precond=precond, window=window)) as f:
        out = f.solve_pairs(src, dst, want_volt=True)
    assert (np.abs(out["R"] - Rref) / Rref).max() < 1e-6
    assert (np.abs(out["volt"] - Vref).max(axis=0) / Rref).max() < 1e-5


@pytest.mark.parametrize("precond", ["jacobi", "amg"])
@pytest.mark.parametrize("pw", [1, 2, 4, 8])
def test_pairs_match_oracle_fp64(pw, precond):
    A = holey_raster(60, 45, seed=5)
    n = A.shape[0]
    nodes = graph.focal_nodes(n, 6, seed=7)
    src, dst = graph.all_pairs(nodes)           # 15 pairs -> panels 8+4+2+1 at pw = 8
    Vref = co.solve_pairs_direct(A, src, dst)
    Rref = Vref[dst, np.arange(len(src))]
    with cb.B200Factor(A, cb.CUDASolver(panel_width=pw, precond=precond)) as f:
        out = f.solve_pairs(src, dst, want_volt=True, want_curr=True, accumulate=True)
        cum, mx = f.read_currents()
    assert np.abs(out["R"] - Rref).max() / Rref.max() < 1e-6
    assert (np.abs(out["R"] - Rref) / Rref).max() < 1e-6
    assert (np.abs(out["volt"] - Vref).max(axis=0) / Rref).max() < 1e-5
    assert out["relres"].max() < 1e-4 and out["iters"].min() > 0
    cur_ref = np.column_stack([co.get_node_currents(A, Vref[:, c]) for c in range(len(src))])
    assert np.abs(out["curr"] - cur_ref).max() < 1e-5
    assert np.abs(cum - cur_ref.sum(axis=1)).max() < 1e-4
    assert np.abs(mx - cur_ref.max(axis=1)).max() < 1e-5


@pytest.mark.parametrize("precond", ["jacobi", "amg"])
def test_pairs_fp32(precond):
    A = holey_raster(60, 45, seed=5)
    nodes = graph.focal_nodes(A.shape[0], 5, seed=7)
    src, dst = graph.all_pairs(nodes)
    Vref = co.solve_pairs_direct(A, src, dst)
    Rref = Vref[dst, np.arange(len(src))]
    with cb.B200Factor(A, cb.CUDASolver(precision="single", precond=precond, f32_compute=True)) as f:
        out = f.solve_pairs(src, dst, want_volt=True)
    assert out["R"].dtype == np.float32
    assert (np.abs(out["R"] - Rref) / Rref).max() < 1e-3
    assert out["relres"].max() < 1e-4
    # default for precision = single: Float32 at the boundary, fp64 on the device
    with cb.B200Factor(A.astype(np.float32), cb.CUDASolver(precision="single", precond=precond)) as f:
        out = f.solve_pairs(src, dst, want_volt=True)
    assert out["R"].dtype == np.float32 and out["volt"].dtype == np.float32
    assert (np.abs(out["R"] - Rref) / Rref).max() < 2e-6      # only the fp32 rounding of G and R
    assert out["relres"].max() < 1e-5


def test_amg_cuts_iterations_and_agrees_with_jacobi():
    A = holey_raster(200, 150, seed=21)
    nodes = graph.focal_nodes(A.shape[0], 5, seed=3)
    src, dst = graph.all_pairs(nodes)
    with cb.B200Factor(A, cb.CUDASolver(precond="jacobi")) as f:
        oj = f.solve_pairs(src, dst)
    with cb.B200Factor(A, cb.CUDASolver(precond="amg")) as f:
        oa = f.solve_pairs(src, dst, want_curr=True, accumulate=True)
        oa2 = f.solve_pairs(src, dst)
    assert (np.abs(oa["R"] - oj["R"]) / oj["R"]).max() < 1e-6
    assert oa["iters"].max() * 8 < oj["iters"].min(), (oa["iters"], oj["iters"])
    assert oa["relres"].max() < 1e-4
    assert np.array_equal(oa["R"], oa2["R"]), "AMG path must be bit-reproducible"


def test_mixed_precision_cycle_matches_fp64_cycle():
    """fp32 V-cycle inside fp64 CG (default) vs the all-fp64 cycle: same answers to the
    solver tolerance, comparable iteration counts, fp64-level residual gate."""
    A = holey_raster(220, 160, seed=31)
    nodes = graph.focal_nodes(A.shape[0], 5, seed=3)
    src, dst = graph.all_pairs(nodes)
    Vref = co.solve_pairs_direct(A, src, dst)
    Rref = Vref[dst, np.arange(len(src))]
    res = {}
    for mixed in (True, False):
        with cb.B200Factor(A, cb.CUDASolver(precond="amg", mixed=mixed, window="on")) as f:
            res[mixed] = f.solve_pairs(src, dst, want_volt=True)
    for mixed, o in res.items():
        assert (np.abs(o["R"] - Rref) / Rref).max() < 1e-6, mixed
        assert (np.abs(o["volt"] - Vref).max(axis=0) / Rref).max() < 1e-5, mixed
        assert o["relres"].max() < 1e-5, mixed
    assert res[True]["iters"].max() <= res[False]["iters"].max() + 4


def test_amg_irregular_graph_with_hub():
    """network-style graph (config 5 shape): power-law-ish degrees incl. a hub row
    longer than one shared-memory row block, advanced-mode SPD system."""
    rng = np.random.default_rng(5)
    n = 3000          # (a random graph is an expander: the oracle's sparse LU fills in ~n^2)
    m = 4
    rows = np.repeat(np.arange(m, n), m)
    cols = (rng.random(rows.size) ** 2 * rows).astype(np.int64)      # preferential-ish
    hub = np.arange(1, 2501)
    rows = np.concatenate([rows, np.zeros(hub.size, dtype=np.int64)])
    cols = np.concatenate([cols, hub])
    keep = rows != cols
    W = sp.coo_matrix((rng.uniform(0.1, 1.0, keep.sum()), (rows[keep], cols[keep])), shape=(n, n)).tocsr()
    A = graph.laplacian(W + W.T)
    cc = graph.connected_components(A)
    big = max(cc, key=len) - 1
    A = A[big][:, big].tocsr()
    n = A.shape[0]
    gnd = np.zeros(n); gnd[n // 2] = 1.0
    M = (A + sp.diags(gnd)).tocsr()
    b = np.zeros(n); b[rng.choice(n, 16, replace=False)] = 1.0
    import scipy.sparse.linalg as spla
    xref = spla.splu(M.tocsc()).solve(b)
    for precond in ("jacobi", "amg"):
        with cb.B200Factor(M, cb.CUDASolver(precond=precond, rtol=1e-9)) as f:
            x, iters, relres = f.solve_rhs(b)
        assert np.abs(x - xref).max() / np.abs(xref).max() < 1e-6, precond
        assert relres.max() < 1e-6


def test_weights_and_determinism():
    A = holey_raster(40, 40, seed=9)
    nodes = graph.focal_nodes(A.shape[0], 5, seed=1)
    src, dst = graph.all_pairs(nodes)
    w = np.arange(1, len(src) + 1, dtype=float)
    outs = []
    for _ in range(2):
        with cb.B200Factor(A, cb.CUDASolver()) as f:
            o = f.solve_pairs(src, dst, weight=w, want_curr=True, accumulate=True)
            cum, _ = f.read_currents()
        outs.append((o["R"].copy(), cum.copy(), o["curr"].copy()))
    assert np.array_equal(outs[0][0], outs[1][0]), "resistances must be bit-reproducible"
    assert np.array_equal(outs[0][1], outs[1][1])
    assert np.abs(outs[0][1] - outs[0][2] @ w).max() < 1e-9 * np.abs(outs[0][1]).max()


@pytest.mark.parametrize("precond", ["jacobi", "amg"])
def test_graph_and_plain_launch_agree(precond):
    """device-side WHILE-graph loop, host-polled graph chunks and plain launches run the
    same iterations: identical resistances and identical per-pair iteration counts."""
    A = holey_raster(50, 50, seed=11)
    nodes = graph.focal_nodes(A.shape[0], 4, seed=2)
    src, dst = graph.all_pairs(nodes)
    r, it = [], []
    for ug in (True, "chunk", False):
        with cb.B200Factor(A, cb.CUDASolver(use_graph=ug, precond=precond)) as f:
            o = f.solve_pairs(src, dst)
            r.append(o["R"]); it.append(o["iters"])
            o2 = f.solve_pairs(src, dst)           # second launch of the cached graph
            assert np.array_equal(o2["R"], o["R"])
    assert np.array_equal(r[0], r[1]) and np.array_equal(r[0], r[2])
    assert np.array_equal(it[0], it[1]) and np.array_equal(it[0], it[2])


def test_device_loop_stops_at_itmax():
    """the WHILE graph is bounded by itmax; with too few iterations the true-residual gate
    raises the reference's error (core.jl:640-641)."""
    A = holey_raster(60, 60, seed=12)
    nodes = graph.focal_nodes(A.shape[0], 2, seed=2)
    src, dst = graph.all_pairs(nodes)
    with cb.B200Factor(A, cb.CUDASolver(precond="jacobi", itmax=3)) as f:
        with pytest.raises(cb.SolverResidualError):
            f.solve_pairs(src, dst)


def test_solve_rhs_spd_and_residual_gate():
    """advanced-mode shape: Laplacian + finite grounds on the diagonal is SPD."""
    A = holey_raster(50, 40, seed=13)
    n = A.shape[0]
    rng = np.random.default_rng(4)
    gnd = np.zeros(n); gnd[rng.choice(n, 5, replace=False)] = rng.random(5) + 0.5
    M = (A + sp.diags(gnd)).tocsr()
    B = rng.standard_normal((n, 3))
    import scipy.sparse.linalg as spla
    Xref = spla.splu(M.tocsc()).solve(B)
    with cb.B200Factor(M, cb.CUDASolver(rtol=1e-10)) as f:
        X, iters, relres = f.solve_rhs(B)
        x1, _, _ = f.solve_rhs(B[:, 0])
        assert x1.shape == (n,)
        with pytest.raises(cb.SolverResidualError):
            f.solve_rhs(B, itmax=3)              # cannot converge in 3 iterations -> gate trips
    assert np.abs(X - Xref).max() / np.abs(Xref).max() < 1e-7
    assert np.abs(x1 - Xref[:, 0]).max() / np.abs(Xref).max() < 1e-7
    assert relres.max() < 1e-8


def test_solve_rhs_pipeline_many_panels():
    """hook #2 with 21 columns = panels 8+8+4+1: uploads/downloads are double-buffered on
    copy streams; every column must equal the same column solved alone."""
    A = holey_raster(64, 48, seed=21)
    n = A.shape[0]
    nodes = graph.focal_nodes(n, 22, seed=4)
    B = np.zeros((n, 21), order="F")
    for c in range(21):
        B[nodes[c], c] -= 1.0 + c
        B[nodes[c + 1], c] += 1.0 + c
    with cb.B200Factor(A, cb.CUDASolver()) as f:
        X, it, rr = f.solve_rhs(B)
        assert rr.max() < 1e-5
        for c in (0, 7, 8, 15, 16, 19, 20):
            x1, _, _ = f.solve_rhs(B[:, c].copy())
            d = (X[:, c] - X[:, c].mean()) - (x1 - x1.mean())
            assert np.abs(d).max() <= 1e-5 * np.abs(x1 - x1.mean()).max()
        X2, _, _ = f.solve_rhs(B)           # slots and events are reused across calls
        assert np.array_equal(X, X2)
    Lr = A.tocsr()
    assert np.abs(Lr @ X - B).max() / np.abs(B).max() < 1e-4


@pytest.mark.parametrize("precond", ["jacobi", "amg"])
def test_network_all_to_one_batched(precond):
    """config C5 in small: power-law graph (hub rows -> direct-gather blocks), every
    all-to-one iteration as a column of one batch; voltages equal the grounded direct
    solve, through hook #2 and through the device-resident sparse-RHS driver."""
    import scipy.sparse.linalg as spla
    from circuitscape_b200 import core
    n = 1500
    L = graph.power_law_laplacian(n, m=5, seed=11)
    focal = graph.focal_nodes(n, 11, seed=7)
    with cb.B200Factor(L, cb.CUDASolver(precond=precond, rtol=1e-10)) as f:
        V, it, rr, cols = core.all_to_one_batched(f, focal)
        FV, it2, rr2, _ = core.all_to_one_batched(f, focal, device_resident=True, accumulate=True)
        cum, mx = f.read_currents()
        o = f.solve_sources([(focal, np.r_[-10.0, np.ones(10)])], [focal[0]], probe=focal[:3],
                            want_volt=True, want_curr=True)
    assert rr.max() < 1e-6 and it.max() < 200
    assert np.array_equal(it, it2)
    assert np.abs(FV - V[focal].T).max() < 1e-9 * np.abs(V).max()
    assert np.abs(o["volt"][:, 0] - V[:, 0]).max() < 1e-9 * np.abs(V).max()
    assert np.allclose(o["probe_volt"][0], V[focal[:3], 0], rtol=0, atol=1e-9 * np.abs(V).max())
    cum_ref = np.zeros(n)
    for c in (0, 4, 10):
        g = focal[c]
        keep = np.setdiff1d(np.arange(n), [g])
        b = np.zeros(n); b[focal] = 1.0
        v = np.zeros(n)
        v[keep] = spla.splu(L[keep][:, keep].tocsc()).solve(b[keep])
        assert np.abs(V[:, c] - v).max() < 1e-6 * np.abs(v).max()
    for c in range(len(focal)):
        cum_ref += core.node_currents_host(L, V[:, c])
    assert np.abs(cum - cum_ref).max() < 1e-8 * np.abs(cum_ref).max()
    assert np.abs(o["curr"][:, 0] - core.node_currents_host(L, V[:, 0])).max() < 1e-8 * np.abs(cum_ref).max()


def test_solve_sources_rejects_bad_input():
    A = holey_raster(20, 20, seed=3)
    with cb.B200Factor(A, cb.CUDASolver()) as f:
        with pytest.raises(cb.B200Error):
            f.solve_sources([([0, A.shape[0]], [1.0, -1.0])], [0])
        with pytest.raises(cb.B200Error):
            f.solve_sources([([0, 1], [1.0, -1.0])], [-1])


def test_compute_omniscape_current_on_device():
    """src/utils.jl:145-257 through hook #3 on the GPU; the reference's own example window
    (test/internal.jl:5-43) and a 40x30 window with holes against a host direct solve."""
    import scipy.sparse as sp
    import scipy.sparse.linalg as spla
    from circuitscape_b200 import core
    conductance = np.array([[1, 5, 1.], [2, 1, 1], [9, 1, 6]])
    source = np.array([[1, 0, 0.], [0, 0, 0], [0, 1, 0]])
    ground = np.array([[0, 0, 1.], [0, 0, 0], [0, 0, 0]])
    cur = cb.compute_omniscape_current(conductance, source, ground,
                                       {"connect_four_neighbors_only": "False", "solver": "cuda"})
    assert abs(cur[0, 2] - 2.0) < 1e-6 and cur.min() >= 0
    rng = np.random.default_rng(5)
    g = rng.uniform(0.5, 2.0, (40, 30)); g[rng.random(g.shape) < 0.1] = 0.0
    src = np.zeros_like(g); src[2, 3] = 1.0; src[30, 20] = 0.5
    gnd = np.zeros_like(g); gnd[6, 1] = 2.0; gnd[35, 28] = 1.0
    for k in (src, gnd):
        k[g <= 0] = 0
    cur = cb.compute_omniscape_current(g, src, gnd, {"connect_four_neighbors_only": "True", "solver": "cuda",
                                                     "gpu_rtol": "1e-10"})
    nodemap = graph.construct_node_map(g, None)
    G = graph.laplacian(graph.construct_graph(g, nodemap, False, True))
    s, gr, f = core.sources_and_grounds_from_maps(src, gnd, nodemap, G.shape[0], "rmvsrc")
    ref = np.zeros_like(g)
    for c in graph.connected_components(G):
        rows = np.asarray(c) - 1
        if s[rows].sum() == 0 or gr[rows].sum() == 0:
            continue
        A = G[rows][:, rows]
        v = spla.splu((A + sp.diags(f[rows])).tocsc()).solve(s[rows])
        nc = core.node_currents_host(A, v, f[rows])
        for r_, val in zip(rows, nc):
            ref[nodemap == r_ + 1] += val
    assert np.abs(cur - ref).max() < 1e-7 * ref.max()


@pytest.mark.parametrize("precond", ["jacobi", "amg"])
def test_superposed_pairs_equal_direct_pairs(precond):
    """v(i,j) = u_j - u_i from np-1 point solves == one solve per pair (resistances, voltages,
    per-pair node currents, cumulative / max maps), each pair through its own residual gate."""
    A = holey_raster(70, 60, seed=31)
    nodes = graph.focal_nodes(A.shape[0], 6, seed=3)
    src, dst = graph.all_pairs(nodes)
    w = np.arange(1, len(src) + 1, dtype=np.float64)
    nn, inv = np.unique(np.concatenate([src, dst]), return_inverse=True)
    pi, pj = inv[:len(src)], inv[len(src):]
    with cb.B200Factor(A, cb.CUDASolver(precond=precond, rtol=1e-11)) as f:
        a = f.solve_pairs(src, dst, w, want_volt=True, want_curr=True, accumulate=True)
        ca, ma = f.read_currents()
        f.reset_currents()
        b = f.solve_pairs_superposed(nn, pi, pj, w, want_volt=True, want_curr=True, accumulate=True)
        cb_, mb = f.read_currents()
    assert len(b["iters"]) == len(nn) - 1 and b["iters"].max() > 0
    assert b["relres"].max() < 1e-6
    assert np.abs(b["R"] - a["R"]).max() <= 1e-8 * np.abs(a["R"]).max()
    assert np.abs(b["volt"] - a["volt"]).max() <= 1e-7 * np.abs(a["volt"]).max()
    assert np.abs(b["curr"] - a["curr"]).max() <= 1e-6 * np.abs(a["curr"]).max()
    assert np.abs(cb_ - ca).max() <= 1e-6 * np.abs(ca).max()
    assert np.abs(mb - ma).max() <= 1e-6 * np.abs(ma).max()


@pytest.mark.parametrize("i", [1, 3, 12])
def test_golden_raster_pairwise_superposed(golden, i):
    r, exp = cases.run_raster_pairwise(golden, f"sgVerify{i}", cb.CUDASolver(superpose=True, rtol=1e-8))
    cases.check_raster_pairwise(r, exp)


def test_bad_pairs_rejected():
    A = holey_raster(10, 10, seed=1)
    with cb.B200Factor(A, cb.CUDASolver()) as f:
        with pytest.raises(cb.B200Error):
            f.solve_pairs([0], [0])
        with pytest.raises(cb.B200Error):
            f.solve_pairs([0], [A.shape[0]])


# ---- the reference's golden integration cases through the CUDA library ------
@pytest.mark.parametrize("precond", ["jacobi", "amg"])
@pytest.mark.parametrize("i", range(1, 18))
def test_golden_raster_pairwise(golden, i, precond):
    r, exp = cases.run_raster_pairwise(golden, f"sgVerify{i}", cb.CUDASolver(rtol=1e-8, precond=precond))
    cases.check_raster_pairwise(r, exp, rel=1e-6)


@pytest.mark.parametrize("i", range(1, 4))
def test_golden_network_pairwise(golden, i):
    prob, flags, exp = cases.network_pairwise_problem(golden, f"sgNetworkVerify{i}", cb.CUDASolver(rtol=1e-8))
    cases.check_network_pairwise(cb.single_ground_all_pairs(prob, flags), exp)


@pytest.mark.parametrize("precond", ["jacobi", "amg"])
@pytest.mark.parametrize("name", [f"mgVerify{i}" for i in range(1, 7)] +
                         [f"mgNetworkVerify{i}" for i in range(1, 4)])
def test_golden_advanced(golden, name, precond):
    prob, flags, exp = cases.advanced_problem(golden, name, cb.CUDASolver(rtol=1e-8, precond=precond))
    cases.check_advanced(cb.advanced_kernel(prob, flags), exp, flags)


@pytest.mark.parametrize("name", [f"oneToAllVerify{i}" for i in (1, 4, 7, 10, 12, 13)] +
                         [f"allToOneVerify{i}" for i in (1, 4, 7, 12)])
def test_golden_onetoall(golden, name):
    data, flags, cfg, exp = cases.onetoall_problem(golden, name)
    fl = co.cfg_flags(cfg)
    r = cb.onetoall_kernel(data, flags, cfg, solver=cb.CUDASolver(rtol=1e-8),
                           four_neighbors=fl["four_neighbors"], avg_res=fl["avg_res"])
    cases.check_onetoall(r, exp, flags)


def test_golden_default_rtol_meets_reference_bar(golden):
    """with the reference's own rtol = 1e-6 (src/core.jl:639) the reference's own
    tolerances (1e-3 abs on R, sum d^2 < 1e-6 on maps) must hold."""
    r, exp = cases.run_raster_pairwise(golden, "sgVerify1", cb.CUDASolver())
    cases.check_raster_pairwise(r, exp, rel=1e-5)


# ---- BASELINE size (C2: 1000 x 1000, 8-neighbour, fp64): size-independent properties
@pytest.mark.parametrize("precond", ["jacobi", "amg"])
def test_full_size_properties(precond):
    L, _ = graph.synthetic_raster_laplacian(1000, 1000, seed=42)
    n = L.shape[0]
    nodes = graph.focal_nodes(n, 4, seed=7)
    a, b, c = int(nodes[0]), int(nodes[1]), int(nodes[2])
    with cb.B200Factor(L, cb.CUDASolver(precond=precond)) as f:
        o = f.solve_pairs([a, b, a, b, a], [b, a, c, c, b], want_volt=True)
        R, V = o["R"], o["volt"]
        assert o["relres"].max() < 1e-4                       # src/core.jl:641
        assert abs(R[0] - R[1]) / R[0] < 1e-6                 # symmetry R(a,b) = R(b,a)
        assert abs(R[0] - R[4]) / R[0] < 1e-9                 # same pair solved in another panel
        assert R[2] <= R[0] + R[3] and R[0] <= R[2] + R[3]    # resistance distance is a metric
        # superposition: v_(a->c) = v_(a->b) + v_(b->c) up to a constant
        d = V[:, 2] - (V[:, 0] + (V[:, 3] - V[a, 3]))
        assert np.abs(d - d.mean()).max() / R[2] < 1e-4
        # Kirchhoff: G v = e_dst - e_src
        res = L @ V[:, 0]
        res[b] -= 1.0; res[a] += 1.0
        assert np.linalg.norm(res) / np.sqrt(2) < 1e-4
        # voltages bounded by the poles (maximum principle)
        assert V[:, 0].min() >= -1e-9 and V[:, 0].max() <= R[0] * (1 + 1e-9)


# ---- round 2: the reference goldens through the TMA-staged windowed kernel (the goldens are all far
# below the 20 000-row auto threshold, so window="on" forces k_spmm_win on every operator) and at the
# reference's own default rtol = 1e-6 (src/core.jl:639) with the reference's tolerances
@pytest.mark.parametrize("setup", ["device", "host"])
@pytest.mark.parametrize("i", range(1, 18))
def test_golden_raster_pairwise_windowed(golden, i, setup):
    r, exp = cases.run_raster_pairwise(golden, f"sgVerify{i}", cb.CUDASolver(rtol=1e-8, window="on", setup=setup))
    cases.check_raster_pairwise(r, exp, rel=1e-6)


@pytest.mark.parametrize("i", range(1, 18))
def test_golden_raster_pairwise_default_rtol(golden, i):
    r, exp = cases.run_raster_pairwise(golden, f"sgVerify{i}", cb.CUDASolver())
    cases.check_raster_pairwise(r, exp, rel=1e-5)


@pytest.mark.parametrize("name", [f"mgVerify{i}" for i in range(1, 7)] + [f"mgNetworkVerify{i}" for i in range(1, 4)])
def test_golden_advanced_windowed(golden, name):
    prob, flags, exp = cases.advanced_problem(golden, name, cb.CUDASolver(rtol=1e-8, window="on"))
    cases.check_advanced(cb.advanced_kernel(prob, flags), exp, flags)


@pytest.mark.parametrize("i", range(1, 4))
def test_golden_network_pairwise_windowed_log(golden, i):
    """network goldens with the windowed kernel; log_transform_maps must not touch network currents"""
    prob, flags, exp = cases.network_pairwise_problem(golden, f"sgNetworkVerify{i}",
                                                      cb.CUDASolver(rtol=1e-8, window="on"))
    flags.outputflags.log_transform_maps = True
    cases.check_network_pairwise(cb.single_ground_all_pairs(prob, flags), exp)


# ---- device-resident grounds (cs_b200_set_grounds) -------------------------------------------------
def test_set_grounds_matches_scipy_on_the_modified_system():
    """finite grounds on the diagonal + Dirichlet rows, against SciPy's direct solve of the reference's
    reduced system (src/raster/advanced.jl:274-305); repeated calls start from the pristine operator and
    (None, None) restores the singular Laplacian."""
    import scipy.sparse.linalg as spla
    A = holey_raster(160, 150, seed=12)
    n = A.shape[0]
    rng = np.random.default_rng(5)
    with cb.B200Factor(A, cb.CUDASolver(rtol=1e-10)) as f:
        for trial in range(3):
            fg = np.zeros(n)
            fg[rng.choice(n, 5, replace=False)] = rng.uniform(0.1, 2.0, 5)
            mask = np.zeros(n, dtype=bool)
            mask[rng.choice(n, 4, replace=False)] = True
            b = np.zeros(n)
            b[rng.choice(np.nonzero(~mask)[0], 6, replace=False)] = rng.uniform(0.5, 2.0, 6)
            f.set_grounds(fg if trial != 1 else None, mask)
            x, iters, relres = f.solve_rhs(b)
            M = (A + sp.diags(fg if trial != 1 else np.zeros(n))).tocsr()
            keep = np.nonzero(~mask)[0]
            ref = np.zeros(n)
            ref[keep] = spla.splu(M[keep][:, keep].tocsc()).solve(b[keep])
            assert relres.max() < 1e-4 and iters.max() < 200
            assert np.abs(x - ref).max() <= 1e-7 * np.abs(ref).max(), trial
            # the identity rows are solved like any other row: 0 V to solver tolerance (the host driver
            # writes exact zeros there, as the reference re-inserts them, src/raster/advanced.jl:301-304)
            assert np.abs(x[mask]).max() <= 1e-7 * np.abs(ref).max()
        f.set_grounds(None, None)                        # pristine singular operator again
        nodes = graph.focal_nodes(n, 3, seed=7)
        src, dst = graph.all_pairs(nodes)
        o = f.solve_pairs(src, dst)
    Vref = co.solve_pairs_direct(A, src, dst)
    assert np.abs(o["R"] - Vref[dst, np.arange(len(src))]).max() <= 1e-7 * o["R"].max()


@pytest.mark.parametrize("name", [f"oneToAllVerify{i}" for i in (1, 4, 10, 13)] + [f"allToOneVerify{i}" for i in (1, 7, 12)])
def test_golden_onetoall_resident_grounds(golden, name):
    data, flags, cfg, exp = cases.onetoall_problem(golden, name)
    fl = co.cfg_flags(cfg)
    r = cb.onetoall_kernel(data, flags, cfg, solver=cb.CUDASolver(rtol=1e-8, resident_grounds=True),
                           four_neighbors=fl["four_neighbors"], avg_res=fl["avg_res"])
    cases.check_onetoall(r, exp, flags)

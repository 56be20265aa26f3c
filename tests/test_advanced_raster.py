"""Raster advanced mode (src/raster/advanced.jl:17-80, 151-305) on ONE whole-raster operator: core.raster_advanced,
every solved connected component a column of cs_b200_solve_advanced, the finite grounds on the operator's diagonal
(cs_b200_set_grounds) and the Inf grounds each column's Dirichlet set.

CPU: the front end on a scipy double of the handle (defined here) against the reference goldens, the oracle's
advanced kernel and the product's per-component advanced_kernel; the skip rule per component kind; the [-1] return;
argument rejection without a device.
GPU: the goldens on the device, the entry against a direct solve of each column's reduced system with the
finite-ground node currents, argument checks, the operator form after finite grounds, determinism, and the other
entry points left as they were."""

import numpy as np
import pytest
import scipy.sparse.linalg as spla
from hypothesis import HealthCheck, given, settings, strategies as st
from scipy.sparse import csgraph

import circuitscape_b200 as cb
from circuitscape_b200 import _lib, graph
from circuitscape_b200 import core as core_mod
from circuitscape_b200 import solver as S
from oracle import circuitscape_oracle as co

from . import cases
from .fake_factor import FakeFactor

MG = [f"mgVerify{i}" for i in range(1, 7)]
POLICIES = ["keepall", "rmvsrc", "rmvgnd", "rmvall"]


def _labels(A):
    adj = A.copy()
    adj.setdiag(0)
    adj.eliminate_zeros()
    return csgraph.connected_components(adj, directed=False)[1]


def advanced_direct(A, fg, sets, gset, sources, weight=None, accumulate=False, cum=None, mx=None):
    """Column c of cs_b200_solve_advanced by a direct solve on A (= L0 + diag(fg)): the rows of sets[gset[c]]
    deleted (0 V; none for gset[c] = -1), the reduced system solved on the components the sources touch, node
    currents with the finite-ground term (out.jl:178-207)."""
    n = A.shape[0]
    lab = _labels(A)
    k = len(gset)
    w = np.ones(k) if weight is None else np.asarray(weight, dtype=float)
    V, C = np.zeros((n, k)), np.zeros((n, k))
    for c in range(k):
        rows, vals = (np.asarray(x) for x in sources[c])
        b = np.zeros(n)
        np.add.at(b, rows.astype(np.int64), vals.astype(np.float64))
        g = np.asarray(sets[gset[c]]) if gset[c] >= 0 else np.zeros(0, dtype=np.int64)
        keep = np.nonzero(np.isin(lab, lab[rows]) & ~np.isin(np.arange(n), g))[0]
        V[keep, c] = spla.splu(A[keep][:, keep].tocsc()).solve(b[keep])
        C[:, c] = co.get_node_currents(A, V[:, c], fg)
        if accumulate:
            cum += w[c] * C[:, c]
            mx[:] = np.maximum(mx, C[:, c])
    return V, C


class AdvancedDouble(FakeFactor):
    """CPU double of B200Factor.set_grounds + solve_advanced."""

    fg = None

    def set_grounds(self, finite=None, dirichlet=None):
        super().set_grounds(finite, dirichlet)
        self.fg = None if finite is None else np.asarray(finite, dtype=np.float64).copy()

    def solve_advanced(self, sets, gset, sources, weight=None, want_volt=False, want_curr=False,
                       accumulate=False, **kw):
        assert all(s >= 0 for s in gset) or self.fg is not None
        V, C = advanced_direct(self.A, self.fg, sets, gset, sources, weight, accumulate, self.cum, self.mx)
        k = len(gset)
        return dict(volt=V if want_volt else None, curr=C if want_curr else None,
                    iters=np.zeros(k, dtype=np.int64), relres=np.zeros(k))


def _double_factory(cellmap, polymap, solver, four_neighbors=False, avg_res=False, log_transform=False):
    nodemap = graph.construct_node_map(cellmap, polymap)
    G = graph.laplacian(graph.construct_graph(cellmap, nodemap, avg_res, four_neighbors))
    return AdvancedDouble(G, solver, log_transform=log_transform), nodemap


@pytest.fixture
def cpu_doubles(monkeypatch):
    monkeypatch.setattr(S, "construct_cholesky_factor", lambda m, s, **kw: FakeFactor(m, s, **kw))
    monkeypatch.setattr(S, "multiple_solve", lambda s, m, b: FakeFactor(m, s).solve_rhs(np.asarray(b))[0])
    monkeypatch.setattr(S, "construct_raster_factor", _double_factory)


def _golden_run(golden, name, solver):
    cfg, inp, exp = co.load_case(golden, name)
    flags = cb.Flags.from_cfg(cfg)
    fl = co.cfg_flags(cfg)
    cellmap, polymap, meta, _ = co.load_raster_inputs(cfg, inp)
    source_map, ground_map = co.read_source_and_ground_maps(cfg, inp, meta)
    data = cb.RasterData(cellmap, polymap, None, source_map=source_map, ground_map=ground_map)
    r = cb.raster_advanced(data, flags, cfg, solver=solver, four_neighbors=fl["four_neighbors"], avg_res=fl["avg_res"])
    return r, flags, exp


def _close(a, b, rel):
    return np.abs(a - b).max() <= rel * max(1.0, np.abs(b).max())


def _run_all(g, poly, src, gm, policy, four, avg):
    """raster_advanced, the oracle's advanced kernel and the product's advanced_kernel on one problem;
    None for the oracle when it rejects the set-up"""
    cfg = {"remove_src_or_gnd": policy}
    data = cb.RasterData(g, poly, None, source_map=src, ground_map=gm)
    got = cb.raster_advanced(data, cb.Flags(is_raster=True, is_advanced=True), cfg, solver=cb.CUDASolver(),
                             four_neighbors=four, avg_res=avg)
    nodemap = co.construct_node_map(g, poly)
    G = co.laplacian(co.construct_graph(g, nodemap, avg, four))
    cc = co.connected_components(G)
    s, gr, f = co._sources_grounds_raster(src, gm, nodemap, G.shape[0], policy)
    try:
        want = co.advanced_kernel(G, cc, s, gr, f, nodemap, poly, g)
    except (AssertionError, RuntimeError):
        want = None
    pn = graph.construct_node_map(g, poly)
    PG = graph.laplacian(graph.construct_graph(g, pn, avg, four))
    sp_, gp, fp = core_mod.sources_and_grounds_from_maps(src, gm, pn, PG.shape[0], policy)
    prod = cb.advanced_kernel(cb.AdvancedProblem(PG, graph.connected_components(PG), sp_, gp, fp, pn, poly, g,
                                                 cb.CUDASolver()), cb.Flags(is_raster=True, is_advanced=True))
    return got, want, prod


def _agree(got, want, rel=1e-8):
    assert _close(got.voltmap, want.voltmap, rel)
    assert _close(got.curmap, want.curmap, rel)
    assert _close(got.voltages, want.voltages, rel)


# ---------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", MG)
def test_advanced_goldens_on_the_double(cpu_doubles, golden, name):
    r, flags, exp = _golden_run(golden, name, cb.CUDASolver())
    cases.check_advanced(r, exp, flags)
    assert r.num_solves > 0 and np.array_equal(r.result, r.voltmap)


@st.composite
def advanced_rasters(draw):
    nr, nc = draw(st.integers(3, 8)), draw(st.integers(3, 8))
    rng = np.random.default_rng(draw(st.integers(0, 2**31 - 1)))
    g = rng.uniform(0.2, 4.0, (nr, nc))
    g[rng.random((nr, nc)) < draw(st.sampled_from([0.0, 0.15, 0.3]))] = 0.0
    if draw(st.booleans()):
        g[nr // 2, :] = 0.0                               # a NODATA wall: several components
    poly = None
    if draw(st.booleans()):
        poly = np.zeros((nr, nc), dtype=np.int64)
        poly[rng.random((nr, nc)) < 0.2] = 1
        poly[rng.random((nr, nc)) < 0.1] = 2
    src = np.where(rng.random((nr, nc)) < 0.2, rng.uniform(0.5, 2.0, (nr, nc)), 0.0)
    if draw(st.booleans()):
        src[rng.random((nr, nc)) < 0.1] *= -1.0           # sinks too
    kind = draw(st.sampled_from(["finite", "inf", "mixed"]))
    gm = np.where(rng.random((nr, nc)) < 0.2, rng.uniform(0.5, 2.0, (nr, nc)), 0.0)
    if kind == "inf":
        gm = np.where(gm != 0, np.inf, 0.0)
    elif kind == "mixed":
        gm = np.where((gm != 0) & (rng.random((nr, nc)) < 0.5), np.inf, gm)
    return (g, poly, src, gm, draw(st.sampled_from(POLICIES)), draw(st.booleans()), draw(st.booleans()))


@settings(max_examples=150, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(p=advanced_rasters())
def test_random_rasters_match_oracle_and_advanced_kernel(cpu_doubles, p):
    g, poly, src, gm, policy, four, avg = p
    if graph.construct_node_map(g, poly).max() == 0:
        return
    got, want, prod = _run_all(g, poly, src, gm, policy, four, avg)
    _agree(got, prod)
    if want is not None:
        _agree(got, want)
    assert np.array_equal(got.result, got.voltmap if got.num_solves else np.array([[-1.0]]))


def _kinds_raster():
    """six 2-row components between NODATA walls: only sources, only grounds, cancelling sources (with a finite
    ground), only finite grounds, only Inf grounds (a sink on one of them), and both kinds of ground with a source
    on a finite-ground cell"""
    rng = np.random.default_rng(17)
    g = rng.uniform(0.5, 2.0, (17, 5))
    g[[2, 5, 8, 11, 14], :] = 0.0
    src, gm = np.zeros(g.shape), np.zeros(g.shape)
    src[0, 1] = 1.0                                       # component 0: sources only
    gm[3, 2] = 0.7                                        # component 1: grounds only
    src[6, 0], src[7, 4], gm[6, 3] = 1.5, -1.5, 0.4       # component 2: sources that cancel
    src[9, 1], gm[10, 3], gm[9, 4] = 2.0, 0.6, 0.3        # component 3: finite grounds only
    src[12, 0], gm[13, 4], gm[12, 2] = 1.0, np.inf, np.inf   # component 4: Inf grounds only
    src[13, 2] = -0.25                                    # ... and a sink
    src[15, 0], gm[16, 4], gm[15, 3] = 1.0, np.inf, 0.8   # component 5: both ...
    src[15, 3] = 0.5                                      # ... a source on its finite-ground cell
    src[16, 1], gm[16, 1] = -0.5, np.inf                  # ... and a sink on an Inf ground (deleted)
    return g, src, gm


@pytest.mark.parametrize("policy", POLICIES)
def test_each_component_kind(cpu_doubles, policy, monkeypatch):
    g, src, gm = _kinds_raster()
    gsets = []
    real = AdvancedDouble.solve_advanced
    monkeypatch.setattr(AdvancedDouble, "solve_advanced",
                        lambda self, sets, gset, *a, **kw: gsets.append((list(sets), list(gset))) or
                        real(self, sets, gset, *a, **kw))
    got, want, prod = _run_all(g, None, src, gm, policy, False, False)
    _agree(got, want)
    _agree(got, prod)
    nodemap = graph.construct_node_map(g, None)
    assert got.num_solves == 3                            # components 3, 4 and 5 under every policy
    band = lambda c: slice(3 * c, 3 * c + 2)
    for c in range(6):
        assert np.any(got.voltmap[band(c)] != 0) == (c in {3, 4, 5}), c
    # one chunk: the finite-only component without a ground set, the others with their Inf rows only
    (sets, gset), = gsets
    assert sorted(gset) == [-1, 0, 1]
    inf_cells = [(12, 2), (13, 4), (16, 4)] + ([] if policy == "rmvgnd" else [(16, 1)])
    assert {int(r) for s in sets for r in s} == {int(nodemap[a, b]) - 1 for a, b in inf_cells}


def test_nothing_solved_returns_minus_one(cpu_doubles, monkeypatch):
    monkeypatch.setattr(S, "construct_raster_factor", lambda *a, **kw: pytest.fail("a handle without columns"))
    g, src, gm = _kinds_raster()
    keep = np.zeros(g.shape, dtype=bool)
    keep[:5] = True                                       # components 0 and 1: sources only, grounds only
    got, want, prod = _run_all(np.where(keep, g, 0.0), None, np.where(keep, src, 0.0), np.where(keep, gm, 0.0),
                               "keepall", False, False)
    assert got.num_solves == 0 and np.array_equal(got.result, [[-1.0]])
    assert not got.voltmap.any() and not got.curmap.any()
    _agree(got, want)


def test_solve_advanced_rejects_bad_arguments_without_a_device():
    lib = _lib.load()
    i64 = lambda *v: np.array(v, dtype=np.int64)
    vals = np.ones(8)

    def call(ptr, rows, gset, sptr, srows, nsets=None):
        nsets = len(ptr) - 1 if nsets is None else nsets
        rc = lib.cs_b200_solve_advanced(None, nsets, ptr.ctypes.data, rows.ctypes.data, len(gset), gset.ctypes.data,
                                        sptr.ctypes.data, srows.ctypes.data, vals.ctypes.data, None, 1e-6, 100,
                                        None, None, 0, None, None)
        return rc, lib.cs_b200_last_error(None).decode()

    ptr, rows = i64(0, 2, 3), i64(4, 7, 9)
    sptr, srows = i64(0, 1, 3), i64(5, 1, 2)
    rc, msg = call(ptr, rows, i64(0, -1), sptr, srows)
    assert rc == _lib.ERR_ARG and "no direct grounds" in msg
    rc, msg = call(i64(0), i64(0), i64(-1, -1), sptr, srows)
    assert rc == _lib.ERR_ARG and "no direct grounds" in msg
    rc, msg = call(ptr, rows, i64(0, -2), sptr, srows)
    assert rc == _lib.ERR_ARG and "set index" in msg
    rc, msg = call(ptr, i64(7, 4, 9), i64(0, 1), sptr, srows)
    assert rc == _lib.ERR_ARG and "sorted" in msg
    rc, msg = call(ptr, rows, i64(0, 1), sptr, i64(7, 1, 2))
    assert rc == _lib.ERR_ARG and "on its ground set" in msg
    rc, msg = call(ptr, rows, i64(0, 1), i64(0, 1, 1), srows)
    assert rc == _lib.ERR_ARG and "no sources" in msg
    rc, msg = call(ptr, rows, i64(0, 1), sptr, srows)    # well-formed: only the missing handle is left
    assert rc == _lib.ERR_ARG and "null handle" in msg


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("precond", ["amg", "jacobi"])
@pytest.mark.parametrize("name", MG)
def test_advanced_goldens_on_the_device(golden, name, precond):
    r, flags, exp = _golden_run(golden, name, cb.CUDASolver(rtol=1e-8, precond=precond))
    cases.check_advanced(r, exp, flags)
    assert np.array_equal(r.result, r.voltmap)


def _raster(kind, seed=5):
    """230 x 160 cells: a full raster takes the stencil form, a holey one the windowed records"""
    rng = np.random.default_rng(seed)
    g = 1.0 / rng.uniform(1.0, 10.0, (230, 160))
    if kind == "holes":
        g[rng.random(g.shape) < 0.08] = 0.0
        g[60:64, :] = 0.0                          # a wall: two components
    return g


def _finite(nodemap, n, rng):
    """finite grounds on a vertical band of cells that crosses every component"""
    fg = np.zeros(n)
    rows = np.unique(nodemap[:, 70:74])
    rows = rows[rows > 0] - 1
    fg[rows] = rng.uniform(0.05, 0.5, len(rows))
    return fg


def _columns(lab, rng, k, sizes):
    """k columns: sizes[c % len] Inf-ground rows (0: gset = -1) and 1-3 sources elsewhere in their component"""
    n = len(lab)
    sets, gset, sources = [], [], []
    for c in range(k):
        size = sizes[c % len(sizes)]
        while True:
            gnd = np.unique(rng.choice(n, size, replace=False)) if size else np.zeros(0, dtype=np.int64)
            comp = lab[gnd[0]] if size else lab[rng.integers(n)]
            cand = np.setdiff1d(np.nonzero(lab == comp)[0], gnd)
            if len(cand) >= 3:
                break
        gset.append(len(sets) if size else -1)
        if size:
            sets.append(gnd)
        rows = np.sort(rng.choice(cand, rng.integers(1, 4), replace=False))
        sources.append((rows, rng.uniform(0.5, 2.0, len(rows)) * rng.choice([-1.0, 1.0], len(rows))))
    return sets, np.array(gset), sources


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["full", "holes"])
@pytest.mark.parametrize("prec", ["fp64", "mixed", "single"])
def test_solve_advanced_matches_a_direct_solve(kind, prec):
    g = _raster(kind)
    # fp32 arithmetic on the device stagnates near 1e-4 of ||b|| for point sources: rtol and the bounds follow
    solver = cb.CUDASolver(rtol=1e-6 if prec == "single" else 1e-10, mixed=prec == "mixed",
                           precision="single" if prec == "single" else "double", f32_compute=prec == "single")
    factor, nodemap = S.construct_raster_factor(g, None, solver)
    rng = np.random.default_rng(11)
    with factor:
        fg = _finite(nodemap, factor.n, rng)
        factor.set_grounds(finite=fg)
        assert factor.operator_form() == ("stencil" if kind == "full" else "windowed")
        A = factor.get_csr().astype(np.float64)          # L0 + diag(fg) as the device holds it
        fgd = fg.astype(factor.dtype).astype(np.float64)
        lab = _labels(A)
        tol = 3e-3 if prec == "single" else 1e-7
        for k in range(1, 10):                             # KT 1/2/4/8, ragged panels
            sets, gset, sources = _columns(lab, rng, k, [0, 1, 64])
            w = rng.integers(1, 4, k).astype(np.float64)
            factor.reset_currents()
            cum, mx = np.zeros(factor.n), np.full(factor.n, -np.inf)
            got = factor.solve_advanced(sets, gset, sources, weight=w, want_volt=True, want_curr=True,
                                        accumulate=True, raise_on_residual=prec != "single")
            assert got["relres"].max() < (1e-3 if prec == "single" else 1e-6)
            V, C = advanced_direct(A, fgd, sets, gset, sources, w, True, cum, mx)
            assert np.abs(got["volt"] - V).max() <= tol * np.abs(V).max()
            for c in range(k):
                want_c = core_mod.node_currents_host(A, np.asarray(got["volt"][:, c], dtype=np.float64), fgd)
                assert np.abs(got["curr"][:, c] - want_c).max() <= 10 * tol * np.abs(want_c).max()
                if gset[c] >= 0:                           # the Inf-ground rows hold 0 V exactly
                    assert np.all(got["volt"][sets[gset[c]], c] == 0)
            assert np.abs(got["curr"] - C).max() <= 10 * tol * np.abs(C).max()
            dcum, dmx = factor.read_currents()
            assert np.abs(dcum - cum).max() <= 10 * tol * np.abs(cum).max()
            assert np.abs(dmx - mx).max() <= 10 * tol * np.abs(mx).max()


@pytest.mark.gpu
def test_solve_advanced_rejects_bad_arguments_on_a_handle():
    g = _raster("full")
    factor, nodemap = S.construct_raster_factor(g, None, cb.CUDASolver())
    with factor:
        src = [(np.array([5]), np.ones(1))]
        with pytest.raises(cb.B200Error) as e:             # no finite grounds on the handle
            factor.solve_advanced([], [-1], src)
        assert e.value.code == _lib.ERR_ARG and "no direct grounds" in str(e.value)
        with pytest.raises(cb.B200Error) as e:
            factor.solve_advanced([np.array([9, 3])], [0], src)
        assert e.value.code == _lib.ERR_ARG and "sorted" in str(e.value)
        with pytest.raises(cb.B200Error) as e:
            factor.solve_advanced([np.array([3, factor.n])], [0], src)
        assert e.value.code == _lib.ERR_ARG and "out of range" in str(e.value)
        fg = _finite(nodemap, factor.n, np.random.default_rng(1))
        factor.set_grounds(finite=fg)
        assert factor.solve_advanced([], [-1], src, want_volt=True)["volt"][5, 0] > 0
        factor.set_grounds()                               # back to L0: the finite grounds are gone
        with pytest.raises(cb.B200Error) as e:
            factor.solve_advanced([], [-1], src)
        assert e.value.code == _lib.ERR_ARG


@pytest.mark.gpu
def test_full_raster_keeps_the_half_form_after_finite_grounds():
    g = _raster("full")
    factor, nodemap = S.construct_raster_factor(g, None, cb.CUDASolver())
    with factor:
        factor.set_grounds(finite=_finite(nodemap, factor.n, np.random.default_rng(2)))
        assert factor.operator_form() == "stencil"
        assert factor.levels()[0]["A_stencil_slots"] == 5


@pytest.mark.gpu
def test_advanced_columns_are_deterministic_and_leave_other_entries_alone():
    g = _raster("full", seed=9)
    factor, nodemap = S.construct_raster_factor(g, None, cb.CUDASolver())
    rng = np.random.default_rng(2)
    with factor:
        factor.set_grounds(finite=_finite(nodemap, factor.n, rng))
        lab = np.zeros(factor.n, dtype=np.int64)
        sets, gset, sources = _columns(lab, rng, 16, [0, 1, 3, 60])
        gsets, _, gsources = _columns(lab, rng, 8, [2, 60])
        src = np.array([s[0][0] for s in sources[:4]])
        dst = np.array([s[0][0] for s in sources[4:8]])

        def others():
            factor.reset_currents()
            a = factor.solve_grounded(gsets, np.arange(8), gsources, want_volt=True, want_curr=True, accumulate=True)
            b = factor.solve_sources([(np.array([s, d]), np.array([1.0, -1.0])) for s, d in zip(src, dst)], dst,
                                     want_volt=True, want_curr=True, accumulate=True)
            return a, b, factor.read_currents()

        before = others()
        runs = []
        for _ in range(2):
            factor.reset_currents()
            p = factor.solve_advanced(sets, gset, sources, want_volt=True, want_curr=True, accumulate=True)
            runs.append((p["volt"], p["curr"]) + tuple(factor.read_currents()))
        for x, y in zip(runs[0], runs[1]):
            assert np.array_equal(x, y)
        after = others()
        for x, y in zip(before[:2], after[:2]):
            for key in x:
                if x[key] is not None:
                    assert np.array_equal(x[key], y[key]), key
        for x, y in zip(before[2], after[2]):
            assert np.array_equal(x, y)


@pytest.mark.gpu
def test_front_end_matches_advanced_kernel_on_the_device():
    """a holey raster with polygons and NODATA walls: many components of every kind, finite and Inf grounds"""
    rng = np.random.default_rng(23)
    g = rng.uniform(0.2, 4.0, (140, 110))
    g[rng.random(g.shape) < 0.1] = 0.0
    g[[30, 70, 100], :] = 0.0
    g[:, 55] = 0.0
    poly = np.zeros(g.shape, dtype=np.int64)
    poly[10:14, 10:14] = 1
    poly[80:83, 60:70] = 2
    src = np.where(rng.random(g.shape) < 0.002, rng.uniform(0.5, 2.0, g.shape), 0.0)
    gm = np.where(rng.random(g.shape) < 0.003, rng.uniform(0.1, 1.0, g.shape), 0.0)
    gm[(gm != 0) & (rng.random(g.shape) < 0.4)] = np.inf
    for policy in POLICIES:
        data = cb.RasterData(g, poly, None, source_map=src, ground_map=gm)
        got = cb.raster_advanced(data, cb.Flags(is_raster=True, is_advanced=True), {"remove_src_or_gnd": policy},
                                 solver=cb.CUDASolver(rtol=1e-10))
        nodemap = graph.construct_node_map(g, poly)
        G = graph.laplacian(graph.construct_graph(g, nodemap, False, False))
        s, gr, f = core_mod.sources_and_grounds_from_maps(src, gm, nodemap, G.shape[0], policy)
        want = cb.advanced_kernel(cb.AdvancedProblem(G, graph.connected_components(G), s, gr, f, nodemap, poly, g,
                                                     cb.CUDASolver(rtol=1e-10)),
                                  cb.Flags(is_raster=True, is_advanced=True))
        assert got.num_solves > 4
        _agree(got, want, rel=1e-6)

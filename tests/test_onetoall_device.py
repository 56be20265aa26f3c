"""One-to-all / all-to-one raster jobs (src/raster/onetoall.jl:13-167) with CUDASolver(onetoall_raster=True):
every iteration a column on ONE whole-raster operator, the focal-node ground set changing per column
(cs_b200_solve_grounded), all-to-one with one ground row through the singular form of cs_b200_solve_sources.

CPU: the driver on a scipy double of `solve_grounded` (reduced system solved with splu, defined here)
against the oracle's per-iteration driver, the product's per-iteration path and the reference goldens;
each fallback reason of `plan_onetoall`; argument rejection without a device.
GPU: the goldens on the device, the device entry against a direct solve, a deep hierarchy, determinism,
and the other entry points left as they were."""

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

ONE_TO_ALL = [f"oneToAllVerify{i}" for i in range(1, 14)] + [f"allToOneVerify{i}" for i in range(1, 13)]


def grounded_direct(A, sets, gset, sources, weight=None, accumulate=False, log=False, cum=None, mx=None):
    """Column c of cs_b200_solve_grounded by a direct solve: rows of sets[gset[c]] deleted (0 V), the
    reduced system solved on the components the sources touch, node currents on the full operator."""
    n = A.shape[0]
    adj = A.copy()
    adj.data = (adj.data != 0).astype(np.int8)
    adj.eliminate_zeros()
    lab = csgraph.connected_components(adj, directed=False)[1]
    k = len(gset)
    w = np.ones(k) if weight is None else np.asarray(weight, dtype=float)
    V, C, sv = np.zeros((n, k)), np.zeros((n, k)), np.zeros(k)
    for c in range(k):
        rows, vals = (np.asarray(x) for x in sources[c])
        b = np.zeros(n)
        np.add.at(b, rows.astype(np.int64), vals.astype(np.float64))
        g = np.asarray(sets[gset[c]])
        keep = np.nonzero(np.isin(lab, lab[rows]) & ~np.isin(np.arange(n), g))[0]
        V[keep, c] = spla.splu(A[keep][:, keep].tocsc()).solve(b[keep])
        sv[c] = V[rows[0], c]
        C[:, c] = co.get_node_currents(A, V[:, c])
        if accumulate:
            cur = C[:, c]
            val = np.where(cur > 0, np.log10(np.where(cur > 0, cur, 1.0)), -9999.0) if log else cur
            cum += w[c] * val
            mx[:] = np.maximum(mx, val)
    return sv, V, C


class GroundedDouble(FakeFactor):
    """CPU double of B200Factor.solve_grounded."""

    def solve_grounded(self, sets, gset, sources, weight=None, want_volt=False, want_curr=False,
                       accumulate=False, **kw):
        sv, V, C = grounded_direct(self.A, sets, gset, sources, weight, accumulate, self.log, self.cum, self.mx)
        k = len(gset)
        return dict(src_volt=sv, volt=V if want_volt else None, curr=C if want_curr else None,
                    iters=np.zeros(k, dtype=np.int64), relres=np.zeros(k))

    def solve_sources(self, columns, ref, probe=None, weight=None, want_volt=False, want_curr=False,
                      accumulate=False, **kw):
        """the singular form on an operator of several components: the column's own component, shifted
        to 0 V at ref, is the grounded solve at ref (other components 0; the device leaves them constant)"""
        cols = []
        for (rows, vals), r in zip(columns, ref):
            rows, vals = np.asarray(rows), np.asarray(vals)
            cols.append((rows[rows != r], vals[rows != r]))
        sv, V, C = grounded_direct(self.A, [np.array([r]) for r in ref], np.arange(len(ref)), cols, weight,
                                   accumulate, self.log, self.cum, self.mx)
        k = len(ref)
        return dict(probe_volt=None, volt=V if want_volt else None, curr=C if want_curr else None,
                    iters=np.zeros(k, dtype=np.int64), relres=np.zeros(k))


def _double_factory(cellmap, polymap, solver, four_neighbors=False, avg_res=False, log_transform=False):
    nodemap = graph.construct_node_map(cellmap, polymap)
    G = graph.laplacian(graph.construct_graph(cellmap, nodemap, avg_res, four_neighbors))
    return GroundedDouble(G, solver, log_transform=log_transform), nodemap


@pytest.fixture
def cpu_doubles(monkeypatch):
    monkeypatch.setattr(S, "construct_cholesky_factor", lambda m, s, **kw: FakeFactor(m, s, **kw))
    monkeypatch.setattr(S, "multiple_solve", lambda s, m, b: FakeFactor(m, s).solve_rhs(np.asarray(b))[0])
    monkeypatch.setattr(S, "construct_raster_factor", _double_factory)


def compare(got, want, rel_r=1e-9, rel_map=1e-9):
    assert got.resistances.shape == want.resistances.shape
    assert np.abs(got.resistances - want.resistances).max() <= rel_r * max(1.0, np.abs(want.resistances).max())
    assert set(got.curmaps) == set(want.curmaps) and set(got.voltmaps) == set(want.voltmaps)
    close = lambda a, b: np.abs(a - b).max() <= rel_map * max(1.0, np.abs(b).max())
    for k in want.curmaps:
        assert close(got.curmaps[k], want.curmaps[k])
    for k in want.voltmaps:
        assert close(got.voltmaps[k], want.voltmaps[k])
    assert close(got.cum_curmap, want.cum_curmap)
    if want.max_curmap is not None:
        assert close(got.max_curmap, want.max_curmap)


def _golden_run(golden, name, solver):
    data, flags, cfg, exp = cases.onetoall_problem(golden, name)
    four = co.cfg_bool(cfg, "connect_four_neighbors_only")
    avg = cfg.get("connect_using_avg_resistances", "False") in ("True", "true")
    return cb.onetoall_kernel(data, flags, cfg, solver=solver, four_neighbors=four, avg_res=avg), flags, exp


# ---------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", ONE_TO_ALL)
def test_onetoall_goldens_on_the_doubles(cpu_doubles, golden, name):
    r, flags, exp = _golden_run(golden, name, cb.CUDASolver(onetoall_raster=True))
    cases.check_onetoall(r, exp, flags)


@st.composite
def onetoall_problems(draw):
    nr, nc = draw(st.integers(3, 8)), draw(st.integers(3, 8))
    rng = np.random.default_rng(draw(st.integers(0, 2**31 - 1)))
    g = rng.uniform(0.2, 4.0, (nr, nc))
    g[rng.random((nr, nc)) < draw(st.sampled_from([0.0, 0.15, 0.3]))] = -9999.0
    if draw(st.booleans()):
        g[nr // 2, :] = -9999.0                            # a wall: several components
    npts = draw(st.integers(2, 6))
    cells = rng.choice(nr * nc, size=npts, replace=False)
    pm = np.zeros((nr, nc))
    ids = np.arange(1, npts + 1)
    if draw(st.booleans()) and npts >= 3:
        ids[-1] = ids[0]                                  # focal regions: one id on several cells
        if npts >= 5 and draw(st.booleans()):
            ids[-2] = ids[1]
    pm.ravel()[cells] = ids
    poly = None
    if draw(st.booleans()):
        poly = np.zeros((nr, nc))
        poly[rng.random((nr, nc)) < 0.2] = 1
        poly[rng.random((nr, nc)) < 0.1] = 2
    strengths = None
    if draw(st.booleans()):
        u = np.unique(ids)
        strengths = np.column_stack([u, rng.uniform(0.5, 3.0, len(u))])
    scenario = draw(st.sampled_from(["one-to-all", "all-to-one"]))
    maps = draw(st.sampled_from(["none", "cur", "volt+cur+max", "cum_only"]))
    return g, pm, poly, strengths, scenario, maps, draw(st.booleans())


def _problem(g, pm, poly, strengths, scenario, maps, four):
    nr, nc = g.shape
    meta = np.array([nc, nr, 0.0, 0.0, 1.0])
    cfg = {"scenario": scenario, "data_type": "raster", "habitat_map_is_resistances": "False",
           "write_cur_maps": str(maps in ("cur", "volt+cur+max")), "write_volt_maps": str(maps == "volt+cur+max"),
           "write_max_cur_maps": str(maps == "volt+cur+max"), "write_cum_cur_map_only": str(maps == "cum_only"),
           "use_polygons": str(poly is not None), "use_variable_source_strengths": str(strengths is not None),
           "connect_four_neighbors_only": str(four)}
    inputs = {"habitat_file": ("grid", g, meta), "point_file": ("grid", pm, meta)}
    if poly is not None:
        inputs["polygon_file"] = ("grid", poly, meta)
    if strengths is not None:
        inputs["variable_source_file"] = ("txtlist", strengths, np.zeros(0))
    cellmap, polymap, _, inc = co.load_raster_inputs(cfg, inputs)
    data = cb.RasterData(cellmap, polymap, co.read_point_map("grid", pm, meta),
                         None if strengths is None else strengths.copy(), inc)
    return cfg, inputs, data


def _plan_of(data, cfg, four=False):
    rr, cc_, ids = (np.asarray(a) for a in data.points_rc)
    point_map = np.zeros(data.cellmap.shape, dtype=np.int64)
    point_map[rr - 1, cc_ - 1] = ids
    newpoly = graph.create_new_polymap(data.cellmap, data.polymap, (rr, cc_, ids), point_map)
    nodemap = graph.construct_node_map(data.cellmap, newpoly)
    adj = graph.construct_graph(data.cellmap, nodemap, False, four)
    adj.eliminate_zeros()
    comp_of = csgraph.connected_components(adj, directed=False)[1]
    return core_mod.plan_onetoall(data.cellmap, newpoly, (rr, cc_, ids), nodemap, comp_of,
                                  cfg["scenario"] == "one-to-all", data.strengths, data.included_pairs)


@settings(max_examples=150, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(p=onetoall_problems())
def test_onetoall_columns_match_oracle_and_the_loop(cpu_doubles, p):
    g, pm, poly, strengths, scenario, maps, four = p
    cfg, inputs, data = _problem(g, pm, poly, strengths, scenario, maps, four)
    try:
        want = co.raster_one_to_all(cfg, inputs)
    except (ValueError, IndexError):
        with pytest.raises((ValueError, IndexError)):     # the product rejects them the same way
            cb.onetoall_kernel(data, cb.Flags.from_cfg(cfg), cfg, solver=cb.CUDASolver(onetoall_raster=True),
                               four_neighbors=four)
        return
    flags = cb.Flags.from_cfg(cfg)
    got = cb.onetoall_kernel(data, flags, cfg, solver=cb.CUDASolver(onetoall_raster=True), four_neighbors=four)
    loop = cb.onetoall_kernel(data, flags, cfg, solver=cb.CUDASolver(), four_neighbors=four)
    compare(got, want)
    compare(got, loop)
    assert got.num_solves == loop.num_solves


def _lm_case():
    """a focal region whose first cell is NODATA, in a raster of several components: the component's local
    node numbering differs from L0's"""
    N = -9999.0
    g = np.array([[3.02968197, N, 3.79571608], [N, 1.90727603, N], [2.13672554, 1.50118691, N],
                  [N, 1.14983282, 3.50826361], [N, 0.25732439, 1.38680231], [1.92996258, 2.58616864, 0.621780943]])
    pm = np.array([[0, 0, 0], [0, 0, 1], [0, 0, 0], [0, 0, 0], [2, 0, 1], [3, 0, 0.]])
    return g, pm


@pytest.mark.parametrize("scenario", ["one-to-all", "all-to-one"])
def test_each_fallback_reason_takes_the_per_iteration_path(cpu_doubles, scenario, monkeypatch):
    calls = []
    real = core_mod.multiple_solver
    monkeypatch.setattr(core_mod, "multiple_solver", lambda *a, **kw: calls.append(1) or real(*a, **kw))
    g, pm = _lm_case()
    cfg, inputs, data = _problem(g, pm, None, None, scenario, "volt+cur+max", True)
    plan = _plan_of(data, cfg, four=True)
    assert plan.per_iteration and all("local node map" in plan.reasons[i] for i in plan.per_iteration)
    got = cb.onetoall_kernel(data, cb.Flags.from_cfg(cfg), cfg, solver=cb.CUDASolver(onetoall_raster=True),
                             four_neighbors=True)
    assert calls
    compare(got, co.raster_one_to_all(cfg, inputs))
    # an include list: every iteration through the loop
    rng = np.random.default_rng(3)
    g = rng.uniform(0.5, 2.0, (6, 7))
    pm = np.zeros((6, 7))
    pm[0, 0], pm[2, 5], pm[5, 3], pm[4, 1] = 1, 2, 3, 4
    cfg, inputs, data = _problem(g, pm, None, None, scenario, "cur", False)
    cfg["use_included_pairs"] = "True"
    inputs["included_pairs_file"] = ("pairs_aagrid", np.array([[0, 1, 2, 3, 4], [1, 0, 1, 1, 0], [2, 1, 0, 1, 1],
                                                                [3, 1, 1, 0, 1], [4, 0, 1, 1, 0]], dtype=np.float64),
                                     np.array([1.0, 1.0]))
    cellmap, polymap, _, incp = co.load_raster_inputs(cfg, inputs)
    assert incp is not None
    data = cb.RasterData(cellmap, polymap, data.points_rc, None, incp)
    plan = _plan_of(data, cfg)
    assert plan.per_iteration == list(range(4)) and "include" in plan.reasons[0]
    calls.clear()
    got = cb.onetoall_kernel(data, cb.Flags.from_cfg(cfg), cfg, solver=cb.CUDASolver(onetoall_raster=True))
    assert calls
    compare(got, cb.onetoall_kernel(data, cb.Flags.from_cfg(cfg), cfg, solver=cb.CUDASolver()))
    compare(got, co.raster_one_to_all(cfg, inputs))


def test_clean_iterations_are_columns_and_need_no_loop(cpu_doubles, monkeypatch):
    monkeypatch.setattr(core_mod, "multiple_solver", lambda *a, **kw: pytest.fail("loop solve"))
    g = np.random.default_rng(1).uniform(0.5, 2.0, (9, 8))
    g[4, :6] = -9999.0
    pm = np.zeros((9, 8))
    pm[0, 0], pm[8, 7], pm[2, 6], pm[6, 1] = 1, 2, 3, 4
    for scenario in ("one-to-all", "all-to-one"):
        cfg, inputs, data = _problem(g, pm, None, None, scenario, "volt+cur+max", False)
        plan = _plan_of(data, cfg)
        assert len(plan.columns) == 4 and not plan.per_iteration
        compare(cb.onetoall_kernel(data, cb.Flags.from_cfg(cfg), cfg, solver=cb.CUDASolver(onetoall_raster=True)),
                co.raster_one_to_all(cfg, inputs))


def test_solve_grounded_rejects_bad_arguments_without_a_device():
    lib = _lib.load()
    i64 = lambda *v: np.array(v, dtype=np.int64)
    sv = np.zeros(4)
    vals = np.ones(8)

    def call(ptr, rows, gset, sptr, srows, k=None, nsets=None):
        k = len(gset) if k is None else k
        nsets = len(ptr) - 1 if nsets is None else nsets
        rc = lib.cs_b200_solve_grounded(None, nsets, ptr.ctypes.data, rows.ctypes.data, k, gset.ctypes.data,
                                        sptr.ctypes.data, srows.ctypes.data, vals.ctypes.data, None, 1e-6, 100,
                                        sv.ctypes.data, None, None, 0, None, None)
        return rc, lib.cs_b200_last_error(None).decode()

    ptr, rows = i64(0, 2, 3), i64(4, 7, 9)
    sptr, srows = i64(0, 1, 3), i64(5, 1, 2)
    gs = i64(0, 1)
    assert call(ptr, rows, gs, sptr, srows, k=0)[0] == _lib.ERR_ARG
    rc, msg = call(i64(0, 2, 2), rows, gs, sptr, srows)
    assert rc == _lib.ERR_ARG and "empty" in msg
    rc, msg = call(ptr, i64(7, 4, 9), gs, sptr, srows)
    assert rc == _lib.ERR_ARG and "sorted" in msg
    rc, msg = call(ptr, i64(4, 4, 9), gs, sptr, srows)
    assert rc == _lib.ERR_ARG and "sorted" in msg
    rc, msg = call(ptr, i64(-1, 7, 9), gs, sptr, srows)
    assert rc == _lib.ERR_ARG and "out of range" in msg
    rc, msg = call(ptr, rows, i64(0, 2), sptr, srows)
    assert rc == _lib.ERR_ARG and "set index" in msg
    rc, msg = call(ptr, rows, gs, sptr, i64(7, 1, 2))
    assert rc == _lib.ERR_ARG and "on its ground set" in msg
    rc, msg = call(ptr, rows, gs, sptr, i64(5, 1, 9))
    assert rc == _lib.ERR_ARG and "on its ground set" in msg
    rc, msg = call(ptr, rows, gs, i64(0, 1, 1), srows)
    assert rc == _lib.ERR_ARG and "no sources" in msg
    rc, msg = call(ptr, rows, gs, sptr, i64(5, -1, 2))
    assert rc == _lib.ERR_ARG and "out of range" in msg
    rc, msg = call(ptr, rows, gs, sptr, srows)        # well-formed: only the missing handle is left
    assert rc == _lib.ERR_ARG and "null handle" in msg


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("precond", ["amg", "jacobi"])
@pytest.mark.parametrize("name", ONE_TO_ALL)
def test_onetoall_goldens_on_the_device(golden, name, precond):
    r, flags, exp = _golden_run(golden, name, cb.CUDASolver(rtol=1e-8, precond=precond, onetoall_raster=True))
    cases.check_onetoall(r, exp, flags)


def _raster(kind, seed=5):
    """230 x 160 cells: a full raster takes the stencil form, a holey one the windowed records"""
    rng = np.random.default_rng(seed)
    g = 1.0 / rng.uniform(1.0, 10.0, (230, 160))
    if kind == "holes":
        g[rng.random(g.shape) < 0.08] = 0.0
        g[60:64, :] = 0.0                          # a wall: two components
    return g


def _columns(nodemap, lab, rng, k, sizes):
    """k columns: a ground set of sizes[c % len] random rows, 1-3 sources elsewhere in the set's component"""
    n = int(nodemap.max())
    sets, sources = [], []
    for c in range(k):
        while True:
            gnd = np.unique(rng.choice(n, sizes[c % len(sizes)], replace=False))
            cand = np.setdiff1d(np.nonzero(lab == lab[gnd[0]])[0], gnd)
            if len(cand) >= 3:
                break
        rows = np.sort(rng.choice(cand, rng.integers(1, 4), replace=False))
        sets.append(gnd)
        sources.append((rows, rng.uniform(0.5, 2.0, len(rows))))
    return sets, sources


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["full", "holes"])
@pytest.mark.parametrize("prec", ["fp64", "mixed", "single"])
def test_device_entry_matches_a_direct_solve(kind, prec):
    g = _raster(kind)
    for log in (False, True):
        # fp32 arithmetic on the device stagnates near 1e-4 of ||b|| for point sources: rtol and the bounds follow
        solver = cb.CUDASolver(rtol=1e-6 if prec == "single" else 1e-10, mixed=prec == "mixed",
                               precision="single" if prec == "single" else "double", f32_compute=prec == "single")
        factor, nodemap = S.construct_raster_factor(g, None, solver, log_transform=log)
        with factor:
            assert factor.operator_form() == ("stencil" if kind == "full" else "windowed")
            A = factor.get_csr().astype(np.float64)
            lab = csgraph.connected_components(A, directed=False)[1]
            rng = np.random.default_rng(11)
            tol = 3e-3 if prec == "single" else 1e-7
            for k in range(1, 10):                 # KT 1/2/4/8, ragged panels
                sets, sources = _columns(nodemap, lab, rng, k, [1, 2, 64])
                w = rng.integers(1, 4, k).astype(np.float64)
                factor.reset_currents()
                cum, mx = np.zeros(factor.n), np.full(factor.n, -np.inf)
                got = factor.solve_grounded(sets, np.arange(k), sources, weight=w, want_volt=True, want_curr=True,
                                            accumulate=True, raise_on_residual=prec != "single")
                assert got["relres"].max() < (1e-3 if prec == "single" else 1e-6)
                sv, V, C = grounded_direct(A, sets, np.arange(k), sources, w, True, log, cum, mx)
                assert np.abs(got["src_volt"] - sv).max() <= tol * np.abs(sv).max()
                assert np.abs(got["volt"] - V).max() <= tol * np.abs(V).max()
                assert np.abs(got["curr"] - C).max() <= 10 * tol * np.abs(C).max()
                dcum, dmx = factor.read_currents()
                if log:
                    # log10 turns the relative error of a tiny current into a large absolute one (and one
                    # side of the 1e-8 cut into -9999): the currents are checked above in linear scale, so
                    # here the accumulation of the device's own per-column currents is checked
                    Cd = np.asarray(got["curr"], dtype=np.float64)
                    L = np.where(Cd > 0, np.log10(np.where(Cd > 0, Cd, 1.0)), -9999.0)
                    cum, mx = L @ w, L.max(axis=1)
                assert np.abs(dcum - cum).max() <= 10 * tol * np.abs(cum).max()
                assert np.abs(dmx - mx).max() <= 10 * tol * np.abs(mx).max()
                for c in range(k):                 # the ground rows hold 0 V exactly
                    assert np.all(got["volt"][sets[c], c] == 0)


@pytest.mark.gpu
@pytest.mark.parametrize("kt", [1, 2, 4, 8])
def test_device_entry_at_each_panel_width(kt):
    g = _raster("holes", seed=7)
    factor, nodemap = S.construct_raster_factor(g, None, cb.CUDASolver(rtol=1e-10, panel_width=kt))
    with factor:
        A = factor.get_csr().astype(np.float64)
        lab = csgraph.connected_components(A, directed=False)[1]
        sets, sources = _columns(nodemap, lab, np.random.default_rng(kt), 2 * kt + 1, [1, 2, 60])
        got = factor.solve_grounded(sets, np.arange(len(sets)), sources, want_volt=True)
        sv, V, _ = grounded_direct(A, sets, np.arange(len(sets)), sources)
        assert np.abs(got["src_volt"] - sv).max() <= 1e-7 * np.abs(sv).max()
        assert np.abs(got["volt"] - V).max() <= 1e-7 * np.abs(V).max()


@pytest.mark.gpu
def test_device_entry_on_a_deep_hierarchy():
    """1100 x 900 full raster: the masked V-cycle over the whole hierarchy with point-sized ground sets"""
    g = 1.0 / np.random.default_rng(13).uniform(1.0, 10.0, (1100, 900))
    factor, nodemap = S.construct_raster_factor(g, None, cb.CUDASolver(rtol=1e-10))
    with factor:
        assert factor.operator_form() == "stencil" and len(factor.levels()) >= 5
        rng = np.random.default_rng(4)
        pts = np.unique(rng.choice(factor.n, 17, replace=False))
        sets = [np.delete(pts, c) for c in range(8)]                   # one-to-all: the other points grounded
        sources = [(pts[c:c + 1], np.ones(1)) for c in range(8)]
        got = factor.solve_grounded(sets, np.arange(8), sources)
        A = factor.get_csr().astype(np.float64).tocsc()
        keep = np.setdiff1d(np.arange(factor.n), pts)
        Akk = spla.splu(A[keep][:, keep].tocsc())
        want = np.zeros(8)
        for c in range(8):                        # block elimination of the live point
            w = Akk.solve(-A[keep][:, [pts[c]]].toarray().ravel())
            want[c] = 1.0 / (A[pts[c], pts[c]] + float((A[pts[c], keep] @ w)[0]))
        assert np.abs(got["src_volt"] - want).max() <= 1e-7 * want.max()


@pytest.mark.gpu
def test_grounded_columns_are_deterministic_and_leave_other_entries_alone():
    g = _raster("full", seed=9)
    factor, nodemap = S.construct_raster_factor(g, None, cb.CUDASolver())
    with factor:
        lab = np.zeros(factor.n, dtype=np.int64)
        rng = np.random.default_rng(2)
        sets, sources = _columns(nodemap, lab, rng, 16, [1, 3, 60])
        src = np.array([s[0] for s in sets[:4]])
        dst = np.array([s[-1] for s in sets[4:8]])
        rsets = [np.arange(r, r + 5) for r in (100, 5000, 9000, 20000)]

        def others():
            factor.reset_currents()
            a = factor.solve_pairs(src, dst, want_volt=True, want_curr=True, accumulate=True)
            b = factor.solve_sources([(np.array([s, d]), np.array([1.0, -1.0])) for s, d in zip(src, dst)], dst,
                                     want_volt=True,
                                     want_curr=True, accumulate=True)
            c = factor.solve_region_pairs(rsets, [0, 1], [2, 3], want_volt=True, want_curr=True, accumulate=True)
            return a, b, c, factor.read_currents()

        before = others()
        perm = np.random.default_rng(8).permutation(16)
        runs = []
        for split in ([np.arange(16)], [np.arange(16)], [np.arange(8, 16), np.arange(8)], [perm]):
            factor.reset_currents()
            SV, V, C = np.zeros(16), np.zeros((factor.n, 16)), np.zeros((factor.n, 16))
            for cols in split:
                p = factor.solve_grounded([sets[c] for c in cols], np.arange(len(cols)), [sources[c] for c in cols],
                                          want_volt=True, want_curr=True, accumulate=True)
                SV[cols], V[:, cols], C[:, cols] = p["src_volt"], p["volt"], p["curr"]
            runs.append((SV, V, C) + tuple(factor.read_currents()))
        for r in runs[1:]:
            for x, y in zip(runs[0][:3], r[:3]):
                assert np.array_equal(x, y)
        for x, y in zip(runs[0][3:], runs[1][3:]):
            assert np.array_equal(x, y)
        after = others()
        for x, y in zip(before[:3], after[:3]):
            for key in x:
                if x[key] is not None:
                    assert np.array_equal(x[key], y[key]), key
        for x, y in zip(before[3], after[3]):
            assert np.array_equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("scenario", ["one-to-all", "all-to-one"])
def test_driver_matches_the_loop_on_the_device(scenario):
    rng = np.random.default_rng(21)
    g = rng.uniform(0.2, 4.0, (120, 90))
    g[rng.random(g.shape) < 0.1] = -9999.0
    g[50, :80] = -9999.0
    pm = np.zeros(g.shape)
    cells = rng.choice(g.size, 12, replace=False)
    pm.ravel()[cells] = np.r_[np.arange(1, 11), 3, 7]
    poly = np.zeros(g.shape)
    poly[10:14, 10:14] = 1
    strengths = np.column_stack([np.arange(1, 13), rng.uniform(0.5, 3.0, 12)])
    for st_ in (None, strengths):                  # variable strengths take one id per cell
        if st_ is not None:
            pm.ravel()[cells] = np.arange(1, 13)
        cfg, inputs, data = _problem(g, pm, poly, st_, scenario, "volt+cur+max", False)
        flags = cb.Flags.from_cfg(cfg)
        got = cb.onetoall_kernel(data, flags, cfg, solver=cb.CUDASolver(rtol=1e-10, onetoall_raster=True))
        want = cb.onetoall_kernel(data, flags, cfg, solver=cb.CUDASolver(rtol=1e-10))
        compare(got, want, rel_r=1e-7, rel_map=1e-6)

"""Pairwise mode with focal regions (src/raster/pairwise.jl:72-135) through `raster_pairwise`: every region
pair batched as a column of cs_b200_solve_region_pairs on one whole-raster operator, the pairs that operator
cannot express taking the reference's per-pair path.

CPU: the driver on a scipy double of `solve_region_pairs` (masked Dirichlet solve, defined here) and on
FakeFactor for the per-pair path, against the oracle's independent per-pair driver and the reference goldens.
GPU: the same on the device, the device entry against the double, determinism, and the existing entry
points left as they were."""

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

REGION_GOLDENS = ["sgVerify3", "sgVerify5", "sgVerify6", "sgVerify8", "sgVerify9", "sgVerify10", "sgVerify11"]


class RegionDouble(FakeFactor):
    """CPU double of B200Factor.solve_region_pairs: per column, L u = 0 off the two sets with u = 0 on
    set_a and u = 1 on set_b, solved directly on the L0 components the sets touch; flux = u.L u;
    v = u / flux; every row of a set carries the set's summed current."""

    def solve_region_pairs(self, sets, set_a, set_b, weight=None, want_volt=False, want_curr=False,
                           accumulate=False, **kw):
        A = self.A
        adj = A.copy()
        adj.data = (adj.data != 0).astype(np.int8)
        adj.eliminate_zeros()
        _, lab = csgraph.connected_components(adj, directed=False)
        k = len(set_a)
        w = np.ones(k) if weight is None else np.asarray(weight, dtype=float)
        V, C, R = np.zeros((self.n, k)), np.zeros((self.n, k)), np.zeros(k)
        for c in range(k):
            a, b = np.asarray(sets[set_a[c]]), np.asarray(sets[set_b[c]])
            fixed = np.zeros(self.n, dtype=bool)
            fixed[a] = fixed[b] = True
            inter = np.nonzero(np.isin(lab, lab[np.r_[a, b]]) & ~fixed)[0]
            u = np.zeros(self.n)
            u[b] = 1.0
            if len(inter):
                rhs = -np.asarray(A[inter][:, b].sum(axis=1)).ravel()
                u[inter] = spla.splu(A[inter][:, inter].tocsc()).solve(rhs)
            flux = float(u @ (A @ u))
            assert flux > 0
            V[:, c] = u / flux
            R[c] = 1.0 / flux
            cur = co.get_node_currents(A, V[:, c])
            for s in (a, b):
                cur[s] = cur[s].sum()
            C[:, c] = cur
            if accumulate:
                val = np.where(cur > 0, np.log10(np.where(cur > 0, cur, 1.0)), -9999.0) if self.log else cur
                self.cum += w[c] * val
                self.mx = np.maximum(self.mx, val)
        return dict(R=R, volt=V if want_volt else None, curr=C if want_curr else None,
                    iters=np.zeros(k, dtype=np.int64), relres=np.zeros(k))


def _double_factory(cellmap, polymap, solver, four_neighbors=False, avg_res=False, log_transform=False):
    nodemap = graph.construct_node_map(cellmap, polymap)
    G = graph.laplacian(graph.construct_graph(cellmap, nodemap, avg_res, four_neighbors))
    return RegionDouble(G, solver, log_transform=log_transform), nodemap


@pytest.fixture
def cpu_doubles(monkeypatch):
    monkeypatch.setattr(S, "construct_cholesky_factor", lambda m, s, **kw: FakeFactor(m, s, **kw))
    monkeypatch.setattr(S, "construct_raster_factor", _double_factory)


def _inputs(cfg, inputs):
    cellmap, polymap, meta, inc = co.load_raster_inputs(cfg, inputs)
    pk = inputs["point_file"]
    points_rc = co.read_point_map(pk[0], pk[1], meta)
    fl = co.cfg_flags(cfg)
    return cb.RasterData(cellmap, polymap, points_rc, None, inc), cb.Flags.from_cfg(cfg), fl


def _run(cfg, inputs, solver=None):
    data, flags, fl = _inputs(cfg, inputs)
    return cb.raster_pairwise(data, flags, cfg, solver=solver or cb.CUDASolver(),
                              four_neighbors=fl["four_neighbors"], avg_res=fl["avg_res"])


def _close(got, want, rel):
    return np.abs(got - want).max() <= rel * max(1.0, np.abs(want).max())


def _written(cmap):
    """postprocess_cum_curmap! (src/utils.jl:114-120), which the reference applies to the shared cumulative and
    max maps when it writes them (src/out.jl:467-479); the oracle's focal-region path returns them unclamped"""
    return np.where(cmap < co.NODATA, co.NODATA, cmap)


def compare(got, want, rel_r=1e-8, rel_map=1e-8):
    assert got.resistances.shape == want.resistances.shape
    assert _close(got.resistances, want.resistances, rel_r)
    assert set(got.curmaps) == set(want.curmaps) and set(got.voltmaps) == set(want.voltmaps)
    for key in want.curmaps:
        assert _close(got.curmaps[key], want.curmaps[key], rel_map), key
    for key in want.voltmaps:
        assert _close(got.voltmaps[key], want.voltmaps[key], rel_map), key
    assert _close(got.cum_curmap, _written(want.cum_curmap), rel_map)
    if want.max_curmap is not None:
        assert _close(got.max_curmap, _written(want.max_curmap), rel_map)


# ---------------------------------------------------------------------------
# randomised comparison with the oracle (CPU)
# ---------------------------------------------------------------------------
MAPS = {"none": {}, "volt": {"write_volt_maps": "True"}, "cur": {"write_cur_maps": "True"},
        "cum_only": {"write_cur_maps": "True", "write_cum_cur_map_only": "True"},
        "max": {"write_cur_maps": "True", "write_max_cur_maps": "True"},
        "all_log_null": {"write_cur_maps": "True", "write_volt_maps": "True", "write_max_cur_maps": "True",
                         "log_transform_maps": "True", "set_null_currents_to_nodata": "True",
                         "set_null_voltages_to_nodata": "True"}}


@st.composite
def region_problems(draw):
    nr, nc = draw(st.integers(4, 8)), draw(st.integers(4, 8))
    rng = np.random.default_rng(draw(st.integers(0, 2**31 - 1)))
    g = rng.uniform(0.2, 4.0, (nr, nc))
    g[rng.random((nr, nc)) < draw(st.sampled_from([0.0, 0.15, 0.3]))] = -9999.0
    poly = None
    if draw(st.booleans()):
        poly = np.zeros((nr, nc))
        poly[rng.random((nr, nc)) < 0.15] = 1
        poly[rng.random((nr, nc)) < 0.08] = 2
        if draw(st.booleans()):                   # a polygon that is NODATA everywhere
            r, c = rng.integers(0, nr), rng.integers(0, nc)
            poly[r, c] = 3
            g[r, c] = -9999.0
    nids = draw(st.integers(2, 4))
    npts = draw(st.integers(nids + 1, nids + 5))
    cells = rng.choice(nr * nc, size=npts, replace=False)
    ids = np.concatenate([np.arange(1, nids + 1), rng.integers(1, nids + 1, npts - nids)])
    pm = np.zeros((nr, nc))
    pm.ravel()[cells] = ids
    inc = None
    if nids >= 3 and draw(st.booleans()):
        pairs = np.array([[1, 2], [2, 3]] if draw(st.booleans()) else [[1, 3]], dtype=np.float64)
        inc = (draw(st.sampled_from(["list_include", "list_exclude"])), pairs)
    maps = draw(st.sampled_from(sorted(MAPS)))
    return g, pm, poly, inc, maps, draw(st.booleans()), draw(st.booleans())


def _cfg_inputs(g, pm, poly, inc, maps, four, avg):
    nr, nc = g.shape
    meta = np.array([nc, nr, 0.0, 0.0, 1.0])
    cfg = {"scenario": "pairwise", "data_type": "raster", "habitat_map_is_resistances": "False",
           "use_polygons": str(poly is not None), "connect_four_neighbors_only": str(four),
           "connect_using_avg_resistances": str(avg), "use_included_pairs": str(inc is not None)}
    cfg.update(MAPS[maps])
    inputs = {"habitat_file": ("grid", g, meta), "point_file": ("grid", pm, meta)}
    if poly is not None:
        inputs["polygon_file"] = ("grid", poly, meta)
    if inc is not None:
        inputs["included_pairs_file"] = (inc[0], inc[1], np.zeros(0))
    return cfg, inputs


@settings(max_examples=150, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(p=region_problems())
def test_region_driver_matches_oracle(cpu_doubles, p):
    cfg, inputs = _cfg_inputs(*p)
    try:
        want = co.raster_pairwise(cfg, inputs)
    except NotImplementedError:
        with pytest.raises(graph.RegionPolymapError):
            _run(cfg, inputs)
        return
    compare(_run(cfg, inputs), want)


def _plan(g, pm, poly, four=False, avg=False):
    cfg, inputs = _cfg_inputs(g, pm, poly, None, "none", four, avg)
    data, _, _ = _inputs(cfg, inputs)
    cellmap, polymap = data.cellmap, data.polymap
    nodemap = graph.construct_node_map(cellmap, polymap)
    adj = graph.construct_graph(cellmap, nodemap, avg, four)
    adj.eliminate_zeros()
    _, comp_of = csgraph.connected_components(adj, directed=False)
    pr = tuple(np.asarray(a) for a in data.points_rc)
    return cfg, inputs, core_mod.plan_region_pairs(cellmap, polymap, pr, set(), nodemap, comp_of)


def _trigger_cases():
    """One raster per fallback trigger: (name, g, point map, polygon map)."""
    g = np.full((5, 6), 1.0)
    base = np.zeros((5, 6))
    base[0, 0] = base[1, 0] = 1                   # region 1: two cells
    base[4, 5] = base[3, 5] = 2                   # region 2: two cells
    out = []
    pm = base.copy(); gg = g.copy(); gg[1, 0] = -9999.0        # a NODATA focal cell outside every polygon
    out.append(("non-node cell", gg, pm, None))
    pm = base.copy(); gg = g.copy(); poly = np.zeros_like(g)
    poly[0, 0] = poly[1, 0] = 7; gg[0, 0] = gg[1, 0] = -9999.0  # region 1 absorbs an all-NODATA polygon
    out.append(("all-NODATA polygon", gg, pm, poly))
    pm = np.zeros_like(g); poly = np.zeros_like(g); poly[2, 2:4] = 5
    pm[2, 2] = 1; pm[2, 3] = 2                     # ids 1 and 2 sit on the same polygon; id 3 is a region
    pm[0, 5] = pm[4, 5] = 3
    out.append(("overlap", g.copy(), pm, poly))
    pm = base.copy(); poly = np.zeros_like(g); poly[4, 5] = 4  # region 2: one point on a polygon of several
    out.append(("error branch", g.copy(), pm, poly))
    pm = base.copy(); poly = np.zeros_like(g); poly[2, 2] = 5; poly[2, 4] = 6
    pm[1, 0] = 0; pm[2, 2] = pm[2, 4] = 1          # region 1: first point off-polygon, two others on polygons 5, 6,
    out.append(("polygons merged away from the first point", g.copy(), pm, poly))   # which the map merges
    return out


@pytest.mark.parametrize("name,g,pm,poly", _trigger_cases(), ids=[c[0] for c in _trigger_cases()])
def test_each_fallback_trigger_takes_the_per_pair_path(cpu_doubles, name, g, pm, poly):
    cfg, inputs, plan = _plan(g, pm, poly)
    assert plan.per_pair[0] == (0, 1) and (0, 1) not in plan.batched
    try:
        want = co.raster_pairwise(cfg, inputs)
    except NotImplementedError:
        assert name == "error branch"
        with pytest.raises(graph.RegionPolymapError):
            _run(cfg, inputs)
        return
    compare(_run(cfg, inputs), want)


@pytest.mark.parametrize("maps", ["all_log_null", "max"])
def test_cumulative_maps_are_clamped_once_like_the_reference(cpu_doubles, maps):
    """Cells outside every node are NODATA in each pair's log-transformed / null-to-nodata map; the shared
    cumulative map is clamped at NODATA when written, so they stay NODATA whatever the number of pairs, on
    the batched and on the per-pair path."""
    g = np.full((6, 8), 1.0)
    g[3, 3] = g[0, 7] = -9999.0                    # cells that are no node
    g[5, 0] = -9999.0                              # makes region 1 take the per-pair path
    pm = np.zeros((6, 8))
    pm[0, 0] = pm[5, 0] = 1
    pm[0, 2] = pm[1, 2] = 2
    pm[5, 5] = pm[4, 5] = 3
    pm[2, 7] = pm[3, 7] = 4
    cfg, inputs, plan = _plan(g, pm, None)
    assert plan.batched and plan.per_pair
    cfg.update(MAPS[maps])
    got = _run(cfg, inputs)
    off = (g <= 0)
    assert got.cum_curmap.min() >= co.NODATA
    if maps == "all_log_null":
        assert np.all(got.cum_curmap[off] == co.NODATA) and np.all(got.max_curmap[off] == co.NODATA)
    assert got.max_curmap.min() >= co.NODATA
    compare(got, co.raster_pairwise(cfg, inputs))


def test_clean_regions_are_batched_and_unconnected_pairs_skipped(cpu_doubles):
    g = np.full((6, 7), 1.5)
    g[:, 3] = -9999.0                              # two components
    pm = np.zeros((6, 7))
    pm[0, 0] = pm[1, 1] = 1
    pm[5, 2] = pm[4, 2] = 2
    pm[0, 6] = pm[5, 6] = 3
    cfg, inputs, plan = _plan(g, pm, None)
    assert plan.batched == [(0, 1)] and plan.unconnected == [(0, 2), (1, 2)] and not plan.per_pair
    compare(_run(cfg, inputs), co.raster_pairwise(cfg, inputs))


@pytest.mark.parametrize("name", REGION_GOLDENS)
def test_region_goldens_on_the_doubles(cpu_doubles, golden, name):
    cfg, inp, exp = co.load_case(golden, name)
    data, flags, fl = _inputs(cfg, inp)
    assert len(data.points_rc[2]) != len(np.unique(data.points_rc[2]))
    r = cb.raster_pairwise(data, flags, cfg, solver=cb.CUDASolver(), four_neighbors=fl["four_neighbors"],
                           avg_res=fl["avg_res"])
    cases.check_raster_pairwise(r, exp)


def test_solve_region_pairs_rejects_bad_arguments_without_a_device():
    lib = _lib.load()
    i64 = lambda *v: np.array(v, dtype=np.int64)
    R = np.zeros(4)

    def call(ptr, rows, a, b, k=None, nsets=None):
        k = len(a) if k is None else k
        nsets = len(ptr) - 1 if nsets is None else nsets
        rc = lib.cs_b200_solve_region_pairs(None, nsets, ptr.ctypes.data, rows.ctypes.data, k, a.ctypes.data,
                                            b.ctypes.data, None, 1e-6, 100, R.ctypes.data, None, None, 0, None,
                                            None)
        return rc, lib.cs_b200_last_error(None).decode()

    ptr, rows = i64(0, 2, 3), i64(4, 7, 9)
    assert call(ptr, rows, i64(0), i64(1), k=0)[0] == _lib.ERR_ARG
    rc, msg = call(i64(0, 2, 2), rows, i64(0), i64(1))
    assert rc == _lib.ERR_ARG and "empty" in msg
    rc, msg = call(ptr, i64(7, 4, 9), i64(0), i64(1))
    assert rc == _lib.ERR_ARG and "sorted" in msg
    rc, msg = call(ptr, i64(4, 4, 9), i64(0), i64(1))
    assert rc == _lib.ERR_ARG and "sorted" in msg
    rc, msg = call(ptr, i64(-1, 7, 9), i64(0), i64(1))
    assert rc == _lib.ERR_ARG and "out of range" in msg
    rc, msg = call(ptr, rows, i64(0), i64(2))
    assert rc == _lib.ERR_ARG and "set index" in msg
    rc, msg = call(i64(0, 2, 3), i64(4, 7, 7), i64(0), i64(1))
    assert rc == _lib.ERR_ARG and "overlap" in msg
    rc, msg = call(ptr, rows, i64(0), i64(0))
    assert rc == _lib.ERR_ARG and "overlap" in msg
    rc, msg = call(ptr, rows, i64(0), i64(1))        # well-formed: only the missing handle is left
    assert rc == _lib.ERR_ARG and "null handle" in msg


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("precond", ["amg", "jacobi"])
@pytest.mark.parametrize("name", REGION_GOLDENS)
def test_region_goldens_on_the_device(golden, name, precond):
    cfg, inp, exp = co.load_case(golden, name)
    want = co.raster_pairwise(cfg, inp)
    got = _run(cfg, inp, cb.CUDASolver(rtol=1e-10, precond=precond))
    compare(got, want, rel_r=1e-8, rel_map=1e-6)
    cases.check_raster_pairwise(_run(cfg, inp, cb.CUDASolver(precond=precond)), exp)


@pytest.mark.gpu
def test_both_paths_run_on_the_device():
    g, pm, poly = _trigger_cases()[0][1:]
    pm = pm.copy()
    pm[0, 3] = pm[1, 3] = 3                        # 2-3 is batched; 1-2 and 1-3 meet region 1's NODATA cell
    cfg, inputs, plan = _plan(g, pm, poly)
    assert plan.batched and plan.per_pair
    cfg.update(MAPS["max"])
    want = co.raster_pairwise(cfg, inputs)
    compare(_run(cfg, inputs, cb.CUDASolver(rtol=1e-10)), want, rel_r=1e-8, rel_map=1e-6)


def _double_of(factor):
    return RegionDouble(factor.get_csr().astype(np.float64), factor.solver, log_transform=False)


def _regions_on(nodemap, rng, count, size, nr, nc):
    """`count` random square regions of side `size` as sorted 0-based row sets of the node map."""
    sets = []
    for _ in range(count):
        r0, c0 = rng.integers(0, nr - size), rng.integers(0, nc - size)
        nodes = np.unique(nodemap[r0:r0 + size, c0:c0 + size])
        nodes = nodes[nodes > 0] - 1
        sets.append(nodes)
    return sets


def _disjoint_pairs(sets, k, rng, lab):
    """k random pairs of disjoint sets that share a component (`lab`: component label per row)"""
    out = []
    while len(out) < k:
        a, b = rng.choice(len(sets), 2, replace=False)
        if not np.intersect1d(sets[a], sets[b]).size and np.intersect1d(lab[sets[a]], lab[sets[b]]).size:
            out.append((int(a), int(b)))
    return np.array([p[0] for p in out]), np.array([p[1] for p in out])


def _raster(kind, seed=5):
    """230 x 160 cells: above the 20 000 rows at which a full raster takes the stencil form and a holey
    one the windowed records, small enough for the direct solves of the double"""
    rng = np.random.default_rng(seed)
    g = 1.0 / rng.uniform(1.0, 10.0, (230, 160))
    if kind == "holes":
        g[rng.random(g.shape) < 0.08] = 0.0
        g[60:64, :] = 0.0                          # a wall: two components
    return g


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["full", "holes"])
@pytest.mark.parametrize("prec", ["fp64", "mixed", "single"])
def test_device_entry_matches_the_double(kind, prec):
    g = _raster(kind)
    solver = cb.CUDASolver(rtol=1e-10, mixed=prec == "mixed", precision="single" if prec == "single" else "double",
                           f32_compute=prec == "single")
    factor, nodemap = S.construct_raster_factor(g, None, solver)
    with factor:
        assert factor.operator_form() == ("stencil" if kind == "full" else "windowed")
        rng = np.random.default_rng(11)
        sets = _regions_on(nodemap, rng, 6, 12, *g.shape)
        wall = nodemap[50:74, 60:100]
        sets.append(np.unique(wall[wall > 0]) - 1)                   # spans the wall (both components)
        big = nodemap[120:220, 40:140]
        sets.append(np.unique(big[big > 0]) - 1)                     # 10^4 cells
        sets = [s for s in sets if len(s)]
        double = _double_of(factor)
        lab = csgraph.connected_components(double.A, directed=False)[1]
        tol = 2e-4 if prec == "single" else 1e-7
        for k in range(1, 10):                     # KT 1/2/4/8, ragged panels
            a, b = _disjoint_pairs(sets, k, rng, lab)
            w = rng.integers(1, 4, k).astype(np.float64)
            factor.reset_currents()
            double.reset_currents()
            got = factor.solve_region_pairs(sets, a, b, weight=w, want_volt=True, want_curr=True, accumulate=True)
            want = double.solve_region_pairs(sets, a, b, weight=w, want_volt=True, want_curr=True, accumulate=True)
            assert np.abs(got["R"] - want["R"]).max() <= tol * np.abs(want["R"]).max()
            assert np.abs(got["volt"] - want["volt"]).max() <= tol * np.abs(want["volt"]).max()
            assert np.abs(got["curr"] - want["curr"]).max() <= 10 * tol * np.abs(want["curr"]).max()
            cum, mx = factor.read_currents()
            assert np.abs(cum - double.cum).max() <= 10 * tol * np.abs(double.cum).max()
            assert np.abs(mx - double.mx).max() <= 10 * tol * np.abs(double.mx).max()
            for c in range(k):                     # the sets hold 0 V / R exactly
                assert np.all(got["volt"][sets[a[c]], c] == 0)
                assert np.all(got["volt"][sets[b[c]], c] == got["volt"][sets[b[c]][0], c])


@pytest.mark.gpu
def test_region_pairs_are_deterministic_and_leave_solve_pairs_alone():
    g = _raster("full", seed=9)
    solver = cb.CUDASolver()
    factor, nodemap = S.construct_raster_factor(g, None, solver)
    with factor:
        rng = np.random.default_rng(2)
        sets = _regions_on(nodemap, rng, 8, 10, *g.shape)
        lab = csgraph.connected_components(factor.get_csr(), directed=False)[1]
        a, b = _disjoint_pairs(sets, 16, rng, lab)
        src = np.array([s[0] for s in sets[:4]])
        dst = np.array([s[-1] for s in sets[4:8]])
        factor.reset_currents()
        before = factor.solve_pairs(src, dst, want_volt=True, want_curr=True, accumulate=True)
        launches_before = factor.stats()["kernel_launches"]
        # a column's result depends on its own data and the width of the panel it is solved in (the PCG
        # reductions are fixed-order trees over that width): calls, offsets, order and the other columns of
        # its panel do not matter.  Every column below sits in a KT = 8 panel.
        perm = np.random.default_rng(8).permutation(16)
        runs = []
        for split in ([np.arange(16)], [np.arange(16)], [np.arange(8, 16), np.arange(8)], [perm]):
            factor.reset_currents()
            R = np.zeros(16)
            V, C = np.zeros((factor.n, 16)), np.zeros((factor.n, 16))
            for cols in split:
                p = factor.solve_region_pairs(sets, a[cols], b[cols], want_volt=True, want_curr=True,
                                              accumulate=True)
                R[cols], V[:, cols], C[:, cols] = p["R"], p["volt"], p["curr"]
            cum, mx = factor.read_currents()
            runs.append((R, V, C, cum, mx))
        for r in runs[1:]:
            for x, y in zip(runs[0][:3], r[:3]):
                assert np.array_equal(x, y)
        for x, y in zip(runs[0][3:], runs[1][3:]):    # the accumulated maps: same pairs in the same order
            assert np.array_equal(x, y)
        factor.reset_currents()
        after = factor.solve_pairs(src, dst, want_volt=True, want_curr=True, accumulate=True)
        assert factor.stats()["kernel_launches"] == launches_before
        for key in ("R", "volt", "curr", "iters"):
            assert np.array_equal(before[key], after[key])


def _exact_R(L, sets, a, b):
    """R of each column by block elimination on ONE sparse LU: F = the rows of every set used, N = the rest
    (one component, so L[N, N] is SPD); u_N = -W u_F with W = L[N, N]^-1 L[N, F], and the Schur complement
    S = L[F, F] - L[F, N] W carries the Dirichlet problem on F and the flux u_F.S u_F."""
    L = L.tocsc()
    F = np.unique(np.concatenate([sets[i] for i in np.r_[a, b]]))
    N = np.setdiff1d(np.arange(L.shape[0]), F)
    W = spla.splu(L[N][:, N].tocsc()).solve(L[N][:, F].toarray())
    Sc = L[F][:, F].toarray() - L[F][:, N] @ W
    pos = {int(r): i for i, r in enumerate(F)}
    R = np.zeros(len(a))
    for c in range(len(a)):
        ia = [pos[int(r)] for r in sets[a[c]]]
        ib = [pos[int(r)] for r in sets[b[c]]]
        free = np.setdiff1d(np.arange(len(F)), ia + ib)
        u = np.zeros(len(F))
        u[ib] = 1.0
        if len(free):
            u[free] = np.linalg.solve(Sc[np.ix_(free, free)], -Sc[np.ix_(free, ib)].sum(axis=1))
        R[c] = 1.0 / (u @ Sc @ u)
    return R


@pytest.mark.gpu
def test_device_entry_on_a_deep_hierarchy():
    """1100 x 900 full raster: the masked V-cycle over the whole hierarchy, one KT = 8 panel, R against a
    direct solve"""
    g = 1.0 / np.random.default_rng(13).uniform(1.0, 10.0, (1100, 900))
    factor, nodemap = S.construct_raster_factor(g, None, cb.CUDASolver(rtol=1e-10))
    with factor:
        assert factor.operator_form() == "stencil" and len(factor.levels()) >= 5
        rng = np.random.default_rng(4)
        sets = [np.unique(nodemap[r:r + 3, c:c + 3]) - 1
                for r, c in zip(rng.integers(0, 1097, 8), rng.integers(0, 897, 8))]
        lab = np.zeros(factor.n, dtype=np.int64)
        a, b = _disjoint_pairs(sets, 8, rng, lab)
        got = factor.solve_region_pairs(sets, a, b)
        want = _exact_R(factor.get_csr().astype(np.float64), sets, a, b)
        assert np.abs(got["R"] - want).max() <= 1e-7 * want.max()

"""Raster pairwise mode with focal points (src/raster/pairwise.jl:14-30, src/core.jl:312-515) on ONE whole-raster
handle: CUDASolver(pairwise_raster=True) routes `raster_pairwise` to core._raster_pairs_device, which takes its
node map and operator from the device, its connected components from cs_b200_components, and solves the pairs of
every component as columns of the same panels.

CPU: the driver on a scipy double of a whole-raster handle (components from csgraph; every column solved
exactly on its own component, every other component left at a non-zero constant as the device leaves it)
against the reference goldens and against the existing per-component driver.
GPU: cs_b200_components against csgraph, bit for bit and repeatably; the driver on the device against the
existing driver and the goldens."""

import ctypes
import types

import numpy as np
import pytest
import scipy.sparse as sp
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
from .test_focal_regions import RegionDouble

REGION_GOLDENS = {"sgVerify3", "sgVerify5", "sgVerify6", "sgVerify8", "sgVerify9", "sgVerify10", "sgVerify11"}
GOLDENS = [f"sgVerify{i}" for i in range(1, 18)]
POINT_GOLDENS = [n for n in GOLDENS if n not in REGION_GOLDENS]


def scipy_components(A):
    """what cs_b200_components computes: csgraph labels of the nonzero (NaN included) off-diagonal pattern"""
    adj = sp.csr_matrix(A, copy=True)
    adj.setdiag(0)
    adj.data = (adj.data != 0).astype(np.int8)
    adj.eliminate_zeros()
    ncomp, lab = csgraph.connected_components(adj, directed=False)
    return ncomp, lab.astype(np.int32)


class WholeRasterDouble(RegionDouble):
    """CPU double of a whole-raster B200Factor (the focal-region double's solve_region_pairs included, for the
    region goldens): columns on a block-diagonal operator.  Each column is solved
    exactly on the component of its reference row (ground deleted); every other component gets a non-zero
    constant, different per column, as the device's shifted solution has there."""

    def components(self):
        return scipy_components(getattr(self, "A0", self.A))

    def _solve(self, rhs_rows, rhs_vals, ref):
        n = self.n
        _, lab = self.components()
        rows = np.nonzero(lab == lab[ref])[0]
        keep = rows[rows != ref]
        b = np.zeros(n)
        np.add.at(b, np.asarray(rhs_rows, dtype=np.int64), np.asarray(rhs_vals, dtype=np.float64))
        v = np.full(n, -0.37 * (1 + ref % 7))
        v[rows] = 0.0
        if len(keep):
            v[keep] = spla.splu(self.A[keep][:, keep].tocsc()).solve(b[keep])
        return v

    def _currents(self, V, weight, want_curr, accumulate):
        k = V.shape[1]
        w = np.ones(k) if weight is None else np.asarray(weight, dtype=float)
        C = np.zeros_like(V)
        if want_curr or accumulate:
            for c in range(k):
                C[:, c] = cur = co.get_node_currents(self.A, V[:, c])
                if accumulate:
                    val = np.where(cur > 0, np.log10(np.where(cur > 0, cur, 1.0)), -9999.0) if self.log else cur
                    self.cum += w[c] * val
                    self.mx = np.maximum(self.mx, val)
        return C

    def solve_pairs(self, src, dst, weight=None, want_volt=False, want_curr=False, accumulate=False, **kw):
        src, dst = np.asarray(src), np.asarray(dst)
        k = len(src)
        V = np.column_stack([self._solve([d], [1.0], s) for s, d in zip(src, dst)]) if k else np.zeros((self.n, 0))
        C = self._currents(V, weight, want_curr, accumulate)
        return dict(R=V[dst, np.arange(k)], volt=V if want_volt else None, curr=C if want_curr else None,
                    iters=np.zeros(k, dtype=np.int64), relres=np.zeros(k))

    def solve_sources(self, columns, ref, probe=None, weight=None, want_volt=False, want_curr=False,
                      accumulate=False, **kw):
        k = len(columns)
        V = np.column_stack([self._solve(r, v, int(g)) for (r, v), g in zip(columns, ref)])
        C = self._currents(V, weight, want_curr, accumulate)
        pv = None if probe is None else V[np.asarray(probe)].T.copy()
        return dict(probe_volt=pv, volt=V if want_volt else None, curr=C if want_curr else None,
                    iters=np.zeros(k, dtype=np.int64), relres=np.zeros(k))


def _double_factory(cellmap, polymap, solver, four_neighbors=False, avg_res=False, log_transform=False):
    nodemap = graph.construct_node_map(cellmap, polymap)
    G = graph.laplacian(graph.construct_graph(cellmap, nodemap, avg_res, four_neighbors))
    return WholeRasterDouble(G, solver, log_transform=log_transform), nodemap.astype(np.int32)


@pytest.fixture
def cpu_doubles(monkeypatch):
    monkeypatch.setattr(S, "construct_cholesky_factor", lambda m, s, **kw: FakeFactor(m, s, **kw))
    monkeypatch.setattr(S, "construct_raster_factor", _double_factory)


def _close(got, want, rel):
    return np.abs(got - want).max() <= rel * max(1.0, np.abs(want).max())


def compare(got, want, rel_r=1e-9, rel_map=1e-9):
    assert got.resistances.shape == want.resistances.shape
    assert _close(got.resistances, want.resistances, rel_r)
    assert set(got.curmaps) == set(want.curmaps) and set(got.voltmaps) == set(want.voltmaps)
    for key in want.curmaps:
        assert _close(got.curmaps[key], want.curmaps[key], rel_map), key
    for key in want.voltmaps:
        assert _close(got.voltmaps[key], want.voltmaps[key], rel_map), key
    assert _close(got.cum_curmap, want.cum_curmap, rel_map)
    assert (got.max_curmap is None) == (want.max_curmap is None)
    if want.max_curmap is not None:
        assert _close(got.max_curmap, want.max_curmap, rel_map)
    assert got.num_solves == want.num_solves


def _golden_inputs(golden, name):
    cfg, inp, exp = co.load_case(golden, name)
    cellmap, polymap, meta, inc = co.load_raster_inputs(cfg, inp)
    pk = inp["point_file"]
    data = cb.RasterData(cellmap, polymap, co.read_point_map(pk[0], pk[1], meta), None, inc)
    return data, cb.Flags.from_cfg(cfg), cfg, co.cfg_flags(cfg), exp


def _run(data, flags, cfg, solver, four=False, avg=False):
    return cb.raster_pairwise(data, flags, cfg, solver=solver, four_neighbors=four, avg_res=avg)


# ---------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", GOLDENS)
def test_goldens_on_the_doubles(cpu_doubles, golden, name, monkeypatch):
    data, flags, cfg, fl, exp = _golden_inputs(golden, name)
    calls = []
    real = core_mod._raster_pairs_device
    monkeypatch.setattr(core_mod, "_raster_pairs_device", lambda *a: calls.append(1) or real(*a))
    r = _run(data, flags, cfg, cb.CUDASolver(pairwise_raster=True), fl["four_neighbors"], fl["avg_res"])
    assert bool(calls) == (name not in REGION_GOLDENS)      # focal regions keep their own driver
    cases.check_raster_pairwise(r, exp)


def test_without_the_flag_the_existing_driver_runs(cpu_doubles, golden, monkeypatch):
    data, flags, cfg, fl, exp = _golden_inputs(golden, "sgVerify1")
    calls = []
    real = core_mod.single_ground_all_pairs
    monkeypatch.setattr(core_mod, "single_ground_all_pairs", lambda *a, **kw: calls.append(1) or real(*a, **kw))
    monkeypatch.setattr(core_mod, "_raster_pairs_device", lambda *a: pytest.fail("device driver without the flag"))
    cases.check_raster_pairwise(_run(data, flags, cfg, cb.CUDASolver(), fl["four_neighbors"], fl["avg_res"]), exp)
    assert calls == [1]


MAPS = {"shortcut": {}, "volt": {"write_volt_maps": "True"}, "cur": {"write_cur_maps": "True"},
        "cum_only": {"write_cur_maps": "True", "write_cum_cur_map_only": "True"},
        "max": {"write_cur_maps": "True", "write_max_cur_maps": "True"},
        "max_only": {"write_max_cur_maps": "True"},
        "log": {"write_cur_maps": "True", "write_max_cur_maps": "True", "log_transform_maps": "True"},
        "null": {"write_cur_maps": "True", "write_volt_maps": "True", "write_max_cur_maps": "True",
                 "set_null_currents_to_nodata": "True", "set_null_voltages_to_nodata": "True"},
        "all_log_null": {"write_cur_maps": "True", "write_volt_maps": "True", "write_max_cur_maps": "True",
                         "log_transform_maps": "True", "set_null_currents_to_nodata": "True",
                         "set_null_voltages_to_nodata": "True"}}


def _lm_polygon_case():
    """a polygon with a NODATA cell in a raster of several components: the NODATA cell moves a node, so the
    component's construct_local_node_map numbers its cells unlike the node map"""
    N = -9999.0
    g = np.array([[1.0, 2.0, N, 1.5, 2.5],
                  [N, N, N, N, N],
                  [N, 3.0, 1.0, N, 2.0],
                  [2.0, 1.0, 0.5, N, 1.0]])
    poly = np.zeros(g.shape)
    poly[2, 0] = poly[3, 2] = 4          # NODATA cell (2, 0) merged with (3, 2)
    return g, poly


@st.composite
def pairwise_problems(draw):
    nr, nc = draw(st.integers(4, 9)), draw(st.integers(4, 9))
    rng = np.random.default_rng(draw(st.integers(0, 2**31 - 1)))
    g = rng.uniform(0.2, 4.0, (nr, nc))
    g[rng.random((nr, nc)) < draw(st.sampled_from([0.0, 0.1, 0.25]))] = -9999.0
    for _ in range(draw(st.integers(0, 2))):                 # NODATA walls: several components
        if draw(st.booleans()):
            g[rng.integers(1, nr - 1), :] = -9999.0
        else:
            g[:, rng.integers(1, nc - 1)] = -9999.0
    poly = None
    if draw(st.booleans()):
        poly = np.zeros((nr, nc))
        poly[rng.random((nr, nc)) < 0.12] = 1
        poly[rng.random((nr, nc)) < 0.08] = 2
        if draw(st.booleans()):                             # a polygon cell on NODATA
            r, c = rng.integers(0, nr), rng.integers(0, nc)
            poly[r, c] = 3
            g[r, c] = -9999.0
            cells = rng.choice(nr * nc, size=2, replace=False)
            poly.ravel()[cells] = 3
    npts = draw(st.integers(2, 8))
    cells = rng.choice(nr * nc, size=npts, replace=True if draw(st.booleans()) else False)
    rr, cc_ = cells % nr + 1, cells // nr + 1
    ids = np.sort(rng.choice(np.arange(1, 40), size=npts, replace=False))
    inc = None
    if npts >= 3 and draw(st.booleans()):
        mode = draw(st.sampled_from(["include", "exclude"]))
        pid = np.sort(rng.choice(ids, size=min(npts, 4), replace=False))
        mat = (rng.random((len(pid), len(pid))) < 0.5).astype(float)
        mat = np.maximum(mat, mat.T)
        inc = types.SimpleNamespace(mode=mode, point_ids=pid, mat=mat)
    maps = draw(st.sampled_from(sorted(MAPS)))
    return (g, poly, (rr, cc_, ids), inc, maps, draw(st.booleans()), draw(st.booleans()),
            draw(st.sampled_from(["double", "single"])), draw(st.booleans()))


def _random_run(p, solver_kw):
    g, poly, prc, inc, maps, four, avg, precision, superpose = p
    cellmap = np.where(g == -9999.0, 0.0, g)
    cfg = dict(MAPS[maps])
    flags = cb.Flags.from_cfg(cfg)
    data = cb.RasterData(cellmap, poly, prc, None, inc)
    solver = cb.CUDASolver(precision=precision, superpose=superpose, **solver_kw)
    return _run(data, flags, cfg, solver, four, avg)


@settings(max_examples=200, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(p=pairwise_problems())
def test_device_driver_matches_the_existing_driver(cpu_doubles, p):
    compare(_random_run(p, dict(pairwise_raster=True)), _random_run(p, {}))


@pytest.mark.parametrize("maps", sorted(MAPS))
def test_a_component_with_its_own_local_map(cpu_doubles, maps, monkeypatch):
    g, poly = _lm_polygon_case()
    cellmap = np.where(g == -9999.0, 0.0, g)
    nodemap = graph.construct_node_map(cellmap, poly)
    _, comp_of = scipy_components(graph.laplacian(graph.construct_graph(cellmap, nodemap, False, False)))
    own = [ci for ci in np.unique(comp_of) if not core_mod._local_map_is_global(nodemap, comp_of, ci, poly)]
    assert own                                               # the case exercises the own-map path
    prc = (np.array([1, 1, 3, 4, 4, 1]), np.array([1, 4, 2, 1, 5, 5]), np.array([1, 2, 3, 4, 5, 6]))
    for superpose in (False, True):
        p = (g, poly, prc, None, maps, False, False, "double", superpose)
        compare(_random_run(p, dict(pairwise_raster=True)), _random_run(p, {}))


def test_points_off_the_graph_and_on_one_node(cpu_doubles):
    g = np.full((5, 6), 1.0)
    g[:, 3] = 0.0
    g[4, 5] = 0.0
    prc = (np.array([1, 1, 5, 2, 3, 5]), np.array([1, 1, 6, 5, 2, 1]), np.array([1, 2, 3, 4, 5, 6]))
    for maps in ("shortcut", "all_log_null"):
        p = (g, None, prc, None, maps, False, False, "double", False)
        got = _random_run(p, dict(pairwise_raster=True))
        compare(got, _random_run(p, {}))
        R = got.resistances[1:, 1:]
        assert R[0, 1] == 0.0 and np.all(R[2, [0, 1, 3, 4, 5]] == -1)   # one node; a point on NODATA


def test_solve_columns_share_panels_across_components(cpu_doubles, monkeypatch):
    g = np.full((6, 9), 1.0)
    g[:, 4] = 0.0
    prc = (np.array([1, 6, 1, 6]), np.array([1, 3, 6, 9]), np.array([1, 2, 3, 4]))
    calls = []
    real = WholeRasterDouble.solve_pairs
    monkeypatch.setattr(WholeRasterDouble, "solve_pairs", lambda self, *a, **kw: calls.append(len(a[0])) or
                        real(self, *a, **kw))
    p = (g, None, prc, None, "cur", False, False, "double", False)
    compare(_random_run(p, dict(pairwise_raster=True)), _random_run(p, {}))
    assert calls == [2]                       # one panel holds the pair of each component


def test_components_rejects_bad_arguments_without_a_device():
    lib = _lib.load()
    assert "cs_b200_components" in _lib.EXPORTED_SYMBOLS
    n = ctypes.c_int64()
    assert lib.cs_b200_components(None, ctypes.byref(n), None) == _lib.ERR_ARG


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
def _raster(kind, nr=120, nc=140, seed=11):
    rng = np.random.default_rng(seed)
    g = rng.uniform(1.0, 10.0, (nr, nc))
    poly = None
    if kind == "holes":
        g[rng.random(g.shape) < 0.3] = 0.0
    elif kind == "walls":
        g[nr // 3, :] = 0.0
        g[:, nc // 2] = 0.0
        g[2 * nr // 3, : nc // 4] = 0.0
    elif kind == "checkerboard":
        g[(np.add.outer(np.arange(nr), np.arange(nc)) % 2) == 1] = 0.0
    elif kind == "polygon_bridge":
        g[:, nc // 2] = 0.0
        poly = np.zeros(g.shape)
        poly[5, nc // 2 - 3] = poly[40, nc // 2 + 4] = 7      # one polygon on both sides of the wall
    elif kind == "serpentine":
        g[:] = 0.0
        g[::2, :] = 1.0
        for r in range(1, nr, 2):
            g[r, nc - 1 if (r // 2) % 2 == 0 else 0] = 1.0
    return g, poly


def _device_labels(g, poly, four=False, solver=None):
    f, nodemap = S.construct_raster_factor(g, poly, solver or cb.CUDASolver(), four_neighbors=four)
    with f:
        ncomp, lab = f.components()
        ncomp2, lab2 = f.components()
        A = f.get_csr()
    assert ncomp == ncomp2 and np.array_equal(lab, lab2)        # repeatable, bit for bit
    return ncomp, lab, A, nodemap


@pytest.mark.gpu
@pytest.mark.parametrize("four", [False, True])
@pytest.mark.parametrize("kind", ["full", "holes", "walls", "checkerboard", "polygon_bridge"])
def test_components_match_csgraph(kind, four):
    g, poly = _raster(kind)
    ncomp, lab, A, nodemap = _device_labels(g, poly, four)
    want_n, want = scipy_components(A)
    assert ncomp == want_n and lab.dtype == np.int32 and np.array_equal(lab, want)
    host = graph.construct_graph(np.where(g > 0, g, 0.0), graph.construct_node_map(g, poly), False, four)
    host.eliminate_zeros()
    assert np.array_equal(lab, csgraph.connected_components(host, directed=False)[1])
    if kind == "checkerboard" and four:
        assert ncomp == np.count_nonzero(nodemap)               # only the diagonals connect
    if kind == "polygon_bridge":
        assert ncomp == 1


@pytest.mark.gpu
def test_components_of_a_long_serpentine():
    g, _ = _raster("serpentine", nr=1999, nc=2000)
    ncomp, lab, A, _ = _device_labels(g, None, four=True)
    assert ncomp == 1 and not lab.any()
    ncomp, lab, A, _ = _device_labels(g, None, four=False)
    assert np.array_equal(lab, scipy_components(A)[1])


@pytest.mark.gpu
def test_components_of_the_bench_raster_with_walls():
    rng = np.random.default_rng(42)
    g = 1.0 / rng.uniform(1.0, 10.0, (3163, 3163))
    g[1000, :] = g[:, 2000] = g[2500, :2000] = 0.0
    ncomp, lab, A, _ = _device_labels(g, None)
    want_n, want = scipy_components(A)
    assert ncomp == want_n == 5 and np.array_equal(lab, want)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2])
def test_components_of_csr_handles(seed):
    L = sp.csr_matrix(graph.power_law_laplacian(20000, seed=seed))
    rng = np.random.default_rng(seed)
    n = L.shape[0]
    iso = rng.choice(n, 300, replace=False)                      # isolated nodes: their rows and columns 0
    keep = np.ones(n)
    keep[iso] = 0.0
    D = sp.diags(keep)
    L = (D @ L @ D + sp.diags(1.0 - keep)).tocsr()
    L = L.tocoo()
    L.data[(rng.random(L.nnz) < 0.05) & (L.row != L.col)] = 0.0   # stored zeros are no edges
    L = sp.csr_matrix((L.data, (L.row, L.col)), shape=L.shape)
    L.sort_indices()
    assert (L.data == 0).any()
    with cb.B200Factor(L, cb.CUDASolver(precond="jacobi")) as f:
        ncomp, lab = f.components()
        want_n, want = scipy_components(L)
        assert ncomp == want_n and np.array_equal(lab, want)
        mask = np.zeros(n, dtype=np.uint8)
        mask[rng.choice(n, 50, replace=False)] = 1
        f.set_grounds(finite=np.full(n, 0.01), dirichlet=mask)  # identity rows do not split components
        ncomp2, lab2 = f.components()
        assert ncomp2 == ncomp and np.array_equal(lab2, lab)


@pytest.mark.gpu
@pytest.mark.parametrize("precond", ["amg", "jacobi"])
@pytest.mark.parametrize("name", POINT_GOLDENS)
def test_goldens_on_the_device(golden, name, precond):
    data, flags, cfg, fl, exp = _golden_inputs(golden, name)
    run = lambda **kw: _run(data, flags, cfg, cb.CUDASolver(precond=precond, **kw), fl["four_neighbors"],
                            fl["avg_res"])
    got = run(pairwise_raster=True)
    cases.check_raster_pairwise(got, exp)
    compare(run(pairwise_raster=True, rtol=1e-10), run(rtol=1e-10), rel_r=1e-8, rel_map=1e-8)


@pytest.mark.gpu
@settings(max_examples=25, deadline=None, derandomize=True)
@given(p=pairwise_problems())
def test_device_driver_matches_the_existing_driver_on_the_device(p):
    p = p[:7] + ("double",) + p[8:]
    compare(_random_run(p, dict(pairwise_raster=True, rtol=1e-10)), _random_run(p, dict(rtol=1e-10)),
            rel_r=1e-8, rel_map=1e-8)


@pytest.mark.gpu
@pytest.mark.parametrize("maps", ["shortcut", "all_log_null", "max"])
def test_multi_component_raster_on_the_device(maps):
    rng = np.random.default_rng(7)
    g = rng.uniform(1.0, 10.0, (160, 200))
    g[:, 100] = 0.0
    g[80, :] = 0.0
    g[rng.random(g.shape) < 0.05] = 0.0
    cells = rng.choice(g.size, 14, replace=False)
    prc = (cells % 160 + 1, cells // 160 + 1, np.arange(1, 15))
    p = (g, None, prc, None, maps, False, False, "double", False)
    got = _random_run(p, dict(pairwise_raster=True, rtol=1e-10))
    # the whole-raster and the per-component hierarchies stop at different iterates of a 32 000-node component,
    # and the maps (log10 of small currents above all) carry those last digits: they are held to 1e-6 of their
    # maximum, as the focal-region driver's are, R to 1e-8
    compare(got, _random_run(p, dict(rtol=1e-10)), rel_r=1e-8, rel_map=1e-6)

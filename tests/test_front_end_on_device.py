"""CUDASolver(front_end_on_device=True): raster advanced mode, one-to-all / all-to-one (onetoall_raster) and focal
regions take their node map, component labels and advanced mode's columns from the whole-raster handle
(B200Factor.components, B200Factor.plan_advanced / cs_b200_plan_advanced) instead of a host graph.

CPU: doubles of the handle (subclasses of the existing ones, with components() and plan_advanced() restated from
the host functions); with the switch on the host graph, labels and node values are never built outside the
documented fallbacks, and every output equals the switch-off output exactly; argument rejection without a device;
the new kernels have no stack and no spills.
GPU: cs_b200_plan_advanced against the host restatement bit for bit, the operator and a solve after it against
set_grounds from the host, repeats, errors, and the three drivers end to end with the switch on against off."""

import ctypes
import os
import subprocess

import numpy as np
import pytest
from hypothesis import HealthCheck, given, settings, strategies as st
from scipy.sparse import csgraph

import circuitscape_b200 as cb
from circuitscape_b200 import _lib, graph
from circuitscape_b200 import core as core_mod
from circuitscape_b200 import solver as S
from oracle import circuitscape_oracle as co

from . import cases
from .fake_factor import FakeFactor
from .test_advanced_raster import MG, POLICIES, AdvancedDouble, advanced_rasters
from .test_focal_regions import REGION_GOLDENS, _cfg_inputs, _inputs, region_problems
from .test_onetoall_device import ONE_TO_ALL, GroundedDouble, _problem, onetoall_problems
from .test_raster_pairwise_device import WholeRasterDouble

_construct_graph = graph.construct_graph          # the doubles' own operator, kept from the monkeypatches
ON = dict(front_end_on_device=True)


def _labels(A):
    adj = A.copy().tocsr()
    adj.setdiag(0)
    adj.eliminate_zeros()
    return csgraph.connected_components(adj, directed=False)


def plan_restated(nodemap, source_map, ground_map, policy, comp_of):
    """cs_b200_plan_advanced restated from sources_and_grounds_from_maps, resolve_conflicts and raster_advanced's
    column loop: -> (plan dict as B200Factor.plan_advanced returns it, s, g, f)."""
    nodemap = np.asarray(nodemap, dtype=np.int64)
    comp_of = np.asarray(comp_of, dtype=np.int64)
    n = len(comp_of)
    s, g = np.zeros(n), np.zeros(n)
    for target, cmap in ((s, source_map), (g, ground_map)):
        cm = np.asarray(cmap, dtype=np.float64)
        sel = (cm != 0) & (nodemap != 0)
        np.add.at(target, nodemap[sel] - 1, cm[sel])   # boolean selection: row-major, np.add.at's order
    f = np.where(np.isfinite(g), g, 0.0)
    both = (s != 0) & (g != 0)
    if policy in ("rmvsrc", "rmvall"):
        s[both] = 0
    elif policy == "rmvgnd":
        g[both] = 0
    g[np.isinf(g) & (s > 0)] = 0
    col_comp, sets, srcs, nsolved = [], [], [], 0
    col_of_row = np.full(n, -1, dtype=np.int32)
    ncomp = int(comp_of.max()) + 1 if n else 0
    order = np.argsort(comp_of, kind="stable")
    for c, rows in enumerate(np.split(order, np.cumsum(np.bincount(comp_of, minlength=ncomp))[:-1]) if n else []):
        if s[rows].sum() == 0 or g[rows].sum() == 0:       # numpy's pairwise sums, as raster_advanced's
            continue
        nsolved += 1
        inf = g[rows] == np.inf
        src = rows[(s[rows] != 0) & ~inf]
        if not len(src):
            continue
        col_of_row[rows] = len(col_comp)
        col_comp.append(c)
        sets.append(rows[inf])
        srcs.append(src)
    ptr = lambda parts: np.r_[0, np.cumsum([len(p) for p in parts])].astype(np.int64)
    cat = lambda parts: np.concatenate(parts).astype(np.int64) if parts else np.zeros(0, dtype=np.int64)
    src_rows = cat(srcs)
    plan = dict(nsolved=nsolved, finite_applied=bool(np.any(f != 0)), col_comp=np.array(col_comp, dtype=np.int64),
                set_ptr=ptr(sets), set_rows=cat(sets), src_ptr=ptr(srcs), src_rows=src_rows, src_vals=s[src_rows],
                col_of_row=col_of_row)
    return plan, s, g, f


class _FrontEnd:
    """components() and plan_advanced() of a whole-raster handle, on a double"""

    def components(self):
        return _labels(getattr(self, "A0", self.A))

    def plan_advanced(self, nodemap, source_map, ground_map, policy):
        plan, _, _, f = plan_restated(nodemap, source_map, ground_map, policy, self.components()[1])
        if plan["finite_applied"]:
            self.set_grounds(finite=f)
        return plan


class FrontAdvancedDouble(_FrontEnd, AdvancedDouble):
    pass


class FrontGroundedDouble(_FrontEnd, GroundedDouble):
    pass


class FrontRegionDouble(_FrontEnd, WholeRasterDouble):
    pass


def _factory(cls):
    def make(cellmap, polymap, solver, four_neighbors=False, avg_res=False, log_transform=False):
        nodemap = graph.construct_node_map(cellmap, polymap)
        G = graph.laplacian(_construct_graph(cellmap, nodemap, avg_res, four_neighbors))
        return cls(G, solver, log_transform=log_transform), nodemap
    return make


@pytest.fixture
def doubles(monkeypatch):
    """state["use"](cls): the whole-raster handle becomes a `cls` double; while state["on"] is set the host front
    end (construct_graph, _component_labels, sources_and_grounds_from_maps) fails the test"""
    monkeypatch.setattr(S, "construct_cholesky_factor", lambda m, s, **kw: FakeFactor(m, s, **kw))
    monkeypatch.setattr(S, "multiple_solve", lambda s, m, b: FakeFactor(m, s).solve_rhs(np.asarray(b))[0])
    state = {"on": False}
    for mod, name in ((graph, "construct_graph"), (core_mod, "_component_labels"),
                      (core_mod, "sources_and_grounds_from_maps")):
        real = getattr(mod, name)

        def guarded(*a, _real=real, _name=name, **kw):
            if state["on"]:
                pytest.fail(f"{_name} with the front end on the device")
            return _real(*a, **kw)
        monkeypatch.setattr(mod, name, guarded)

    def use(cls):
        monkeypatch.setattr(S, "construct_raster_factor", _factory(cls))
    state["use"] = use
    return state


def _same(a, b):
    """two driver outputs bit for bit: every array field, dict of maps and number"""
    fields = [k for k in vars(b) if k not in ("stats",)]
    assert set(vars(a)) == set(vars(b))
    for k in fields:
        x, y = getattr(a, k), getattr(b, k)
        if isinstance(y, dict):
            assert set(x) == set(y), k
            for key in y:
                assert np.array_equal(x[key], y[key]), (k, key)
        elif isinstance(y, np.ndarray) or isinstance(x, np.ndarray):
            assert np.array_equal(np.asarray(x), np.asarray(y)), k
        else:
            assert x == y, k


def _advanced(g, poly, src, gm, policy, four, avg, solver):
    data = cb.RasterData(g, poly, None, source_map=src, ground_map=gm)
    return cb.raster_advanced(data, cb.Flags(is_raster=True, is_advanced=True), {"remove_src_or_gnd": policy},
                              solver=solver, four_neighbors=four, avg_res=avg)


def _advanced_on_off(doubles, *args, **solver_kw):
    doubles["use"](FrontAdvancedDouble)
    off = _advanced(*args, cb.CUDASolver(**solver_kw))
    doubles["on"] = True
    on = _advanced(*args, cb.CUDASolver(**ON, **solver_kw))
    doubles["on"] = False
    _same(on, off)
    return on


def _mg(golden, name):
    cfg, inp, _ = co.load_case(golden, name)
    fl = co.cfg_flags(cfg)
    cellmap, polymap, meta, _ = co.load_raster_inputs(cfg, inp)
    src, gm = co.read_source_and_ground_maps(cfg, inp, meta)
    return cellmap, polymap, src, gm, cfg.get("remove_src_or_gnd", "keepall"), fl["four_neighbors"], fl["avg_res"]


def walls_case(nr=40, nc=60, step=4, seed=3):
    """NODATA walls every `step` rows and columns: ((nr - 1) // step + 1) * ((nc - 1) // step + 1) components"""
    rng = np.random.default_rng(seed)
    g = rng.uniform(0.5, 3.0, (nr, nc))
    g[step - 1::step, :] = 0.0
    g[:, step - 1::step] = 0.0
    src = np.where(rng.random(g.shape) < 0.1, rng.choice([-1.0, 1.0], g.shape), 0.0)
    gm = np.where(rng.random(g.shape) < 0.1, rng.uniform(0.2, 1.0, g.shape), 0.0)
    gm[rng.random(g.shape) < 0.05] = np.inf
    return g, src, gm


def kinds_case():
    """one component per case between NODATA walls: cancelling sources (+1 / -1), a component whose sources all sit
    on Inf grounds (solved, no column), finite grounds only, Inf and finite grounds on one polygon node, sources only"""
    g = np.ones((14, 6))
    g[[2, 5, 8, 11], :] = 0.0
    src, gm = np.zeros(g.shape), np.zeros(g.shape)
    poly = np.zeros(g.shape)
    src[0, 0], src[1, 5], gm[0, 3] = 1.0, -1.0, 0.5          # cancelling: not solved
    src[3, 1], gm[3, 1], gm[4, 4] = 1.0, np.inf, 0.7        # ... the source on its Inf ground: solved, no column
    src[6, 2], gm[7, 4] = 2.0, 0.3                          # finite grounds only
    poly[9, 0] = poly[10, 3] = 5                            # one polygon node: an Inf and a finite ground cell
    src[9, 5], gm[9, 0], gm[10, 3] = 1.5, np.inf, 0.4
    src[12, 1] = 1.0                                        # sources only
    return g, poly, src, gm


def decimal_case(nr=61, nc=700, seed=5):
    """every other row NODATA, the rest cut into segments of 1 to ~600 cells (one component each, rows ascending
    from left to right); each segment has three one-decimal sources that cancel in decimal, a, b and -(a + b), and
    one finite ground.  Whether a component is solved then depends on the summation order: numpy's pairwise sum
    and a sequential sum disagree on a good share of them."""
    rng = np.random.default_rng(seed)
    g = rng.uniform(0.5, 3.0, (nr, nc))
    g[1::2, :] = 0.0
    src, gm = np.zeros(g.shape), np.zeros(g.shape)
    for r in range(0, nr, 2):
        cuts = np.sort(rng.choice(np.arange(1, nc - 1), size=rng.integers(0, 6), replace=False))
        g[r, cuts] = 0.0
        for a, b in zip(np.r_[0, cuts + 1], np.r_[cuts, nc]):
            if b - a < 3:
                continue
            cells = rng.choice(np.arange(a, b), size=3, replace=False)
            x, y = np.round(rng.uniform(-0.9, 0.9, 2), 1)
            src[r, cells] = x, y, -np.round(x + y, 1)
            gm[r, rng.integers(a, b)] = 0.5
    return g, src, gm


# ---------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("name", MG)
def test_advanced_goldens_switch_on_equals_off(doubles, golden, name):
    on = _advanced_on_off(doubles, *_mg(golden, name))
    assert on.num_solves > 0


@settings(max_examples=150, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(p=advanced_rasters())
def test_advanced_random_rasters_switch_on_equals_off(doubles, p):
    g, poly, src, gm, policy, four, avg = p
    if graph.construct_node_map(g, poly).max() == 0:
        return
    _advanced_on_off(doubles, g, poly, src, gm, policy, four, avg)


@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("four", [False, True])
def test_advanced_walls_and_component_kinds(doubles, policy, four):
    g, src, gm = walls_case()
    ncomp = _labels(graph.laplacian(_construct_graph(g, graph.construct_node_map(g, None), False, four)))[0]
    assert ncomp >= 50
    _advanced_on_off(doubles, g, None, src, gm, policy, four, False)
    g, poly, src, gm = kinds_case()
    on = _advanced_on_off(doubles, g, poly, src, gm, policy, four, True)
    assert on.num_solves >= 2


def test_advanced_decimal_cancellation_follows_numpys_sum(doubles):
    """a 16-node component whose 1st, 9th and 2nd rows carry 0.3, 0.4 and -0.7: numpy's pairwise sum is 0 (not
    solved), a sequential one is 5.55e-17"""
    g = np.ones((1, 16))
    src, gm = np.zeros(g.shape), np.zeros(g.shape)
    src[0, 0], src[0, 8], src[0, 1] = 0.3, 0.4, -0.7
    gm[0, 5] = 0.5
    on = _advanced_on_off(doubles, g, None, src, gm, "keepall", False, False)
    assert on.num_solves == 0 and np.array_equal(on.result, [[-1.0]])
    g, src, gm = decimal_case(21, 300)
    _advanced_on_off(doubles, g, None, src, gm, "keepall", False, False)


@pytest.mark.parametrize("policy", ["", "remove_nothing"])
def test_advanced_unknown_policy_is_keepall(doubles, policy):
    g, poly, src, gm = kinds_case()
    on = _advanced_on_off(doubles, g, poly, src, gm, policy, False, False)
    _same(on, _advanced(g, poly, src, gm, "keepall", False, False, cb.CUDASolver(**ON)))


def test_advanced_own_map_component(doubles):
    """a merged polygon with a NODATA cell: construct_local_node_map numbers the component unlike the node map"""
    g = np.array([[1.0, 0.0, 2.0], [0.0, 1.5, 0.0], [2.0, 1.0, 0.0], [0.0, 1.2, 3.0]])
    poly = np.array([[0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0.]])
    poly[0, 2] = poly[1, 1] = poly[1, 0] = 4
    src, gm = np.zeros(g.shape), np.zeros(g.shape)
    src[3, 2], gm[0, 0], gm[2, 0] = 1.0, np.inf, 0.5
    _advanced_on_off(doubles, g, poly, src, gm, "keepall", False, False)


def test_advanced_nothing_solved(doubles, monkeypatch):
    g, poly, src, gm = kinds_case()
    keep = np.zeros(g.shape, dtype=bool)
    keep[:2] = True                                         # the cancelling component only
    on = _advanced_on_off(doubles, np.where(keep, g, 0.0), None, np.where(keep, src, 0.0),
                          np.where(keep, gm, 0.0), "keepall", False, False)
    assert on.num_solves == 0 and np.array_equal(on.result, [[-1.0]])


def _onetoall(data, cfg, four, solver):
    return cb.onetoall_kernel(data, cb.Flags.from_cfg(cfg), cfg, solver=solver, four_neighbors=four,
                              avg_res=cfg.get("connect_using_avg_resistances", "False") in ("True", "true"))


def _onetoall_on_off(doubles, monkeypatch, data, cfg, four):
    doubles["use"](FrontGroundedDouble)
    off = _onetoall(data, cfg, four, cb.CUDASolver(onetoall_raster=True))
    plans = []
    real = core_mod.plan_onetoall
    monkeypatch.setattr(core_mod, "plan_onetoall", lambda *a, **kw: plans.append(real(*a, **kw)) or plans[-1])
    graphs = []
    monkeypatch.setattr(graph, "construct_graph", lambda *a, _g=graph.construct_graph, **kw: graphs.append(1) or _g(*a, **kw))
    labels = []
    monkeypatch.setattr(core_mod, "_component_labels",
                        lambda *a, _l=core_mod._component_labels, **kw: labels.append(1) or _l(*a, **kw))
    on = _onetoall(data, cfg, four, cb.CUDASolver(onetoall_raster=True, **ON))
    _same(on, off)
    if data.included_pairs is None:
        assert not labels                                   # the labels come from the handle
        assert bool(graphs) == bool(plans[0].per_iteration)  # the host graph only for the loop's iterations
    return on


@pytest.mark.parametrize("name", ONE_TO_ALL)
def test_onetoall_goldens_switch_on_equals_off(doubles, monkeypatch, golden, name):
    data, flags, cfg, exp = cases.onetoall_problem(golden, name)
    on = _onetoall_on_off(doubles, monkeypatch, data, cfg, co.cfg_bool(cfg, "connect_four_neighbors_only"))
    cases.check_onetoall(on, exp, flags)


@settings(max_examples=100, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(p=onetoall_problems())
def test_onetoall_random_switch_on_equals_off(doubles, monkeypatch, p):
    g, pm, poly, strengths, scenario, maps, four = p
    cfg, inputs, data = _problem(g, pm, poly, strengths, scenario, maps, four)
    try:
        co.raster_one_to_all(cfg, inputs)
    except (ValueError, IndexError):
        return
    with monkeypatch.context() as m:
        _onetoall_on_off(doubles, m, data, cfg, four)


@pytest.mark.parametrize("scenario", ["one-to-all", "all-to-one"])
def test_onetoall_include_list_takes_the_loop(doubles, monkeypatch, scenario):
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
    data = cb.RasterData(cellmap, polymap, data.points_rc, None, incp)
    _onetoall_on_off(doubles, monkeypatch, data, cfg, False)


def _regions(cfg, inputs, solver):
    data, flags, fl = _inputs(cfg, inputs)
    return cb.raster_pairwise(data, flags, cfg, solver=solver, four_neighbors=fl["four_neighbors"],
                              avg_res=fl["avg_res"])


def _regions_on_off(doubles, monkeypatch, cfg, inputs):
    doubles["use"](FrontRegionDouble)
    off = _regions(cfg, inputs, cb.CUDASolver())
    plans = []
    real = core_mod.plan_region_pairs
    monkeypatch.setattr(core_mod, "plan_region_pairs", lambda *a, **kw: plans.append(real(*a, **kw)) or plans[-1])
    graphs = []
    monkeypatch.setattr(graph, "construct_graph", lambda *a, _g=graph.construct_graph, **kw: graphs.append(1) or _g(*a, **kw))
    monkeypatch.setattr(core_mod, "_component_labels", lambda *a, **kw: pytest.fail("host labels"))
    on = _regions(cfg, inputs, cb.CUDASolver(**ON))
    _same(on, off)
    assert bool(graphs) == bool(plans[0].per_pair)          # the host graph only for the per-pair path
    return on


@pytest.mark.parametrize("name", REGION_GOLDENS)
def test_region_goldens_switch_on_equals_off(doubles, monkeypatch, golden, name):
    cfg, inp, exp = co.load_case(golden, name)
    _regions_on_off(doubles, monkeypatch, cfg, inp)


@settings(max_examples=100, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(p=region_problems())
def test_region_random_switch_on_equals_off(doubles, monkeypatch, p):
    cfg, inputs = _cfg_inputs(*p)
    try:
        co.raster_pairwise(cfg, inputs)
    except NotImplementedError:
        return
    with monkeypatch.context() as m:
        _regions_on_off(doubles, m, cfg, inputs)


def test_restatement_sums_in_row_major_order():
    """one polygon node over three cells 1e16, 1, -1e16 (row-major order): 0, not 1"""
    nodemap = np.array([[1, 1], [1, 2]])
    src = np.array([[1e16, 1.0], [-1e16, 0.0]])
    plan, s, _, _ = plan_restated(nodemap, src, np.zeros((2, 2)), "keepall", np.array([0, 1]))
    assert s[0] == 0.0
    src = np.array([[1e16, -1e16], [1.0, 0.0]])
    plan, s, _, _ = plan_restated(nodemap, src, np.zeros((2, 2)), "keepall", np.array([0, 1]))
    assert s[0] == 1.0


def test_plan_entries_reject_bad_arguments_without_a_device():
    lib = _lib.load()
    for name in ("cs_b200_plan_advanced", "cs_b200_read_advanced_plan"):
        assert name in _lib.EXPORTED_SYMBOLS
    i64 = [ctypes.c_int64() for _ in range(4)]
    fin = ctypes.c_int()
    nm = np.ones((2, 2), dtype=np.int32)
    m = np.zeros((2, 2))
    assert lib.cs_b200_plan_advanced(None, 2, 2, _lib._ptr(nm), _lib._ptr(m), _lib._ptr(m), _lib.F64, 0,
                                     *(ctypes.byref(x) for x in i64), ctypes.byref(fin)) == _lib.ERR_ARG
    assert lib.cs_b200_read_advanced_plan(None, *([None] * 7)) == _lib.ERR_ARG


def test_new_kernels_have_no_stack_and_no_spills():
    obj = os.path.join(os.path.dirname(_lib.LIB_PATH), "obj", "cs_b200.o")
    out = subprocess.run([os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump"),
                          "--dump-resource-usage", obj], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    found = 0
    for i, line in enumerate(lines):
        if "Function" in line and "k_adv_" in line:
            found += 1
            assert "STACK:0 " in lines[i + 1] and "LOCAL:0 " in lines[i + 1], (line, lines[i + 1])
    assert found == 11     # cells, rows, 4 node_values, counts, sums, ptrs, mark, widen


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
def _raster(kind, nr=120, nc=140, seed=7, dtype=np.float64):
    rng = np.random.default_rng(seed)
    g = rng.uniform(1.0, 10.0, (nr, nc))
    poly = None
    src = np.where(rng.random(g.shape) < 0.02, rng.uniform(0.5, 2.0, g.shape), 0.0)
    src[rng.random(g.shape) < 0.01] = -1.0
    gm = np.where(rng.random(g.shape) < 0.02, rng.uniform(0.1, 1.0, g.shape), 0.0)
    gm[rng.random(g.shape) < 0.005] = np.inf
    if kind == "holes":
        g[rng.random(g.shape) < 0.3] = 0.0
    elif kind == "walls":
        g[::6, :] = 0.0
        g[:, ::6] = 0.0
    elif kind == "poly":
        poly = np.zeros(g.shape)
        poly[3, 4] = poly[3, 90] = poly[70, 10] = 9           # one node: 1e16, 1, -1e16 in row-major order
        src[3, 4], src[3, 90], src[70, 10] = 1e16, 1.0, -1e16
        poly[20, 20] = poly[21, 50] = 4                        # one node: Inf and finite ground
        gm[20, 20], gm[21, 50] = np.inf, 0.25
        poly[50:54, 60:64] = 2
    elif kind == "no_finite":
        gm = np.where(gm != 0, np.inf, 0.0)
    elif kind == "decimal":
        g, src, gm = decimal_case()
    return g, poly, src.astype(dtype), gm.astype(dtype)


def _device_plan(g, poly, src, gm, policy, solver=None):
    f, nodemap = S.construct_raster_factor(g, poly, solver or cb.CUDASolver())
    return f, np.asarray(nodemap), f.plan_advanced(nodemap, src, gm, policy)


def _plans_equal(a, b):
    for k in b:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
        if isinstance(b[k], np.ndarray) and b[k].dtype.kind == "f":
            assert np.asarray(a[k]).tobytes() == b[k].tobytes(), k


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["full", "holes", "walls", "poly", "no_finite", "decimal"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("policy", POLICIES)
def test_plan_matches_the_host_restatement(kind, dtype, policy):
    g, poly, src, gm = _raster(kind, dtype=dtype)
    f, nodemap, got = _device_plan(g, poly, src, gm, policy)
    with f:
        ncomp, lab = f.components()
        if kind == "walls":
            assert ncomp >= 300
        want, s_, g_, fin = plan_restated(nodemap, src, gm, policy, lab)
        if kind == "decimal" and dtype == np.float64 and policy == "keepall":
            # the case tells numpy's summation tree from a sequential sum on many components
            seq = [c for c in range(ncomp) if np.cumsum(s_[lab == c])[-1] != 0]
            pair = [c for c in range(ncomp) if s_[lab == c].sum() != 0]
            assert len(set(seq) ^ set(pair)) >= 10
        _plans_equal(got, want)
        A_dev = f.get_csr()
        form = f.operator_form()
        again = f.plan_advanced(nodemap, src, gm, policy)        # repeats, on the grounded handle too
        _plans_equal(again, got)
        assert np.array_equal(f.get_csr().data, A_dev.data)
    # the operator and a solve against set_grounds(finite=f) from the host
    h, _ = S.construct_raster_factor(g, poly, cb.CUDASolver())
    with h:
        A0 = h.get_csr()
        form0 = h.operator_form()
        if want["finite_applied"]:
            h.set_grounds(finite=fin)
        A_host = h.get_csr()
        assert A_host.data.tobytes() == A_dev.data.tobytes()
        assert np.array_equal(A_host.indices, A_dev.indices) and np.array_equal(A_host.indptr, A_dev.indptr)
        assert form == h.operator_form()
        if not want["finite_applied"]:
            assert A0.data.tobytes() == A_dev.data.tobytes() and form == form0
        k = min(len(want["col_comp"]), 8)
        if k:
            sets, gset = [], []                                  # -1: finite grounds only
            for j in range(k):
                rows = want["set_rows"][want["set_ptr"][j]:want["set_ptr"][j + 1]]
                gset.append(len(sets) if len(rows) else -1)
                if len(rows):
                    sets.append(rows)
            srcs = [(want["src_rows"][want["src_ptr"][j]:want["src_ptr"][j + 1]],
                     want["src_vals"][want["src_ptr"][j]:want["src_ptr"][j + 1]]) for j in range(k)]
            if all(x >= 0 for x in gset) or want["finite_applied"]:
                a = h.solve_advanced(sets, gset, srcs, want_volt=True, want_curr=True)
                f2, _, p2 = _device_plan(g, poly, src, gm, policy)
                with f2:
                    b = f2.solve_advanced(sets, gset, srcs, want_volt=True, want_curr=True)
                assert a["volt"].tobytes() == b["volt"].tobytes() and a["curr"].tobytes() == b["curr"].tobytes()


@pytest.mark.gpu
def test_plan_on_a_3163_raster_with_a_ground_band():
    nr = nc = 3163
    rng = np.random.default_rng(1)
    g = rng.uniform(1.0, 10.0, (nr, nc))
    src = np.zeros(g.shape)
    src[rng.integers(0, nr, 50), rng.integers(0, nc, 50)] = 1.0
    gm = np.zeros(g.shape)
    gm[:, -10:] = 0.5
    f, nodemap, got = _device_plan(g, None, src, gm, "keepall")
    with f:
        lab = f.components()[1]
        assert f.operator_form() == "stencil"
    want = plan_restated(nodemap, src, gm, "keepall", lab)[0]
    _plans_equal(got, want)
    assert got["finite_applied"] and len(got["col_comp"]) == 1


@pytest.mark.gpu
def test_plan_rejects_bad_node_maps_and_a_read_without_a_plan():
    g, poly, src, gm = _raster("full", 30, 40)
    f, nodemap = S.construct_raster_factor(g, poly, cb.CUDASolver())
    with f:
        A0 = f.get_csr()
        for bad in (np.where(nodemap == 5, 0, nodemap), np.where(nodemap == 5, f.n + 1, nodemap),
                    np.where(nodemap == 5, -1, nodemap)):
            with pytest.raises(_lib.B200Error) as e:
                f.plan_advanced(bad, src, gm, "keepall")
            assert e.value.code == _lib.ERR_ARG
        assert f.get_csr().data.tobytes() == A0.data.tobytes()
        _plans_equal(f.plan_advanced(nodemap, src, gm, "remove"),   # any other name is keepall
                     f.plan_advanced(nodemap, src, gm, "keepall"))
        args = [np.empty(8, dtype=np.int64) for _ in range(5)] + [np.empty(8), np.empty(f.n, dtype=np.int32)]
        assert f._lib.cs_b200_read_advanced_plan(f._h, *(_lib._ptr(a) for a in args)) == _lib.ERR_ARG


@pytest.mark.gpu
@pytest.mark.parametrize("name", MG)
def test_advanced_goldens_switch_on_equals_off_on_the_device(golden, name):
    args = _mg(golden, name)
    _same(_advanced(*args, cb.CUDASolver(**ON)), _advanced(*args, cb.CUDASolver()))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["full", "holes", "walls", "poly"])
@pytest.mark.parametrize("policy", POLICIES)
def test_advanced_random_switch_on_equals_off_on_the_device(kind, policy):
    g, poly, src, gm = _raster(kind)
    if kind == "poly":
        src[3, 4] = src[70, 10] = 0.0                       # the polygon node keeps a unit source
    _same(_advanced(g, poly, src, gm, policy, False, False, cb.CUDASolver(**ON)),
          _advanced(g, poly, src, gm, policy, False, False, cb.CUDASolver()))


@pytest.mark.gpu
def test_advanced_decimal_cancellation_switch_on_equals_off_on_the_device():
    g, src, gm = decimal_case(21, 300)
    _same(_advanced(g, None, src, gm, "keepall", False, False, cb.CUDASolver(**ON)),
          _advanced(g, None, src, gm, "keepall", False, False, cb.CUDASolver()))


@pytest.mark.gpu
def test_plan_sums_of_one_large_component_follow_numpys_tree():
    """one 1000 x 1000 component: three decimal sources that cancel placed many ways, each plan checked against
    numpy's pairwise sum of the component (the recursion splits down to 128-term blocks)"""
    g = np.ones((1000, 1000))
    f, nodemap = S.construct_raster_factor(g, None, cb.CUDASolver())
    rng = np.random.default_rng(9)
    seen = set()
    with f:
        lab = f.components()[1]
        for _ in range(24):
            src, gm = np.zeros(g.shape), np.zeros(g.shape)
            cells = rng.choice(g.size, size=3 + 200 * (_ % 2), replace=False)
            vals = np.round(rng.uniform(-0.9, 0.9, len(cells)), 1)
            vals[-1] = -np.round(vals[:-1].sum(), 1)
            src.ravel()[cells] = vals
            gm[rng.integers(0, 1000), rng.integers(0, 1000)] = np.inf
            got = f.plan_advanced(nodemap, src, gm, "keepall")
            want = plan_restated(nodemap, src, gm, "keepall", lab)[0]
            _plans_equal(got, want)
            seen.add(got["nsolved"])
    assert seen == {0, 1}                                   # both outcomes occur


@pytest.mark.gpu
@pytest.mark.parametrize("name", ONE_TO_ALL)
def test_onetoall_goldens_switch_on_equals_off_on_the_device(golden, name):
    data, flags, cfg, exp = cases.onetoall_problem(golden, name)
    four = co.cfg_bool(cfg, "connect_four_neighbors_only")
    _same(_onetoall(data, cfg, four, cb.CUDASolver(onetoall_raster=True, **ON)),
          _onetoall(data, cfg, four, cb.CUDASolver(onetoall_raster=True)))


@pytest.mark.gpu
@pytest.mark.parametrize("scenario", ["one-to-all", "all-to-one"])
@pytest.mark.parametrize("seed", [1, 2])
def test_onetoall_random_switch_on_equals_off_on_the_device(scenario, seed):
    rng = np.random.default_rng(seed)
    g = rng.uniform(0.5, 4.0, (50, 60))
    g[rng.random(g.shape) < 0.1] = -9999.0
    g[25, :] = -9999.0
    pm = np.zeros(g.shape)
    cells = rng.choice(g.size, size=8, replace=False)
    pm.ravel()[cells] = np.arange(1, 9)
    cfg, inputs, data = _problem(g, pm, None, None, scenario, "volt+cur+max", False)
    _same(_onetoall(data, cfg, False, cb.CUDASolver(onetoall_raster=True, **ON)),
          _onetoall(data, cfg, False, cb.CUDASolver(onetoall_raster=True)))


@pytest.mark.gpu
@pytest.mark.parametrize("name", REGION_GOLDENS)
def test_region_goldens_switch_on_equals_off_on_the_device(golden, name):
    cfg, inp, exp = co.load_case(golden, name)
    _same(_regions(cfg, inp, cb.CUDASolver(**ON)), _regions(cfg, inp, cb.CUDASolver()))


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2])
def test_region_random_switch_on_equals_off_on_the_device(seed):
    rng = np.random.default_rng(seed)
    g = rng.uniform(0.5, 4.0, (40, 50))
    g[rng.random(g.shape) < 0.1] = -9999.0
    pm = np.zeros(g.shape)
    for p in range(1, 5):
        r, c = rng.integers(0, 37), rng.integers(0, 47)
        pm[r:r + 2, c:c + 2] = p
    cfg, inputs = _cfg_inputs(g, pm, None, None, "max", False, False)
    _same(_regions(cfg, inputs, cb.CUDASolver(**ON)), _regions(cfg, inputs, cb.CUDASolver()))

"""Digest of every host driver in circuitscape_b200.core, for comparing two versions of the drivers call by call.

For each driver call it records a SHA-256 of every array of the returned object (resistances, per-pair maps in
their key order, cumulative / max maps, cum_node, cum_branch, branch, every AdvancedOutput / OneToAllOutput
field), num_solves and iterations, stats() without the timing fields, the sequence of `sink` calls with a digest
of each grid, and how the call ended (returned, or the exception and its message).  Inputs are the reference
goldens of tests/golden/reference_cases.npz and seeded rasters and networks, so two versions of the drivers that
compute the same thing write the same lines.

Covered: `solve` on rasters (shortcut, every map flag, log transform, both null flags, include / exclude lists,
superposition, with and without a sink) and on networks (host and device branch currents, superposition);
`raster_pairwise` through the existing driver, `pairwise_raster=True` and the focal-region driver (batched,
per-pair and unconnected pairs); `onetoall_kernel` both directions through the loop, `batch_*`,
`onetoall_raster` (with per-iteration fallbacks) and `resident_grounds`; `raster_advanced`, `network_advanced`
and `advanced_kernel` on rasters and networks; `compute_omniscape_current`.  Seeded rasters have several
components, polygons (one whose component numbers its cells unlike the node map), NODATA, include / exclude
lists and source strengths.

    python profiles/driver_digest.py --out digest.jsonl             # on the device
    python profiles/driver_digest.py --doubles --out digest.jsonl   # on the tests' CPU doubles, no device
    python profiles/driver_digest.py --compare a.jsonl b.jsonl      # differences between two runs; exit 1 if any
"""
import argparse
import dataclasses
import hashlib
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

TIMING = ("setup_ms", "solve_ms", "kernel_ms", "setup_s", "solve_s")
NODATA = -9999.0
MAPS = {"shortcut": {}, "volt": {"write_volt_maps": "True"}, "cur": {"write_cur_maps": "True"},
        "cum_only": {"write_cur_maps": "True", "write_cum_cur_map_only": "True"},
        "max_only": {"write_max_cur_maps": "True"},
        "log": {"write_cur_maps": "True", "write_max_cur_maps": "True", "log_transform_maps": "True"},
        "null": {"write_cur_maps": "True", "write_volt_maps": "True", "write_max_cur_maps": "True",
                 "set_null_currents_to_nodata": "True", "set_null_voltages_to_nodata": "True"},
        "all_log_null": {"write_cur_maps": "True", "write_volt_maps": "True", "write_max_cur_maps": "True",
                         "log_transform_maps": "True", "set_null_currents_to_nodata": "True",
                         "set_null_voltages_to_nodata": "True"}}


def digest(a):
    a = np.ascontiguousarray(a)
    return f"{a.dtype}{list(a.shape)}:" + hashlib.sha256(a.tobytes()).hexdigest()


def summary(x):
    """JSON-able digest of a driver result: arrays hashed, dicts as (key, value) lists in their order,
    timing fields dropped"""
    if x is None or isinstance(x, (bool, int, float, str)):
        return x
    if isinstance(x, np.generic):
        return x.item()
    if isinstance(x, np.ndarray):
        return digest(x)
    if dataclasses.is_dataclass(x):
        return {f.name: summary(getattr(x, f.name)) for f in dataclasses.fields(x)}
    if isinstance(x, dict):
        return [[summary(k), summary(v)] for k, v in x.items() if k not in TIMING]
    if isinstance(x, (list, tuple)):
        return [summary(v) for v in x]
    return repr(x)


class Sink:
    """records every call a driver makes on its sink"""

    def __init__(self):
        self.calls = []

    def voltmap(self, key, grid):
        self.calls.append(["voltmap", summary(key), digest(grid)])

    def curmap(self, key, grid):
        self.calls.append(["curmap", summary(key), digest(grid)])

    def network(self, key, comp, volt, cur, branch):
        self.calls.append(["network", summary(key), summary(comp), summary(volt), summary(cur), summary(branch)])


# ---------------------------------------------------------------------------
# the tests' CPU doubles (--doubles)
# ---------------------------------------------------------------------------
_REAL = {}


def use(kind, doubles):
    """point the solver module's factories at the CPU doubles the tests of `kind`'s driver use"""
    from circuitscape_b200 import solver as S
    if not doubles:
        return
    from tests.fake_factor import FakeFactor
    from tests import test_advanced_raster, test_network_device, test_onetoall_device, test_raster_pairwise_device
    for name in ("construct_cholesky_factor", "multiple_solve", "construct_raster_factor"):
        _REAL.setdefault(name, getattr(S, name))
    factor = test_network_device.NetworkDouble if kind == "network" else FakeFactor
    S.construct_cholesky_factor = lambda m, s, **kw: factor(m, s, **kw)
    S.multiple_solve = lambda s, m, b: FakeFactor(m, s).solve_rhs(np.asarray(b))[0]
    S.construct_raster_factor = {"pairs": test_raster_pairwise_device._double_factory,
                                 "onetoall": test_onetoall_device._double_factory,
                                 "advanced": test_advanced_raster._double_factory}.get(kind, _REAL[
                                     "construct_raster_factor"])


# ---------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------
def raster(seed, nr=11, nc=13, holes=0.1, walls=1, poly=True):
    """a seeded conductance raster (0 = no node) with NODATA walls and, optionally, a polygon map"""
    rng = np.random.default_rng(seed)
    g = rng.uniform(0.2, 4.0, (nr, nc))
    g[rng.random((nr, nc)) < holes] = 0.0
    for w in range(walls):
        if w % 2 == 0:
            g[:, rng.integers(2, nc - 2)] = 0.0
        else:
            g[rng.integers(2, nr - 2), :] = 0.0
    pm = None
    if poly:
        pm = np.zeros((nr, nc))
        pm[rng.random((nr, nc)) < 0.06] = 1
        pm[rng.random((nr, nc)) < 0.05] = 2
        r, c = rng.integers(0, nr), rng.integers(0, nc)       # a polygon cell on NODATA
        pm[r, c] = 3
        g[r, c] = 0.0
        pm.ravel()[rng.choice(nr * nc, size=2, replace=False)] = 3
    return g, pm


def own_map_raster():
    """a polygon with a NODATA cell in a raster of several components: that component's local node map numbers
    its cells unlike the node map"""
    N = 0.0
    g = np.array([[1.0, 2.0, N, 1.5, 2.5, 1.0],
                  [N, N, N, N, N, N],
                  [N, 3.0, 1.0, N, 2.0, 1.0],
                  [2.0, 1.0, 0.5, N, 1.0, 3.0]])
    poly = np.zeros(g.shape)
    poly[2, 0] = poly[3, 2] = 4
    prc = (np.array([1, 1, 3, 4, 4, 1, 3]), np.array([1, 4, 2, 1, 5, 6, 6]), np.array([1, 2, 3, 4, 5, 6, 7]))
    return g, poly, prc


def points(seed, g, npts, repeat=False):
    """(rows, cols, ids) 1-based, sorted by id, all but the last on a node of `g`; with repeat, ids on several cells
    (focal regions)"""
    rng = np.random.default_rng(seed)
    nr, nc = g.shape
    cells = rng.choice(np.flatnonzero(g.ravel(order="F") > 0), size=npts, replace=False)
    cells[-1] = rng.integers(0, nr * nc)                     # possibly off the graph
    if repeat:
        ids = np.sort(rng.integers(1, max(2, npts // 2) + 1, size=npts))
    else:
        ids = np.sort(rng.choice(np.arange(1, 40), size=npts, replace=False))
    return cells % nr + 1, cells // nr + 1, ids


def inc_list(seed, ids, mode):
    rng = np.random.default_rng(seed)
    pid = np.array(sorted(set(int(i) for i in ids)))
    mat = (rng.random((len(pid), len(pid))) < 0.5).astype(float)
    return types.SimpleNamespace(mode=mode, point_ids=pid, mat=np.maximum(mat, mat.T))


def network(seed, n=40, comps=3):
    """(i, j, v) 1-based edges of a seeded graph with several components, and focal nodes"""
    rng = np.random.default_rng(seed)
    i, j = [], []
    bounds = np.linspace(0, n, comps + 1).astype(int)
    for a, b in zip(bounds[:-1], bounds[1:]):
        for k in range(a + 1, b):                             # a spanning chain, then random chords
            i.append(k), j.append(rng.integers(a, k))
        for _ in range(b - a):
            x, y = rng.integers(a, b, size=2)
            if x != y:
                i.append(x), j.append(y)
    i, j = np.array(i) + 1.0, np.array(j) + 1.0
    keys = {}
    for a, b in zip(i, j):
        keys.setdefault((min(a, b), max(a, b)), None)
    i, j = np.array([k[0] for k in keys]), np.array([k[1] for k in keys])
    return i, j, rng.uniform(0.5, 3.0, len(i)), np.sort(rng.choice(np.arange(1, n + 1), size=7, replace=False))


def network_problem(i, j, v, fp, solver):
    import scipy.sparse as sp
    import circuitscape_b200 as cb
    from circuitscape_b200 import graph
    m = int(max(i.max(), j.max()))
    A = sp.coo_matrix((v, (i - 1, j - 1)), shape=(m, m)).tocsr()
    A = (A + A.T).tocsr()
    return cb.GraphProblem(graph.laplacian(A), graph.connected_components(A), fp, fp, set(), None, None, None,
                           solver, (i, j))


# ---------------------------------------------------------------------------
# the calls
# ---------------------------------------------------------------------------
def run(out_path, doubles):
    import circuitscape_b200 as cb
    from circuitscape_b200 import core, graph
    from oracle import circuitscape_oracle as co
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import cases
    golden = np.load(os.path.join(ROOT, "tests", "golden", "reference_cases.npz"))
    CS = cb.CUDASolver
    fh = open(out_path, "w")

    def call(case, fn, sink=None):
        rec = dict(case=case)
        try:
            rec["out"] = summary(fn())
            rec["ended"] = "returned"
        except Exception as e:                                # noqa: BLE001 -- the failure is the result
            rec["ended"] = f"{type(e).__name__}: {e}"
        if sink is not None:
            rec["sink"] = sink.calls
        fh.write(json.dumps(rec, sort_keys=True) + "\n")
        fh.flush()

    def golden_raster(name):
        cfg, inp, exp = co.load_case(golden, name)
        cellmap, polymap, meta, inc = co.load_raster_inputs(cfg, inp)
        pk = inp["point_file"]
        fl = co.cfg_flags(cfg)
        return cfg, cb.RasterData(cellmap, polymap, co.read_point_map(pk[0], pk[1], meta), None, inc), fl

    def pairwise(case, data, cfg, solver, four=False, avg=False, with_sink=False):
        sink = Sink() if with_sink else None
        call(case, lambda: cb.raster_pairwise(data, cb.Flags.from_cfg(cfg), cfg, solver=solver, four_neighbors=four,
                                              avg_res=avg, sink=sink), sink)

    # -- raster pairwise: goldens -------------------------------------------------------------------------
    use("pairs", doubles)
    for k in range(1, 18):
        name = f"sgVerify{k}"
        cfg, data, fl = golden_raster(name)
        for tag, solver in (("default", CS()), ("superpose", CS(superpose=True)),
                            ("pairwise_raster", CS(pairwise_raster=True)),
                            ("pairwise_raster_superpose", CS(pairwise_raster=True, superpose=True))):
            pairwise(f"golden/{name}/raster_pairwise/{tag}", data, cfg, solver, fl["four_neighbors"], fl["avg_res"])
        pairwise(f"golden/{name}/raster_pairwise/sink", data, cfg, CS(), fl["four_neighbors"], fl["avg_res"], True)
        sink = Sink()
        call(f"golden/{name}/single_ground_all_pairs/sink", lambda: cases.run_raster_pairwise(golden, name, CS(), sink)[0],
             sink)

    # -- raster pairwise: seeded rasters, every map flag set, through each driver -------------------------
    g_own, poly_own, prc_own = own_map_raster()
    with_points = lambda name, g, pm, seed, npts, repeat=False: (name, g, pm, points(seed, g, npts, repeat))
    rasters = [with_points("walls", *raster(1, poly=False), 11, 6), with_points("poly", *raster(2), 12, 7),
               with_points("holes", *raster(3, holes=0.25, walls=2), 13, 6), ("own_map", g_own, poly_own, prc_own)]
    for rname, g, pm, prc in rasters:
        for maps in MAPS:
            cfg = dict(MAPS[maps])
            for inc_mode in (None, "include", "exclude"):
                inc = None if inc_mode is None else inc_list(len(rname) + len(maps), prc[2], inc_mode)
                data = cb.RasterData(g, pm, prc, None, inc)
                for tag, solver in (("default", CS()), ("superpose", CS(superpose=True)),
                                    ("pairwise_raster", CS(pairwise_raster=True)),
                                    ("pairwise_raster_superpose", CS(pairwise_raster=True, superpose=True)),
                                    ("single", CS(precision="single")),
                                    ("pairwise_raster_single", CS(pairwise_raster=True, precision="single"))):
                    pairwise(f"seeded/{rname}/{maps}/{inc_mode}/{tag}", data, cfg, solver)
                for tag, solver in (("default", CS()), ("pairwise_raster", CS(pairwise_raster=True))):
                    pairwise(f"seeded/{rname}/{maps}/{inc_mode}/{tag}/sink", data, cfg, solver, with_sink=True)
        for four, avg in ((True, False), (False, True)):
            data = cb.RasterData(g, pm, prc, None, None)
            for tag, solver in (("default", CS()), ("pairwise_raster", CS(pairwise_raster=True))):
                pairwise(f"seeded/{rname}/cur/four{four}_avg{avg}/{tag}", data, MAPS["cur"], solver, four, avg)

    # -- focal regions: batched, per-pair (overlapping regions, polygon merges) and unconnected pairs ------
    regions = [with_points(f"regions_{tag}", *raster(seed, poly=poly, walls=2, holes=0.15), seed + 10, 10, True)
               for tag, seed, poly in (("unconnected", 5, False), ("off_graph", 12, False),
                                       ("poly_merges", 5, True), ("overlap", 9, True))]
    for rname, g, pm, prc in regions:
        for maps in MAPS:
            cfg = dict(MAPS[maps])
            for inc_mode in (None, "exclude"):
                inc = None if inc_mode is None else inc_list(7, prc[2], inc_mode)
                data = cb.RasterData(g, pm, prc, None, inc)
                pairwise(f"{rname}/{maps}/{inc_mode}", data, cfg, CS())
                pairwise(f"{rname}/{maps}/{inc_mode}/sink", data, cfg, CS(), with_sink=True)

    # -- network pairwise -----------------------------------------------------------------------------------
    use("network", doubles)
    nets = [(f"golden/sgNetworkVerify{k}", None) for k in range(1, 4)] + [("seeded/net1", network(21)),
                                                                          ("seeded/net2", network(22, 60, 4))]
    for nname, raw in nets:
        for maps in ("cur", "volt", "null"):
            for tag, kw in (("host", {}), ("device_branch", dict(branch_on_device=True)),
                            ("superpose", dict(superpose=True)),
                            ("device_branch_superpose", dict(branch_on_device=True, superpose=True))):
                for with_sink in (False, True):
                    if raw is None:
                        prob, flags, _ = cases.network_pairwise_problem(golden, nname.split("/")[1], CS(**kw))
                    else:
                        prob = network_problem(*raw, CS(**kw))
                        cfg = dict(MAPS[maps], data_type="network")
                        flags = cb.Flags.from_cfg(cfg)
                    sink = Sink() if with_sink else None
                    call(f"{nname}/{maps}/{tag}/{'sink' if with_sink else 'kept'}",
                         lambda: cb.single_ground_all_pairs(prob, flags, sink=sink), sink)
            if raw is None:
                break                                         # the golden's own flags

    # -- advanced mode ------------------------------------------------------------------------------------
    for k in range(1, 4):
        name = f"mgNetworkVerify{k}"
        prob, flags, _ = cases.advanced_problem(golden, name, CS())
        call(f"golden/{name}/network_advanced", lambda: cb.network_advanced(prob, flags))
        call(f"golden/{name}/advanced_kernel", lambda: cb.advanced_kernel(prob, flags))
    for seed in (31, 32):
        i, j, v, _ = network(seed, 50, 4)
        prob = network_problem(i, j, v, np.array([1]), CS())
        rng = np.random.default_rng(seed)
        n = prob.G.shape[0]
        for kind in ("finite", "inf", "mixed"):
            s = np.where(rng.random(n) < 0.3, rng.uniform(0.5, 2.0, n), 0.0)
            gr = np.where(rng.random(n) < 0.3, rng.uniform(0.5, 2.0, n), 0.0)
            if kind != "finite":
                gr = np.where((gr != 0) & (rng.random(n) < (1.0 if kind == "inf" else 0.5)), np.inf, gr)
            for policy in ("keepall", "rmvsrc"):
                ap = cb.AdvancedProblem(prob.G, prob.cc, *cb.resolve_conflicts(s, gr, policy), solver=CS())
                fl = cb.Flags(is_raster=False, is_advanced=True)
                call(f"seeded/net{seed}/{kind}/{policy}/network_advanced", lambda: cb.network_advanced(ap, fl))
                call(f"seeded/net{seed}/{kind}/{policy}/advanced_kernel", lambda: cb.advanced_kernel(ap, fl))

    use("advanced", doubles)
    for k in range(1, 7):
        name = f"mgVerify{k}"
        cfg, inp, _ = co.load_case(golden, name)
        flags = cb.Flags.from_cfg(cfg)
        fl = co.cfg_flags(cfg)
        cellmap, polymap, meta, _ = co.load_raster_inputs(cfg, inp)
        sm, gm = co.read_source_and_ground_maps(cfg, inp, meta)
        data = cb.RasterData(cellmap, polymap, None, source_map=sm, ground_map=gm)
        call(f"golden/{name}/raster_advanced", lambda: cb.raster_advanced(data, flags, cfg, solver=CS(),
                                                                          four_neighbors=fl["four_neighbors"],
                                                                          avg_res=fl["avg_res"]))
        prob, flags, _ = cases.advanced_problem(golden, name, CS())
        call(f"golden/{name}/advanced_kernel", lambda: cb.advanced_kernel(prob, flags))
    fl = cb.Flags(is_raster=True, is_advanced=True)
    for rname, g, pm, _ in rasters:
        rng = np.random.default_rng(len(rname))
        for kind in ("finite", "inf", "mixed", "none"):
            sm = np.where(rng.random(g.shape) < 0.15, rng.uniform(0.5, 2.0, g.shape), 0.0)
            gm = np.where(rng.random(g.shape) < 0.15, rng.uniform(0.5, 2.0, g.shape), 0.0)
            if kind in ("inf", "mixed"):
                gm = np.where((gm != 0) & (rng.random(g.shape) < (1.0 if kind == "inf" else 0.5)), np.inf, gm)
            if kind == "none":
                gm = np.zeros(g.shape)
            for policy in ("keepall", "rmvsrc", "rmvgnd", "rmvall"):
                cfg = {"remove_src_or_gnd": policy}
                data = cb.RasterData(g, pm, None, source_map=sm, ground_map=gm)
                call(f"seeded/{rname}/{kind}/{policy}/raster_advanced",
                     lambda: cb.raster_advanced(data, fl, cfg, solver=CS()))
                nm = graph.construct_node_map(g, pm)
                G = graph.laplacian(graph.construct_graph(g, nm, False, False))
                s, gr, f = core.sources_and_grounds_from_maps(sm, gm, nm, G.shape[0], policy)
                ap = cb.AdvancedProblem(G, graph.connected_components(G), s, gr, f, nm, pm, g, CS())
                call(f"seeded/{rname}/{kind}/{policy}/advanced_kernel", lambda: cb.advanced_kernel(ap, fl))

    # -- one-to-all / all-to-one ----------------------------------------------------------------------------
    use("onetoall", doubles)
    variants = (("loop", {}), ("batch", dict(batch_one_to_all=True, batch_all_to_one=True)),
                ("onetoall_raster", dict(onetoall_raster=True)), ("resident", dict(resident_grounds=True)))
    for name in [f"oneToAllVerify{i}" for i in range(1, 14)] + [f"allToOneVerify{i}" for i in range(1, 13)]:
        data, flags, cfg, _ = cases.onetoall_problem(golden, name)
        four = co.cfg_bool(cfg, "connect_four_neighbors_only")
        avg = cfg.get("connect_using_avg_resistances", "False") in ("True", "true")
        for tag, kw in variants:
            call(f"golden/{name}/onetoall_kernel/{tag}",
                 lambda: cb.onetoall_kernel(data, flags, cfg, solver=CS(**kw), four_neighbors=four, avg_res=avg))
    for rname, g, pm, prc in rasters + regions:
        rng = np.random.default_rng(len(rname) + 100)
        strengths = np.column_stack([prc[2], rng.uniform(0.5, 3.0, len(prc[2]))])   # one row per point
        for maps in ("cur", "volt", "max_only", "null"):
            cfg = dict(MAPS[maps])
            flags = cb.Flags.from_cfg(cfg)
            for one_to_all in (True, False):
                for st_tag, st_ in (("unit", None), ("strengths", strengths)):
                    for inc_mode in (None, "include"):
                        inc = None if inc_mode is None else inc_list(3, prc[2], inc_mode)
                        data = cb.RasterData(g, pm, prc, st_, inc)
                        for tag, kw in variants:
                            call(f"seeded/{rname}/{maps}/{one_to_all}/{st_tag}/{inc_mode}/{tag}",
                                 lambda: cb.onetoall_kernel(data, flags, cfg, solver=CS(**kw), one_to_all=one_to_all))

    # -- Omniscape's moving-window solve ----------------------------------------------------------------------
    use("host", doubles)
    for seed in (41, 42):
        g, _ = raster(seed, 9, 10, holes=0.15, walls=1, poly=False)
        rng = np.random.default_rng(seed)
        src = np.where(rng.random(g.shape) < 0.2, rng.uniform(0.5, 2.0, g.shape), 0.0)
        gnd = np.where(rng.random(g.shape) < 0.2, rng.uniform(0.5, 2.0, g.shape), 0.0)
        for four in ("False", "True"):
            cs_cfg = {"connect_four_neighbors_only": four}
            call(f"seeded/omniscape{seed}/four{four}",
                 lambda: core.compute_omniscape_current(np.where(g == 0, NODATA, g), src, gnd, cs_cfg, solver=CS()))
    fh.close()


def compare(a_path, b_path):
    """prints every difference between two runs and returns how many there are"""
    a = {r["case"]: r for r in map(json.loads, open(a_path))}
    b = {r["case"]: r for r in map(json.loads, open(b_path))}
    print(f"{len(a)} / {len(b)} calls; same cases: {sorted(a) == sorted(b)}")
    diffs = 0
    for case in sorted(set(a) ^ set(b)):
        print("missing from", b_path if case in a else a_path, case)
        diffs += 1
    ended = {}
    for case in sorted(set(a) & set(b)):
        ra, rb = a[case], b[case]
        kind = ra["ended"].split(":")[0]
        ended[kind] = ended.get(kind, 0) + 1
        for key in ("ended", "out", "sink"):
            if ra.get(key) != rb.get(key):
                print("DIFF", case, key)
                diffs += 1
    print("outcomes:", ended)
    print("differences:", diffs)
    return diffs


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--doubles", action="store_true", help="the tests' CPU doubles instead of the device")
    ap.add_argument("--compare", nargs=2)
    args = ap.parse_args()
    if args.compare:
        sys.exit(1 if compare(*args.compare) else 0)
    run(args.out, args.doubles)

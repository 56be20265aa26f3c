"""Digest of every batched solve entry of B200Factor, for comparing two builds call by call.

For each call it records a SHA-256 of every returned array (and of the cumulative / max current maps
after an accumulating call), how the call ended (returned, or the exception and its message), the
handle's last_error text and stats() without the timing fields.  Inputs are seeded, so two builds that
compute the same thing write the same digests.

Covered: solve_rhs, solve_pairs, solve_pairs_superposed, solve_region_pairs, solve_grounded and
solve_sources with k = 15 columns (panels of 8, 4, 2 and 1), on a stencil-form raster, a windowed
operator (raster with NODATA holes) and a plain-CSR operator; fp64 and mixed AMG, fp32 AMG
(f32_compute) and fp64 Jacobi; the device-graph, chunked and plain loop drivers; with no optional
output and with volt, curr, accumulate, weights (and probe rows).  One configuration also runs every
entry at rtol 0.5 / itmax 1 (residual gate) and rtol 1e-14 / itmax 12 (itmax stop), and one region
pair has no conducting path.

With --profile every call runs once more with the per-launch profile on, and its record also holds the
profile's accounting: per kernel class the algorithmic bytes and launches, and profile_bytes() (no times).

    python profiles/entry_digest.py --out digest.jsonl          # one JSON line per call
    python profiles/entry_digest.py --profile --out digest.jsonl
    python profiles/entry_digest.py --compare a.jsonl b.jsonl   # differences between two runs; exit 1 if any
"""
import argparse
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

K = 15
TIMING = ("setup_ms", "solve_ms", "kernel_ms")


def digest(a):
    a = np.ascontiguousarray(a)
    return f"{a.dtype}{list(a.shape)}:" + hashlib.sha256(a.tobytes()).hexdigest()


def operators():
    from circuitscape_b200 import graph
    holes = 1.0 / np.random.default_rng(3).uniform(1.0, 10.0, size=(190, 130))
    holes[np.random.default_rng(4).random(holes.shape) < 0.04] = 0.0
    nm = graph.construct_node_map(holes, None)
    G = graph.laplacian(graph.construct_graph(holes, nm, False, False))
    big = max(graph.connected_components(G), key=len) - 1
    windowed = G[big][:, big].tocsr()
    return [("stencil", graph.synthetic_raster_laplacian(160, 150, seed=5)[0], {}),
            ("windowed", windowed, {}),
            ("csr", windowed[:9000][:, :9000].tocsr(), {"window": "off", "stencil": "off"})]


def configs():
    return [("f64", dict(mixed=False)), ("mixed", dict(mixed=True)),
            ("f32", dict(precision="single", f32_compute=True)), ("jacobi", dict(precond="jacobi"))]


def inputs(n, seed):
    rng = np.random.default_rng(seed)
    pick = rng.choice(n, size=120, replace=False)
    nodes = pick[:6]                                           # 6 focal nodes -> 15 pairs
    pi, pj = np.triu_indices(6, 1)
    src, dst = pick[6:21], pick[21:36]
    sets = [np.sort(pick[36 + 8 * s:44 + 8 * s]) for s in range(6)]   # disjoint, 8 rows each
    set_a, set_b = pi.copy(), pj.copy()
    gsets = sets[:4]
    gset = rng.integers(0, 4, size=K)
    free = pick[84:120]
    sources = []
    for c in range(K):
        rows = np.sort(rng.choice(free, size=1 + c % 3, replace=False))
        sources.append((rows, rng.uniform(0.5, 2.0, size=len(rows))))
    columns = []
    for c in range(K):
        rows = np.sort(rng.choice(free, size=2 + c % 3, replace=False))
        v = rng.uniform(0.5, 2.0, size=len(rows))
        v[-1] = -v[:-1].sum()
        columns.append((rows, v))
    rhs = rng.standard_normal((n, K))
    rhs -= rhs.mean(axis=0)
    return dict(nodes=nodes, pi=pi, pj=pj, src=src, dst=dst, sets=sets, set_a=set_a, set_b=set_b, gsets=gsets,
                gset=gset, sources=sources, columns=columns, ref=free[rng.integers(0, 8, size=K)],
                probe=pick[100:105], rhs=rhs, weight=rng.uniform(0.5, 3.0, size=K))


def calls(x, full, **lim):
    """(name, method name, kwargs, accumulates) of every entry, with or without the optional outputs"""
    opt = dict(want_volt=True, want_curr=True, accumulate=True, weight=x["weight"]) if full else {}
    return [("rhs", "solve_rhs", dict(rhs=x["rhs"], **lim), False),
            ("pairs", "solve_pairs", dict(src=x["src"], dst=x["dst"], **opt, **lim), full),
            ("superposed", "solve_pairs_superposed", dict(nodes=x["nodes"], pi=x["pi"], pj=x["pj"], **opt, **lim),
             full),
            ("region", "solve_region_pairs", dict(sets=x["sets"], set_a=x["set_a"], set_b=x["set_b"], **opt, **lim),
             full),
            ("grounded", "solve_grounded", dict(sets=x["gsets"], gset=x["gset"], sources=x["sources"], **opt, **lim),
             full),
            ("sources", "solve_sources", dict(columns=x["columns"], ref=x["ref"],
                                              probe=x["probe"] if full else None, **opt, **lim), full)]


def run_call(f, method, kw, accumulates, profile=False):
    rec = {}
    try:
        out = getattr(f, method)(**kw)
        rec["ended"] = "returned"
        items = out.items() if isinstance(out, dict) else zip(("x", "iters", "relres"), out)
        rec["arrays"] = {k: None if v is None else digest(v) for k, v in sorted(items)}
    except Exception as e:                                   # noqa: BLE001 -- the failure is the result
        rec["ended"] = f"{type(e).__name__}: {e}"
    msg = f._lib.cs_b200_last_error(f._h)
    rec["last_error"] = msg.decode() if msg else ""
    rec["stats"] = {k: v for k, v in f.stats().items() if k not in TIMING}
    if accumulates:
        cum, mx = f.read_currents()
        rec["maps"] = [digest(cum), digest(mx)]
        f.reset_currents()
    if profile:
        f.profile_spmm(True)
        try:
            getattr(f, method)(**kw)
        except Exception:                                    # noqa: BLE001 -- recorded above
            pass
        rec["profile"] = dict(classes={c: [b, n] for c, (_, b, n) in sorted(f.profile_classes().items())},
                              bytes=f.profile_bytes())
        f.profile_spmm(False)
        if accumulates:
            f.reset_currents()
    return rec


def run(out_path, profile=False):
    import circuitscape_b200 as cb
    from circuitscape_b200 import solver as S
    with open(out_path, "w") as fh:
        def emit(case, rec):
            fh.write(json.dumps(dict(case=case, **rec), sort_keys=True) + "\n")

        for oname, L, oopts in operators():
            x = inputs(L.shape[0], seed=11)
            for cname, copts in configs():
                for loop in (True, "chunk", False):
                    with cb.B200Factor(L, cb.CUDASolver(use_graph=loop, **oopts, **copts)) as f:
                        form = f.operator_form()
                        for full in (False, True):
                            for name, method, kw, acc in calls(x, full):
                                case = f"{oname}({form})/{cname}/{loop}/{'full' if full else 'bare'}/{name}"
                                emit(case, run_call(f, method, kw, acc, profile))
                        if oname == "stencil" and cname == "f64" and loop is True:
                            for tag, lim in (("gate", dict(rtol=0.5, itmax=1)), ("itmax", dict(rtol=1e-14, itmax=12))):
                                for name, method, kw, acc in calls(x, True, **lim):
                                    kw.setdefault("raise_on_residual", False)
                                    emit(f"{oname}/{cname}/{tag}/{name}", run_call(f, method, kw, acc, profile))
        # a region pair with no conducting path: set 2 is a 2 x 2 island of unit conductance (4 neighbours),
        # so L 1 is exactly zero on it and the flux into it is exactly zero
        g = 1.0 / np.random.default_rng(8).uniform(1.0, 10.0, size=(60, 50))
        g[47:53, 37:43] = 0.0
        g[49:51, 39:41] = 1.0
        f, nodemap = S.construct_raster_factor(g, None, cb.CUDASolver(), four_neighbors=True)
        with f:
            sets = [np.sort(nodemap[r0:r0 + 5, c0:c0 + 5].ravel() - 1) for r0, c0 in ((0, 0), (30, 0))]
            sets.append(np.sort(nodemap[49:51, 39:41].ravel() - 1))
            kw = dict(sets=sets, set_a=np.array([0, 0, 1]), set_b=np.array([1, 2, 2]), want_volt=True)
            emit("split/region_no_path", run_call(f, "solve_region_pairs", kw, False, profile))


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
        ended[ra["ended"].split(":")[0]] = ended.get(ra["ended"].split(":")[0], 0) + 1
        for key in ("ended", "last_error", "arrays", "maps", "profile"):
            if ra.get(key) != rb.get(key):
                print("DIFF", case, key, ra.get(key), rb.get(key))
                diffs += 1
        for k, v in ra["stats"].items():
            if rb["stats"].get(k) != v:
                print("stats", case, k, v, rb["stats"].get(k))
                diffs += 1
    print("outcomes:", ended)
    errs = sorted({r["last_error"][:60] for r in a.values() if r["last_error"]})
    print("last_error texts:", errs)
    print("differences:", diffs)
    return diffs


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2)
    ap.add_argument("--profile", action="store_true", help="also record the per-class profile accounting")
    args = ap.parse_args()
    if args.compare:
        sys.exit(1 if compare(*args.compare) else 0)
    else:
        run(args.out, args.profile)

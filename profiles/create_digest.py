"""Digest of what every create entry of libcsb200 leaves behind, for comparing two builds create by create.

For each create it records a SHA-256 of the handle's operator (get_csr), of every levels() matrix with its
omega, windowed and stencil flags, the finest operator's form, stats() without the timing fields, the node map
of the raster entries, and one solve_pairs with accumulated currents (R, iterations, residuals, current maps);
for a failing create, the error code and the text of cs_b200_last_error(NULL).  Inputs are seeded, so two builds
that compute the same thing write the same digests.

Covered: cs_b200_create, cs_b200_create_from_device, cs_b200_create_from_raster, cs_b200_create_from_raster_poly
(without and with polygons) and cs_b200_create_bcast (one rank; recorded as skipped where NCCL cannot be
loaded), each under setup host / device, fp64 / fp32 (f32_compute) and AMG / Jacobi, on a full raster (stencil
form) and on a raster with NODATA lakes (windowed form).  Failing creates: an all-zero raster through both raster
entries, a rowptr that does not span [0, nnz], a bad panel width.

    python profiles/create_digest.py --out digest.jsonl          # one JSON line per create
    python profiles/create_digest.py --compare a.jsonl b.jsonl   # differences between two runs; exit 1 if any
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

TIMING = ("setup_ms", "solve_ms", "kernel_ms")


def digest(a):
    a = np.ascontiguousarray(a)
    return f"{a.dtype}{list(a.shape)}:" + hashlib.sha256(a.tobytes()).hexdigest()


def csr_digest(m):
    return None if m is None else [list(m.shape), digest(m.indptr), digest(m.indices), digest(m.data)]


def rasters():
    """(name, conductance, polygon map): a full raster and one with rectangular NODATA lakes; the polygon
    map joins a few blocks of cells into single nodes"""
    full = 1.0 / np.random.default_rng(5).uniform(1.0, 10.0, size=(190, 160))
    lakes = 1.0 / np.random.default_rng(6).uniform(1.0, 10.0, size=(200, 170))
    rng = np.random.default_rng(7)
    for _ in range(12):
        r, c = rng.integers(5, 180), rng.integers(5, 150)
        lakes[r:r + rng.integers(3, 12), c:c + rng.integers(3, 12)] = 0.0
    poly = np.zeros(full.shape, dtype=np.int32)
    for k, (r, c) in enumerate(((10, 10), (100, 40), (150, 120))):
        poly[r:r + 4, c:c + 5] = k + 1
    return [("full", full, poly), ("lakes", lakes, None)]


def configs():
    return [("f64-amg", dict(mixed=False)), ("mixed-amg", dict()),
            ("f32-amg", dict(precision="single", f32_compute=True)), ("f64-jacobi", dict(precond="jacobi")),
            ("f32-jacobi", dict(precision="single", f32_compute=True, precond="jacobi"))]


def entries(g, poly):
    import circuitscape_b200 as cb
    from circuitscape_b200 import dist, graph
    nodemap = graph.construct_node_map(g, None)
    A = graph.laplacian(graph.construct_graph(g, nodemap, False, False)).tocsr()

    def from_device(s):
        import torch
        dev = torch.device("cuda", s.device)
        vt = np.float64 if np.dtype(s.device_dtype) == np.float64 else np.float32
        rp = torch.from_numpy(A.indptr.astype(np.int32)).to(dev)
        ci = torch.from_numpy(A.indices.astype(np.int32)).to(dev)
        va = torch.from_numpy(np.ascontiguousarray(A.data, dtype=vt)).to(dev)
        return dist.factor_from_device(A.shape[0], A.nnz, rp, ci, va, s), None

    def bcast(s):
        return dist.Comm(s.device, 0, 1, lambda raw: raw).create_factor(A, s), None

    out = [("create", lambda s: (cb.B200Factor(A, s), None)),
           ("from_device", from_device),
           ("from_raster", lambda s: (cb.B200Factor.from_raster(g, s), None)),
           ("from_raster_poly", lambda s: cb.B200Factor.from_raster_polygons(g, None, s))]
    if poly is not None:
        out.append(("from_raster_poly+polygons", lambda s: cb.B200Factor.from_raster_polygons(g, poly, s)))
    out.append(("bcast", bcast))
    return out


def record(make, solver):
    from circuitscape_b200 import _lib, graph
    rec = {}
    try:
        f, nodemap = make(solver)
    except Exception as e:                                   # noqa: BLE001 -- the failure is the result
        rec["ended"] = f"{type(e).__name__} {getattr(e, 'code', '')}: {e}"
        rec["last_error"] = (_lib.load().cs_b200_last_error(None) or b"").decode()
        return rec
    with f:
        rec["ended"] = "created"
        rec["form"] = f.operator_form()
        rec["csr"] = csr_digest(f.get_csr())
        rec["levels"] = [{k: (csr_digest(v) if k in ("A", "P", "R") else v) for k, v in sorted(lv.items())}
                         for lv in f.levels()]
        rec["nodemap"] = None if nodemap is None else digest(nodemap)
        nodes = graph.focal_nodes(f.n, 4, seed=7)
        src, dst = graph.all_pairs(nodes)
        f.reset_currents()
        try:
            out = f.solve_pairs(src, dst, accumulate=True)
            rec["solve"] = {k: digest(v) for k, v in sorted(out.items()) if v is not None}
            rec["maps"] = [digest(m) for m in f.read_currents()]
        except Exception as e:                               # noqa: BLE001 -- the failure is the result
            rec["solve"] = f"{type(e).__name__}: {e}"
        rec["stats"] = {k: v for k, v in f.stats().items() if k not in TIMING}
    return rec


def failing(setup):
    """(name, create) of creates that must fail"""
    import circuitscape_b200 as cb
    from circuitscape_b200 import _lib, graph
    s = cb.CUDASolver(setup=setup)
    A = graph.synthetic_raster_laplacian(30, 20, seed=3)[0].tocsr()
    lib = _lib.load()

    def bad_rowptr(bits):
        def make(_):
            it = np.int64 if bits == 64 else np.int32
            rp = A.indptr.astype(it)
            rp[-1] += 1
            ci = A.indices.astype(it)
            va = np.ascontiguousarray(A.data, dtype=np.float64)
            h = C.c_void_p()
            opts = cb.B200Factor._opts(s)
            rc = lib.cs_b200_create(A.shape[0], A.nnz, _lib._ptr(rp), _lib._ptr(ci), _lib._ptr(va), bits, 0, _lib.F64,
                                    0, C.byref(opts), C.byref(h))
            if h.value:
                lib.cs_b200_destroy(h)
            _lib.check(lib, None, rc)
        return make

    return [("zero_raster/from_raster", lambda _: (cb.B200Factor.from_raster(np.zeros((40, 30)), s), None)),
            ("zero_raster/from_raster_poly", lambda _: cb.B200Factor.from_raster_polygons(np.zeros((40, 30)), None, s)),
            ("rowptr_span/32", bad_rowptr(32)), ("rowptr_span/64", bad_rowptr(64)),
            ("panel_width", lambda _: (cb.B200Factor(A, cb.CUDASolver(setup=setup, panel_width=3)), None))]


def run(out_path):
    import torch  # noqa: F401 -- before the library loads NCCL, so that torch binds its own
    import circuitscape_b200 as cb
    from circuitscape_b200 import _lib
    with open(out_path, "w") as fh:
        def emit(case, rec):
            fh.write(json.dumps(dict(case=case, **rec), sort_keys=True) + "\n")
            fh.flush()

        ident = (C.c_char * 128)()
        nccl = _lib.load().cs_b200_comm_unique_id(C.cast(ident, C.c_void_p)) != _lib.ERR_UNSUPPORTED
        for rname, g, poly in rasters():
            for ename, make in entries(g, poly):
                for setup in ("host", "device"):
                    for cname, copts in configs():
                        case = f"{rname}/{ename}/{setup}/{cname}"
                        if ename == "bcast" and not nccl:
                            emit(case, {"ended": "skipped: NCCL cannot be loaded"})
                            continue
                        emit(case, record(make, cb.CUDASolver(setup=setup, **copts)))
        for setup in ("host", "device"):
            for name, make in failing(setup):
                emit(f"fail/{name}/{setup}", record(make, None))


def compare(a_path, b_path):
    """prints every difference between two runs and returns how many there are"""
    a = {r["case"]: r for r in map(json.loads, open(a_path))}
    b = {r["case"]: r for r in map(json.loads, open(b_path))}
    print(f"{len(a)} / {len(b)} creates; same cases: {sorted(a) == sorted(b)}")
    diffs = 0
    for case in sorted(set(a) ^ set(b)):
        print("missing from", b_path if case in a else a_path, case)
        diffs += 1
    ended = {}
    for case in sorted(set(a) & set(b)):
        ra, rb = a[case], b[case]
        ended[ra["ended"].split(":")[0]] = ended.get(ra["ended"].split(":")[0], 0) + 1
        for key in sorted(set(ra) | set(rb)):
            if ra.get(key) != rb.get(key):
                print("DIFF", case, key, str(ra.get(key))[:200], str(rb.get(key))[:200])
                diffs += 1
    print("outcomes:", ended)
    print("forms:", sorted({(r["case"].split("/")[0], r.get("form")) for r in a.values() if "form" in r}))
    print("differences:", diffs)
    return diffs


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2)
    args = ap.parse_args()
    if args.compare:
        sys.exit(1 if compare(*args.compare) else 0)
    else:
        run(args.out)

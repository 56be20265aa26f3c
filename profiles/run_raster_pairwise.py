"""Raster pairwise mode with focal points on the 3163 x 3163 bench raster: CUDASolver(pairwise_raster=True) (one
whole-raster handle, components labelled on the device by cs_b200_components, every pair a column of the same
panels) against the existing driver (host node map, graph, Laplacian and SciPy components, one handle per
component) on the same inputs, end to end from raster_pairwise's arguments to its output, the two paths
alternated.  Prints a JSON line after every case; an optional first argument picks cases (comma-separated),
`--size N` shrinks the rasters for a dry run, `--reps K` sets the alternations (default 2).

Raster: R ~ U[1, 10] (seed 42), the bench.py generator; default CUDASolver settings.  Cases:
  full_cum:       16 focal points (120 pairs), cumulative current map (write_cum_cur_map_only).
  full_shortcut:  the same points, no maps: the shortcut (one anchor's columns, probe rows).
  walls8:         NODATA walls cut the raster into 4 x 2 = 8 components with 4 points each (48 pairs), cumulative
                  map -- every column sweeps all n rows here, where a per-component handle sweeps only its own.
  fragmented:     30 % of the cells NODATA (seed 5): one large component and thousands of small ones; 16 points on
                  nodes, cumulative map -- do the small components deepen the whole-raster hierarchy?
Per case and path: best end-to-end seconds, setup seconds (handle creates), solve seconds (the batched solve
calls), host seconds (the rest: node map, graph, components, pairs, maps), PCG iterations per column (p50, max);
for the new path the cs_b200_components call time (CUDA events around the call, labels download included, best
of 5); the largest relative resistance difference and the cumulative map difference relative to its maximum."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import circuitscape_b200 as cb
from circuitscape_b200 import solver as S

SIZE = 3163
CUM = {"write_cur_maps": "True", "write_cum_cur_map_only": "True"}


def inputs(name, size):
    g = 1.0 / np.random.default_rng(42).uniform(1.0, 10.0, size=(size, size))
    rng = np.random.default_rng(7)
    cfg = {} if name == "full_shortcut" else dict(CUM)
    if name == "walls8":
        rw = np.linspace(0, size, 5).astype(int)[1:-1]
        cw = size // 2
        g[rw, :] = 0.0
        g[:, cw] = 0.0
        rb = np.r_[0, rw + 1, size]
        cells = []
        for i in range(4):
            for c0, c1 in ((0, cw), (cw + 1, size)):
                r = rng.integers(rb[i], rb[i + 1] - 1, 4)
                c = rng.integers(c0, c1, 4)
                cells += list(c * size + r)
        cells = np.array(cells)
    else:
        if name == "fragmented":
            g[np.random.default_rng(5).random(g.shape) < 0.3] = 0.0
        on = np.flatnonzero((g > 0).ravel(order="F"))
        cells = rng.choice(on, 16, replace=False)
    rr, cc_ = cells % size + 1, cells // size + 1
    data = cb.RasterData(g, None, (rr, cc_, np.arange(1, len(cells) + 1)))
    return data, cb.Flags(is_raster=True, outputflags=cb.OutputFlags(**{k: True for k in cfg})), cfg


class Recorder:
    """times the handle creates and the batched solve calls, and collects per-column iterations"""
    SOLVES = ("solve_pairs", "solve_sources", "solve_pairs_superposed")

    def __enter__(self):
        self.setup_s = self.solve_s = 0.0
        self.iters = []
        self._saved = {("S", "construct_cholesky_factor"): S.construct_cholesky_factor,
                       ("S", "construct_raster_factor"): S.construct_raster_factor}
        for m in self.SOLVES:
            self._saved[("F", m)] = getattr(cb.B200Factor, m)
        rec = self

        def timed_create(fn):
            def create(*a, **kw):
                t0 = time.perf_counter()
                f = fn(*a, **kw)
                rec.setup_s += time.perf_counter() - t0
                return f
            return create

        def timed_solve(fn):
            def solve(f, *a, **kw):
                t0 = time.perf_counter()
                res = fn(f, *a, **kw)
                rec.solve_s += time.perf_counter() - t0
                rec.iters += list(np.asarray(res["iters"]))
                return res
            return solve
        S.construct_cholesky_factor = timed_create(S.construct_cholesky_factor)
        S.construct_raster_factor = timed_create(S.construct_raster_factor)
        for m in self.SOLVES:
            setattr(cb.B200Factor, m, timed_solve(getattr(cb.B200Factor, m)))
        return self

    def __exit__(self, *a):
        for (where, name), fn in self._saved.items():
            setattr(S if where == "S" else cb.B200Factor, name, fn)


def run(data, flags, cfg, new):
    with Recorder() as rec:
        t0 = time.perf_counter()
        out = cb.raster_pairwise(data, flags, cfg, solver=cb.CUDASolver(pairwise_raster=new))
        e2e = time.perf_counter() - t0
    it = np.asarray(rec.iters)
    return out, {"e2e_s": round(e2e, 2), "setup_s": round(rec.setup_s, 2), "solve_s": round(rec.solve_s, 2),
                 "host_s": round(e2e - rec.setup_s - rec.solve_s, 2), "columns": len(it),
                 "iters_p50": int(np.median(it)) if len(it) else 0, "iters_max": int(it.max()) if len(it) else 0}


def components_ms(data):
    import torch
    f, _ = S.construct_raster_factor(data.cellmap, None, cb.CUDASolver())
    with f:
        f.components()
        best, ncomp = np.inf, 0
        for _ in range(5):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            ncomp, _ = f.components()
            b.record()
            b.synchronize()
            best = min(best, a.elapsed_time(b))
        levels = len(f.levels())
    return round(best, 2), ncomp, levels


def case(name, size, reps):
    data, flags, cfg = inputs(name, size)
    best = {}
    outs = {}
    for _ in range(reps):
        for new in (True, False):
            out, st = run(data, flags, cfg, new)
            key = "pairwise_raster" if new else "existing"
            outs[key] = out
            if key not in best or st["e2e_s"] < best[key]["e2e_s"]:
                best[key] = st
    ms, ncomp, levels = components_ms(data)
    a, b = outs["pairwise_raster"], outs["existing"]
    Ra, Rb = a.resistances[1:, 1:], b.resistances[1:, 1:]
    ok = Rb > 0
    res = {"pairs": int(np.count_nonzero(np.triu(ok, 1))), "components": ncomp, "levels": levels,
           "components_call_ms": ms, **best,
           "max_rel_dR": float(np.max(np.abs(Ra[ok] - Rb[ok]) / Rb[ok])) if ok.any() else 0.0,
           "R_invalid_equal": bool(np.array_equal(Ra[~ok], Rb[~ok]))}
    if cfg:
        res["max_dcum_over_max_cum"] = float(np.abs(a.cum_curmap - b.cum_curmap).max() / np.abs(b.cum_curmap).max())
    return res


def main():
    args = sys.argv[1:]
    size, reps = SIZE, 2
    for flag in ("--size", "--reps"):
        if flag in args:
            i = args.index(flag)
            v = int(args[i + 1])
            del args[i:i + 2]
            size, reps = (v, reps) if flag == "--size" else (size, v)
    names = ["full_cum", "full_shortcut", "walls8", "fragmented"]
    pick = args[0].split(",") if args else names
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"gpu": smi[0] if smi else "unknown", "raster": f"{size}x{size}", "reps": reps}
    for name in names:
        if name in pick:
            res[name] = case(name, size, reps)
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()

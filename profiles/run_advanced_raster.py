"""Raster advanced mode on the 3163 x 3163 bench raster: core.raster_advanced (every solved component a column of
cs_b200_solve_advanced on one whole-raster handle) against core.advanced_kernel (one handle, hierarchy and solve
per component through hook #3, node currents on the host) on the same inputs.  Prints a JSON line after every
case; an optional first argument picks cases (comma-separated), `--size N` shrinks the raster for a dry run.

Raster: R ~ U[1, 10] (seed 42), the bench.py generator; default CUDASolver settings.  Cases:
  finite:  finite grounds (0.5 S) on a 10-cell-wide vertical band, 300 unit source cells (seed 7) -- one column.
  direct:  the same band as direct (Inf) grounds -- one column, ~31 600 Dirichlet rows.
  walls32: NODATA walls cut the raster into 8 x 4 = 32 components, each with a 3 x 3 patch of finite grounds
           and 10 unit source cells -- 32 columns, cost grows with the number of columns.
Per case and path: end-to-end seconds (the host graph build included), setup seconds (raster_advanced: create
plus set_grounds; advanced_kernel: the per-component creates), solve seconds, PCG iterations, and the largest
voltage / current map differences relative to the maps' maxima."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import circuitscape_b200 as cb
from circuitscape_b200 import core, graph
from circuitscape_b200 import solver as S

SIZE = 3163
FLAGS = cb.Flags(is_raster=True, is_advanced=True)


def raster(size):
    return 1.0 / np.random.default_rng(42).uniform(1.0, 10.0, size=(size, size))


def inputs(name, size):
    g = raster(size)
    rng = np.random.default_rng(7)
    src, gnd = np.zeros(g.shape), np.zeros(g.shape)
    if name in ("finite", "direct"):
        c0 = size // 2
        gnd[:, c0:c0 + 10] = 0.5 if name == "finite" else np.inf
        cells = rng.choice(size * size, 300, replace=False)
        src.ravel()[cells] = 1.0
        src[gnd != 0] = 0.0
        return g, src, gnd
    rw = np.linspace(0, size, 9).astype(int)[1:-1]          # 7 horizontal and 3 vertical walls
    cw = np.linspace(0, size, 5).astype(int)[1:-1]
    g[rw, :] = 0.0
    g[:, cw] = 0.0
    rb = np.r_[0, rw + 1, size]
    cb_ = np.r_[0, cw + 1, size]
    for i in range(8):
        for j in range(4):
            r0, r1, k0, k1 = rb[i], rb[i + 1] - 1, cb_[j], cb_[j + 1] - 1
            rm, km = (r0 + r1) // 2, (k0 + k1) // 2
            gnd[rm - 1:rm + 2, km - 1:km + 2] = 0.5
            rr = rng.integers(r0, r1, 10)
            kk = rng.integers(k0, k1, 10)
            src[rr, kk] = 1.0
    src[(gnd != 0) | (g == 0)] = 0.0
    return g, src, gnd


class Recorder:
    """times the per-component creates and solves of advanced_kernel and collects their iterations"""

    def __init__(self):
        self.create_s = self.solve_s = 0.0
        self.iters = 0

    def __enter__(self):
        self._create, self._solve = S.construct_cholesky_factor, cb.B200Factor.solve_rhs
        rec = self

        def create(*a, **kw):
            t0 = time.perf_counter()
            f = rec._create(*a, **kw)
            rec.create_s += time.perf_counter() - t0
            return f

        def solve(f, *a, **kw):
            t0 = time.perf_counter()
            x, it, rr = rec._solve(f, *a, **kw)
            rec.solve_s += time.perf_counter() - t0
            rec.iters += int(np.sum(it))
            return x, it, rr
        S.construct_cholesky_factor, cb.B200Factor.solve_rhs = create, solve
        return self

    def __exit__(self, *a):
        S.construct_cholesky_factor, cb.B200Factor.solve_rhs = self._create, self._solve


def case(name, size):
    g, src, gnd = inputs(name, size)
    cfg = {"remove_src_or_gnd": "keepall"}
    t0 = time.perf_counter()
    new = core.raster_advanced(cb.RasterData(g, None, None, source_map=src, ground_map=gnd), FLAGS, cfg,
                               solver=cb.CUDASolver())
    new_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    nodemap = graph.construct_node_map(g, None)
    G = graph.laplacian(graph.construct_graph(g, nodemap, False, False))
    s, gr, f = core.sources_and_grounds_from_maps(src, gnd, nodemap, G.shape[0], "keepall")
    prob = cb.AdvancedProblem(G, graph.connected_components(G), s, gr, f, nodemap, None, g, cb.CUDASolver())
    with Recorder() as rec:
        old = core.advanced_kernel(prob, FLAGS)
    old_s = time.perf_counter() - t0
    rel = lambda a, b: float(np.abs(a - b).max() / np.abs(b).max())
    return {"columns": new.stats["columns"], "solved": new.num_solves,
            "raster_advanced": {"e2e_s": round(new_s, 2), "setup_s": round(new.stats["setup_s"], 2),
                                "solve_s": round(new.stats["solve_s"], 2), "iters": new.iterations},
            "advanced_kernel": {"e2e_s": round(old_s, 2), "setup_s": round(rec.create_s, 2),
                                "solve_s": round(rec.solve_s, 2), "iters": rec.iters},
            "max_dvolt_over_max_volt": rel(new.voltmap, old.voltmap),
            "max_dcur_over_max_cur": rel(new.curmap, old.curmap)}


def main():
    args = sys.argv[1:]
    size = SIZE
    if "--size" in args:
        i = args.index("--size")
        size = int(args[i + 1])
        del args[i:i + 2]
    names = ["finite", "direct", "walls32"]
    pick = args[0].split(",") if args else names
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    res = {"gpu": smi[0] if smi else "unknown", "raster": f"{size}x{size}"}
    for name in names:
        if name in pick:
            res[name] = case(name, size)
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()

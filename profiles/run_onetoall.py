"""One-to-all / all-to-one on the 3163 x 3163 bench raster: CUDASolver(onetoall_raster=True) (every iteration a
column on one whole-raster handle) against the per-iteration path (one advanced solve per iteration through
hook #3) and the batch_one_to_all / batch_all_to_one paths.  Prints a JSON line after every case; an
optional argument picks cases (comma-separated, e.g. all_to_one_64).

Raster: 3163 x 3163, R ~ U[1, 10] (seed 42), the bench.py generator.  Focal points: P distinct cells (seed 7),
P = 16 and 64, default CUDASolver settings, cumulative current map on.
  new path:        end-to-end seconds, PCG iterations p50 / max of its columns; the same points as
                   solve_pairs columns (point 0 against each other point) for the iteration counts.
  per-iteration:   the first PER_ITER iterations, timed and extrapolated to P (setup counted once); at
                   P = 16 their R (one-to-all), voltage and current maps against the new path's.
  batch_* paths:   end to end at P = 16 only (batch_one_to_all sends a dense n x P host right-hand side)."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import circuitscape_b200 as cb
from circuitscape_b200 import core
from circuitscape_b200 import solver as S

SIZE = 3163
PER_ITER = 2


class Stop(Exception):
    pass


def raster():
    return 1.0 / np.random.default_rng(42).uniform(1.0, 10.0, size=(SIZE, SIZE))


def points(P):
    cells = np.random.default_rng(7).choice(SIZE * SIZE, size=P, replace=False)
    return (cells // SIZE + 1).astype(np.int64), (cells % SIZE + 1).astype(np.int64), np.arange(1, P + 1)


def flags(maps):
    return cb.Flags(outputflags=cb.OutputFlags(write_cur_maps=maps, write_volt_maps=maps,
                                               write_cum_cur_map_only=not maps))


def recorded(name, store):
    orig = getattr(cb.B200Factor, name)

    def rec(self, *a, **kw):
        r = orig(self, *a, **kw)
        store.append(r["iters"])
        return r
    setattr(cb.B200Factor, name, rec)
    return lambda: setattr(cb.B200Factor, name, orig)


def new_path(g, pts, one_to_all, maps=False):
    iters = []
    undo = [recorded("solve_grounded", iters), recorded("solve_sources", iters)]
    try:
        t0 = time.perf_counter()
        out = core.onetoall_kernel(cb.RasterData(g, None, pts), flags(maps), {}, solver=cb.CUDASolver(onetoall_raster=True),
                                   one_to_all=one_to_all)
        sec = time.perf_counter() - t0
    finally:
        for u in undo:
            u()
    return out, sec, np.concatenate(iters)


def pair_iters(g, pts):
    factor, nodemap = S.construct_raster_factor(g, None, cb.CUDASolver())
    with factor:
        nodes = nodemap[pts[0] - 1, pts[1] - 1] - 1
        r = factor.solve_pairs(np.full(len(nodes) - 1, nodes[0]), nodes[1:])
    return r["iters"]


def per_iteration(g, pts, one_to_all):
    """the first PER_ITER iterations of the loop, with voltage and current maps: (extrapolated s, setup s,
    s per iteration, the loop's OneToAllOutput holding the maps of those iterations)"""
    real, orig_out = core.multiple_solver, core.OneToAllOutput
    marks, captured = [], {}

    def timed(*a, **kw):
        if len(marks) == PER_ITER:
            raise Stop()
        marks.append(time.perf_counter())
        return real(*a, **kw)

    class Capture(orig_out):
        def __init__(self, *a, **kw):
            super().__init__(*a, **kw)
            captured["out"] = self
    core.multiple_solver, core.OneToAllOutput = timed, Capture
    t0 = time.perf_counter()
    try:
        core.onetoall_kernel(cb.RasterData(g, None, pts), flags(True), {}, solver=cb.CUDASolver(), one_to_all=one_to_all)
    except Stop:
        pass
    finally:
        core.multiple_solver, core.OneToAllOutput = real, orig_out
    t1 = time.perf_counter()
    setup, per = marks[0] - t0, (t1 - marks[0]) / PER_ITER
    return setup + per * len(pts[0]), setup, per, captured["out"]


def batch_path(g, pts, one_to_all):
    s = cb.CUDASolver(batch_one_to_all=one_to_all, batch_all_to_one=not one_to_all)
    t0 = time.perf_counter()
    core.onetoall_kernel(cb.RasterData(g, None, pts), flags(False), {}, solver=s, one_to_all=one_to_all)
    return time.perf_counter() - t0


def case(g, P, one_to_all):
    pts = points(P)
    out, sec, it = new_path(g, pts, one_to_all, maps=P == 16)
    it_pairs = pair_iters(g, pts)
    res = {"P": P, "new_s": round(sec, 2), "iters_p50": float(np.median(it)), "iters_max": int(it.max()),
           "pairs_iters_p50": float(np.median(it_pairs)), "pairs_iters_max": int(it_pairs.max())}
    ext, setup, per, ref = per_iteration(g, pts, one_to_all)
    res.update(per_iteration_extrapolated_s=round(ext, 1), per_iteration_setup_s=round(setup, 1),
               per_iteration_s_per_iter=round(per, 1))
    if P == 16:
        ids = list(ref.curmaps)[:PER_ITER]
        if one_to_all:        # R = the source cell's voltage (unit sources)
            k = [int(np.nonzero(pts[2] == n)[0][0]) for n in ids]
            Rn = np.array([out.resistances[i, 1] for i in k])
            Rr = np.array([ref.voltmaps[n][pts[0][i] - 1, pts[1][i] - 1] for n, i in zip(ids, k)])
            res["max_rel_dR_first_iters"] = float(np.max(np.abs(Rn - Rr) / np.abs(Rr)))
        res["max_dcur_over_max_cur_first_iters"] = max(
            float(np.abs(out.curmaps[n] - ref.curmaps[n]).max() / np.abs(ref.curmaps[n]).max()) for n in ids)
        res["max_dvolt_over_max_volt_first_iters"] = max(
            float(np.abs(out.voltmaps[n] - ref.voltmaps[n]).max() / np.abs(ref.voltmaps[n]).max()) for n in ids)
        res["batch_s"] = round(batch_path(g, pts, one_to_all), 1)
    return res


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    names = [f"{s}_{P}" for s in ("one_to_all", "all_to_one") for P in (16, 64)]
    pick = sys.argv[1].split(",") if len(sys.argv) > 1 else names       # e.g. all_to_one_64
    g = raster()
    res = {"gpu": smi[0] if smi else "unknown", "raster": f"{SIZE}x{SIZE}"}
    for name in names:
        if name in pick:
            res[name] = case(g, int(name.rsplit("_", 1)[1]), name.startswith("one"))
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()

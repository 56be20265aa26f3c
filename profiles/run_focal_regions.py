"""Pairwise mode with focal regions: the batched driver (every region pair a column of
cs_b200_solve_region_pairs on one whole-raster operator) against the per-pair path (per-pair polygon
map, host assembly and solve -- the reference's algorithm).  Prints one JSON line.

Raster: 3163 x 3163, R ~ U[1, 10] (seed 42), the bench.py generator.  Regions: square blocks of cells
carrying one focal id, at distinct positions of a coarse grid (seed 7).
  small: 16 regions of 10 x 10 (120 pairs), cumulative current map on.  The per-pair path runs the
         first 8 pairs only and is reported per pair; R and the cumulative map of those 8 pairs are
         compared with the batched driver run on the same 8 pairs (an include list).
  large: 4 regions of 150 x 150 (6 pairs), cumulative map on; both paths on every pair."""
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import circuitscape_b200 as cb
from circuitscape_b200 import graph

SIZE = 3163


def raster():
    return 1.0 / np.random.default_rng(42).uniform(1.0, 10.0, size=(SIZE, SIZE))


def regions(count, side):
    slots = SIZE // (side + 20)
    pick = np.random.default_rng(7).choice(slots * slots, size=count, replace=False)
    rows, cols, ids = [], [], []
    for p, s in enumerate(pick, start=1):
        r0, c0 = (s // slots) * (side + 20) + 10, (s % slots) * (side + 20) + 10
        rr, cc = np.meshgrid(np.arange(r0, r0 + side), np.arange(c0, c0 + side), indexing="ij")
        rows.append(rr.ravel() + 1); cols.append(cc.ravel() + 1); ids.append(np.full(rr.size, p))
    return tuple(np.concatenate(a).astype(np.int64) for a in (rows, cols, ids))


FLAGS = cb.Flags(outputflags=cb.OutputFlags(write_cur_maps=True, write_cum_cur_map_only=True))


def batched(g, points_rc, inc=None):
    iters = []
    orig = cb.B200Factor.solve_region_pairs

    def recording(self, *a, **kw):
        r = orig(self, *a, **kw)
        iters.append(r["iters"])
        return r
    cb.B200Factor.solve_region_pairs = recording
    try:
        t0 = time.perf_counter()
        out = cb.raster_pairwise(cb.RasterData(g, None, points_rc, None, inc), FLAGS, {}, solver=cb.CUDASolver())
        sec = time.perf_counter() - t0
    finally:
        cb.B200Factor.solve_region_pairs = orig
    return out, sec, np.concatenate(iters)


def per_pair(g, points_rc, pairs):
    """the per-pair path of core.raster_pairwise, pair by pair"""
    rr, cc, ids = points_rc
    R, iters, cum, secs = [], [], np.zeros(g.shape), []
    for p1, p2 in pairs:
        t0 = time.perf_counter()
        poly = graph.create_pair_polymap(g, None, points_rc, p1, p2)
        nm = graph.construct_node_map(g, poly)
        G = graph.laplacian(graph.construct_graph(g, nm, False, False))
        x, y = int(np.nonzero(ids == p1)[0][0]), int(np.nonzero(ids == p2)[0][0])
        pn = np.array([nm[rr[x] - 1, cc[x] - 1], nm[rr[y] - 1, cc[y] - 1]])
        r = cb.single_ground_all_pairs(cb.GraphProblem(G, graph.connected_components(G), pn, np.array([p1, p2]),
                                                       set(), nm, poly, g, cb.CUDASolver()), FLAGS)
        secs.append(time.perf_counter() - t0)
        R.append(r.resistances[1, 2]); iters.append(r.iterations); cum += r.cum_curmap
    return np.array(R), np.array(iters), cum, float(np.mean(secs))


def include_only(ids, pairs):
    u = np.unique(ids)
    mat = np.zeros((len(u), len(u)), dtype=np.int64)
    pos = {int(p): k for k, p in enumerate(u)}
    for a, b in pairs:
        mat[pos[a], pos[b]] = mat[pos[b], pos[a]] = 1
    return SimpleNamespace(mode="include", point_ids=u, mat=mat)


def case(g, count, side, n_per_pair):
    pts = regions(count, side)
    out, sec, it_b = batched(g, pts)
    all_pairs = [(i, j) for i in range(1, count + 1) for j in range(i + 1, count + 1)]
    sub = all_pairs[:n_per_pair]
    R_p, it_p, cum_p, sec_p = per_pair(g, pts, sub)
    sub_out, _, _ = batched(g, pts, include_only(pts[2], sub))
    R_b = np.array([sub_out.resistances[a, b] for a, b in sub])
    return {"regions": count, "side": side, "pairs": len(all_pairs), "batched_s": round(sec, 3),
            "batched_s_per_pair": round(sec / len(all_pairs), 4),
            "per_pair_s_per_pair": round(sec_p, 3), "per_pair_pairs_timed": len(sub),
            "per_pair_extrapolated_s": round(sec_p * len(all_pairs), 2),
            "iters_batched_p50": float(np.median(it_b)), "iters_batched_max": int(it_b.max()),
            "iters_per_pair_p50": float(np.median(it_p)), "iters_per_pair_max": int(it_p.max()),
            "max_rel_dR": float(np.max(np.abs(R_b - R_p) / np.abs(R_p))),
            "max_dcum_over_max_cum": float(np.abs(sub_out.cum_curmap - cum_p).max() / np.abs(cum_p).max())}


def main():
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    g = raster()
    res = {"gpu": smi[0] if smi else "unknown", "raster": f"{SIZE}x{SIZE}",
           "small": case(g, 16, 10, 8), "large": case(g, 4, 150, 6)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

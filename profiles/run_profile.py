#!/usr/bin/env python
"""Short driver for ncu captures of the hot kernels at the headline size.

  ncu --set full --clock-control none --import-source on -k regex:k_spmm -c 4 \
      -o prof_spmm python profiles/run_profile.py --rows 3163 --what spmm
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import circuitscape_b200 as cb  # noqa: E402
from circuitscape_b200 import graph  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--rows", type=int, default=3163)
ap.add_argument("--what", default="spmm", choices=["spmm", "cg", "cg8", "solve"])
ap.add_argument("--precision", default="double")
ap.add_argument("--precond", default="jacobi")
ap.add_argument("--no-mixed", action="store_true")
ap.add_argument("--reps", type=int, default=3)
a = ap.parse_args()
L, _ = graph.synthetic_raster_laplacian(a.rows, a.rows, seed=42)
n, nnz = L.shape[0], L.nnz
sv = 8 if a.precision == "double" else 4
with cb.construct_cholesky_factor(L, cb.CUDASolver(precision=a.precision, precond=a.precond, mixed=not a.no_mixed)) as f:
    if a.what == "spmm":
        for k in (1, 8):
            ms = f.bench_spmm(k, reps=a.reps, flush_l2=True)
            b = nnz * (sv + 4) + (n + 1) * 4 + 2 * n * k * sv
            print(f"spmm k={k}: {ms:.4f} ms  {b / ms / 1e6:.1f} GB/s (algorithmic {b} B)")
    elif a.what == "cg8":          # one k = 8 AMG-PCG iteration only (short ncu captures)
        ms = f.bench_cg_iter(8, reps=a.reps)
        print(f"cg_iter k=8: {ms:.4f} ms")
    elif a.what == "cg":
        for k in (1, 8):
            ms = f.bench_cg_iter(k, reps=a.reps)
            print(f"cg_iter k={k}: {ms:.4f} ms")
    else:
        nodes = graph.focal_nodes(n, 5, seed=7)
        src, dst = graph.all_pairs(nodes)
        out = f.solve_pairs(src[:8], dst[:8], accumulate=True)
        print("R", out["R"], "iters", out["iters"], f.stats())

import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import circuitscape_b200 as cb
from circuitscape_b200 import graph
rows = int(sys.argv[1])
L, _ = graph.synthetic_raster_laplacian(rows, rows, seed=42)
n = L.shape[0]
nodes = graph.focal_nodes(n, 5, seed=7)
src, dst = graph.all_pairs(nodes, limit=8)
ref = None
for prec in ("double", "single"):
    with cb.B200Factor(L.astype(np.float64 if prec == "double" else np.float32), cb.CUDASolver(precision=prec)) as f:
        t = time.time()
        o = f.solve_pairs(src, dst, raise_on_residual=False)
        dt = time.time() - t
        R = o["R"].astype(np.float64)
        if ref is None: ref = R
        print(f"{rows}^2 {prec}: {dt*1e3:.1f} ms iters {o['iters'].tolist()} relres {o['relres'].max():.2e} max rel dev R {np.abs(R-ref).max()/ref.max():.2e}", flush=True)

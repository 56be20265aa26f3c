#!/usr/bin/env python
"""Windowed vs plain SpMM on the (square-padded) SA prolongator of a raster (debug aid)."""
import os, sys, ctypes as C, subprocess, tempfile
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, scipy.sparse as sp
import circuitscape_b200 as cb
from circuitscape_b200 import graph
SO = os.path.join(tempfile.mkdtemp(), "libamgh.so")
subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", SO, os.path.join(ROOT, "tests", "amg_host_harness.cpp")])
lib = C.CDLL(SO)
import test_amg_host as t
lib.amgh_build.restype = C.c_void_p; lib.amgh_build.argtypes = [C.c_long, C.c_long, C.c_void_p, C.c_void_p, C.c_void_p]
lib.amgh_nlevels.argtypes = [C.c_void_p]; lib.amgh_dims.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 4
lib.amgh_copy.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]; lib.amgh_pinv.argtypes = [C.c_void_p, C.c_void_p]; lib.amgh_free.argtypes = [C.c_void_p]
rows = int(sys.argv[1]) if len(sys.argv) > 1 else 400
A, _ = graph.synthetic_raster_laplacian(rows, rows, seed=42)
levels, _ = t.build(lib, A)
lvl = int(sys.argv[2]) if len(sys.argv) > 2 else 0
P = sp.csr_matrix(levels[lvl]["P"]); n = P.shape[0]
print("level", lvl, "P shape", P.shape, flush=True)
Psq = sp.csr_matrix((P.data, P.indices, P.indptr), shape=(n, n))
rng = np.random.default_rng(0)
quick = len(sys.argv) > 3
for add in ((True,) if quick else (False, True)):
    if add: os.environ["CS_B200_SPMM_ADD"] = "1"
    for window in (("on",) if quick else ("on", "off")):
        with cb.B200Factor(Psq, cb.CUDASolver(window=window)) as f:
            for k in ((1,) if quick else (1, 2, 4, 8)):
                X = rng.standard_normal((n, k))
                Y = f.spmm(X)
                ref = Psq @ X + (X if add else 0)
                err = np.abs(Y - ref)
                bad = np.argwhere(err > 1e-9)
                if len(bad) and k == 1:
                    AX = Psq @ X
                    br = np.unique(bad[:, 0])
                    print("   bad row range", br.min(), br.max(), "count", len(br), "contiguous", len(br) == br.max() - br.min() + 1)
                    for r in list(br[:4]) + list(br[-2:]):
                        print(f"   row {r}: Y {Y[r,0]:.6f} ref {ref[r,0]:.6f} X {X[r,0]:.6f} AX {AX[r,0]:.6f}  Y-X {Y[r,0]-X[r,0]:.6f}  cols {Psq[r].indices.tolist()}")
                    # is Y - X equal to AX of some other row?
                    d = (Y[:, 0] - X[:, 0])
                    r = br[0]
                    cand = np.argwhere(np.abs(AX[:, 0] - d[r]) < 1e-9).ravel()
                    print("   Y-X of first bad row equals AX of rows", cand[:10].tolist())
                print(f"add={add} window={window} k={k}: max err {err.max():.3e} bad {len(bad)}" +
                      (f" first {bad[:3].tolist()} rows%256 {sorted(set((bad[:,0]%256).tolist()))[:12]} nblocks_bad {len(set((bad[:,0]//256).tolist()))} cols {sorted(set(bad[:,1].tolist()))}" if len(bad) else ""), flush=True)

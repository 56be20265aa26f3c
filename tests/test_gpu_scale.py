"""Parity at the sizes BASELINE.json names (round-1 verdict, "parity at scale"): the 10^7-node
raster against the oracle's CG+AMG run to rtol 1e-10, C3 as written (precision = single, 100 pairs,
4000 x 4000), C5 (power-law network, all-to-one) against a grounded SciPy solve.  Needs an H100 and
a few minutes of host time for the CPU references: `pytest -m gpu`.

Tolerances (SURVEY.md section 8d parity gate): effective resistances 1e-6 relative, voltages
max|dv| / R <= 1e-5 (fp64), every column through the reference's true-residual gate 1e-4
(src/core.jl:641)."""
import multiprocessing as mp

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import circuitscape_b200 as cb
from circuitscape_b200 import graph

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1500)]

_W = {}


def _tight(i):
    from oracle import amg
    A, ml, src, dst = _W["A"], _W["ml"], _W["src"], _W["dst"]
    b = np.zeros(A.shape[0]); b[src[i]] = -1.0; b[dst[i]] = 1.0
    v, it = amg.pcg(A, b, ml, rtol=1e-10, atol=0.0, itmax=1000)
    return v - v[src[i]], it


def test_headline_size_matches_oracle_cg_amg():
    """3163 x 3163 (n = 10 004 569), fp64, 3 pairs: R and voltages against the oracle's SA-AMG-PCG
    (oracle/amg.py, the reference's cg+amg role) converged to rtol 1e-10."""
    from oracle import amg
    L, _ = graph.synthetic_raster_laplacian(3163, 3163, seed=42)
    n = L.shape[0]
    nodes = graph.focal_nodes(n, 17, seed=7)
    src, dst = graph.all_pairs(nodes, limit=3)
    with cb.B200Factor(L, cb.CUDASolver()) as f:
        out = f.solve_pairs(src, dst, want_volt=True)
        lv = f.levels()
    assert out["relres"].max() < 1e-4
    assert lv[0]["A_windowed"] and len(lv) >= 5
    # the hierarchy only preconditions; the operator solved is the Laplacian as assembled.  (The
    # reference's cg+amg path adds eps*||nzval|| to every stored entry first, src/core.jl:161, which by
    # itself moves R by ~2e-6 at this size -- see bench.py `parity.vs_regularised_cg_amg`.)
    A = L.tocsr()
    _W.update(A=A, ml=amg.smoothed_aggregation(A), src=src, dst=dst)
    with mp.get_context("fork").Pool(3) as pool:
        ref = pool.map(_tight, range(3))
    for c, (v, it) in enumerate(ref):
        R = v[dst[c]]
        assert abs(out["R"][c] - R) <= 1e-6 * R, (c, out["R"][c], R)
        assert np.abs(out["volt"][:, c] - v).max() <= 1e-5 * R, c
    _W.clear()


def test_c3_single_precision_100_pairs_4000():
    """BASELINE config C3 as written: 4000 x 4000, 100 focal pairs, `precision = single`
    (src/run.jl:29): Float32 at the boundary; every column passes the true-residual gate and R agrees
    with the fp64 job to fp32 rounding.  The raster goes to the device as 64 MB of conductances
    (cs_b200_create_from_raster), not as the 1.7 GB matrix."""
    rng = np.random.default_rng(42)
    g = 1.0 / rng.uniform(1.0, 10.0, size=(4000, 4000))
    n = g.size
    nodes = graph.focal_nodes(n, 15, seed=7)
    src, dst = graph.all_pairs(nodes, limit=100)
    with cb.B200Factor.from_raster(g, cb.CUDASolver(precision="single")) as f32:
        assert f32.io_dtype == np.float32
        o32 = f32.solve_pairs(src, dst, accumulate=True)
        cum32, _ = f32.read_currents()
    assert o32["R"].dtype == np.float32 and o32["relres"].max() < 1e-4
    with cb.B200Factor.from_raster(g, cb.CUDASolver(precision="double")) as f64:
        o64 = f64.solve_pairs(src, dst, accumulate=True)
        cum64, _ = f64.read_currents()
    assert np.abs(o32["R"] - o64["R"]).max() <= 2e-6 * np.abs(o64["R"]).max()
    assert np.abs(cum32 - cum64).max() <= 1e-5 * np.abs(cum64).max()
    assert o64["iters"].max() <= 40


def test_c5_network_all_to_one_columns_vs_grounded_scipy():
    """BASELINE config C5: Barabasi-Albert-style graph (2e6 nodes, ~1e7 edges), all-to-one over 64
    focal nodes; 8 of the 64 columns are checked against SciPy's CG on the GROUNDED system (row and
    column of the ground removed: the Dirichlet form of src/raster/advanced.jl:276-304)."""
    import circuitscape_b200.core as core
    A = graph.power_law_laplacian(2_000_000, m=5, seed=11)
    n = A.shape[0]
    focal = graph.focal_nodes(n, 64, seed=5)
    with cb.B200Factor(A, cb.CUDASolver()) as f:
        pv, iters, relres, cols = core.all_to_one_batched(f, focal, device_resident=True)
        assert relres.max() < 1e-4 and len(cols) == 64
        columns = []
        for c in range(8):
            w = np.ones(len(focal)); w[c] = -(len(focal) - 1.0)
            columns.append((focal, w))
        o = f.solve_sources(columns, focal[:8], want_volt=True)
    volt = o["volt"]
    assert np.abs(pv[:8] - volt[focal].T).max() <= 1e-9 * np.abs(volt).max()     # probe rows == full columns
    d = A.diagonal()
    for c in range(8):
        gnd = int(focal[c])
        keep = np.ones(n, dtype=bool); keep[gnd] = False
        Ag = A[keep][:, keep].tocsr()
        b = np.zeros(n)
        b[focal] = 1.0
        b[gnd] = 0.0
        bg = b[keep]
        M = spla.LinearOperator(Ag.shape, matvec=lambda x, dg=d[keep]: x / dg)
        x, info = spla.cg(Ag, bg, rtol=1e-10, atol=0.0, maxiter=2000, M=M)
        assert info == 0
        v = np.zeros(n); v[keep] = x
        got = volt[:, c]
        assert np.abs(got - v).max() <= 1e-6 * np.abs(v).max(), c

"""The host-side smoothed-aggregation setup (circuitscape_b200/csrc/amg_host.hpp),
checked without a GPU: Galerkin identities of the hierarchy and convergence of the
Jacobi-smoothed V(1,1)-PCG it defines (the same cycle the device runs)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import scipy.sparse as sp

from circuitscape_b200 import graph

from .reference_ops import vcycle

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("amgh") / "libamgh.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so,
                           os.path.join(HERE, "amg_host_harness.cpp")])
    lib = C.CDLL(so)
    lib.amgh_build.restype = C.c_void_p
    lib.amgh_build.argtypes = [C.c_long, C.c_long, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.amgh_nlevels.argtypes = [C.c_void_p]
    lib.amgh_dims.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 4
    lib.amgh_copy.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.amgh_pinv.argtypes = [C.c_void_p, C.c_void_p]
    lib.amgh_free.argtypes = [C.c_void_p]
    return lib


def build(lib, A):
    A = sp.csr_matrix(A, dtype=np.float64)
    A.sort_indices()
    ptr = np.ascontiguousarray(A.indptr, dtype=np.int32)
    idx = np.ascontiguousarray(A.indices, dtype=np.int32)
    val = np.ascontiguousarray(A.data)
    h = lib.amgh_build(A.shape[0], A.nnz, ptr.ctypes.data, idx.ctypes.data, val.ctypes.data)
    levels = []
    for l in range(lib.amgh_nlevels(h)):
        mats = []
        for which in range(3):
            nr, nc, nnz = C.c_long(), C.c_long(), C.c_long()
            om = C.c_double()
            lib.amgh_dims(h, l, which, C.byref(nr), C.byref(nc), C.byref(nnz), C.byref(om))
            if nr.value == 0:
                mats.append(None)
                continue
            p = np.zeros(nr.value + 1, dtype=np.int32)
            i = np.zeros(nnz.value, dtype=np.int32)
            v = np.zeros(nnz.value)
            lib.amgh_copy(h, l, which, p.ctypes.data, i.ctypes.data, v.ctypes.data)
            mats.append(sp.csr_matrix((v, i, p), shape=(nr.value, nc.value)))
        levels.append(dict(A=mats[0], P=mats[1], R=mats[2], omega=om.value))
    nc = levels[-1]["A"].shape[0]
    pinv = np.zeros((nc, nc))
    lib.amgh_pinv(h, pinv.ctypes.data)
    lib.amgh_free(h)
    return levels, pinv


def pcg(A, b, M, rtol=1e-6, itmax=500):
    x = np.zeros_like(b); r = b.copy(); z = M(r); p = z.copy(); g = r @ z
    eps = 1.5e-8 + rtol * np.sqrt(g); it = 0
    while np.sqrt(abs(g)) > eps and it < itmax:
        Ap = A @ p; a = g / (p @ Ap); x += a * p; r -= a * Ap
        z = M(r); gn = r @ z; p = z + (gn / g) * p; g = gn; it += 1
    return x, it


@pytest.mark.parametrize("kind", ["uniform", "lognormal_holes"])
def test_hierarchy_and_convergence(harness, kind):
    if kind == "uniform":
        A, _ = graph.synthetic_raster_laplacian(120, 90, seed=1)
    else:
        rng = np.random.default_rng(2)
        g = 1.0 / np.exp(rng.normal(0, 1.5, (120, 90)))
        g[rng.random(g.shape) < 0.05] = 0
        nm = graph.construct_node_map(g)
        G = graph.laplacian(graph.construct_graph(g, nm, False, False))
        big = max(graph.connected_components(G), key=len) - 1
        A = G[big][:, big].tocsr()
    levels, pinv = build(harness, A)
    assert len(levels) >= 3 and levels[-1]["A"].shape[0] <= 200
    opc = sum(l["A"].nnz for l in levels) / A.nnz
    assert opc < 1.6
    for l in range(len(levels) - 1):
        L = levels[l]
        assert abs(L["R"] - L["P"].T).max() < 1e-15
        Ac = (L["R"] @ L["A"] @ L["P"]).tocsr()
        assert abs(Ac - levels[l + 1]["A"]).max() < 1e-12 * abs(Ac).max()
        # constants stay in the (near) null space:  A_c (P^T-consistent candidate) ~ 0
        assert np.abs(L["A"] @ np.ones(L["A"].shape[0])).max() < 1e-9 if l == 0 else True
    Ac = levels[-1]["A"].toarray()
    assert np.abs(Ac @ pinv @ Ac - Ac).max() < 1e-9 * np.abs(Ac).max()
    n = A.shape[0]
    b = np.zeros(n); b[3] = -1.0; b[n - 5] = 1.0
    x, it = pcg(A, b, lambda r: vcycle(levels, r, pinv))
    assert it <= 30, it
    assert np.linalg.norm(A @ x - b) / np.sqrt(2) < 1e-4
    import scipy.sparse.linalg as spla
    keep = np.arange(1, n)
    xr = np.zeros(n); xr[1:] = spla.splu(A[keep][:, keep].tocsc()).solve(b[1:])
    Rr = xr[n - 5] - xr[3]
    assert abs((x[n - 5] - x[3]) - Rr) / Rr < 1e-6


def test_spd_with_grounds_and_hub(harness):
    rng = np.random.default_rng(5)
    n = 4000
    rows = np.repeat(np.arange(3, n), 3)
    cols = (rng.random(rows.size) ** 2 * rows).astype(np.int64)
    rows = np.concatenate([rows, np.zeros(600, dtype=np.int64)])
    cols = np.concatenate([cols, np.arange(1, 601)])
    keep = rows != cols
    W = sp.coo_matrix((rng.uniform(0.1, 1, keep.sum()), (rows[keep], cols[keep])), shape=(n, n)).tocsr()
    A = graph.laplacian(W + W.T)
    g = np.zeros(n); g[10] = 2.0
    M = (A + sp.diags(g)).tocsr()
    levels, pinv = build(harness, M)
    # expander-like graph: the densification guard may stop coarsening early (possibly at once,
    # in which case the device solver is plain Jacobi-PCG); whatever hierarchy comes out must
    # still define a convergent symmetric preconditioner
    for l in range(len(levels) - 1):
        assert levels[l + 1]["A"].nnz <= levels[l]["A"].nnz
    b = rng.standard_normal(n)
    M_apply = (lambda r: vcycle(levels, r, pinv)) if len(levels) > 1 else (lambda r: r / M.diagonal())
    x, it = pcg(M, b, M_apply, rtol=1e-8, itmax=2000)
    assert it <= 600, it
    assert np.linalg.norm(M @ x - b) / np.linalg.norm(b) < 1e-6


def test_windowed_form_matches_csr(harness):
    """win_host.hpp: the segment windows, 16-bit local columns, packed permutation and
    row offsets reproduce y = A x exactly (host emulation of the TMA-staged kernel)."""
    harness.winh_spmv.restype = C.c_long
    harness.winh_spmv.argtypes = [C.c_long, C.c_long] + [C.c_void_p] * 7
    rng = np.random.default_rng(0)
    mats = []
    A, _ = graph.synthetic_raster_laplacian(333, 217, seed=1)
    mats.append(("raster", A, True))
    g = 1.0 / np.exp(rng.normal(0, 1.0, (150, 140))); g[rng.random(g.shape) < 0.1] = 0
    nm = graph.construct_node_map(g)
    G = graph.laplacian(graph.construct_graph(g, nm, False, True))
    mats.append(("holes4", G, True))
    n = 6000
    rows = np.repeat(np.arange(3, n), 3); cols = (rng.random(rows.size) ** 2 * rows).astype(np.int64)
    rows = np.concatenate([rows, np.zeros(3000, dtype=np.int64)]); cols = np.concatenate([cols, np.arange(1, 3001)])
    k = rows != cols
    W = sp.coo_matrix((rng.random(k.sum()) + 0.1, (rows[k], cols[k])), shape=(n, n)).tocsr()
    mats.append(("powerlaw", graph.laplacian(W + W.T), False))
    for name, A, expect_win in mats:
        A = sp.csr_matrix(A); A.sort_indices()
        n = A.shape[0]
        x = rng.standard_normal(n)
        y = np.zeros(n)
        ptr = A.indptr.astype(np.int32); idx = A.indices.astype(np.int32); val = A.data.astype(np.float64)
        nb, mw = C.c_long(), C.c_long()
        nwin = harness.winh_spmv(n, A.nnz, ptr.ctypes.data, idx.ctypes.data, val.ctypes.data,
                                 x.ctypes.data, y.ctypes.data, C.byref(nb), C.byref(mw))
        assert nwin >= 0, (name, nwin)
        ref = A @ x
        assert np.abs(y - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max()), name
        if expect_win:
            assert nwin >= 0.95 * nb.value, (name, nwin, nb.value)
            assert mw.value <= 512


from hypothesis import HealthCheck, given, settings, strategies as st  # noqa: E402
import scipy.sparse.linalg as spla  # noqa: E402


@settings(max_examples=25, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(nr=st.integers(15, 40), nc=st.integers(15, 40), seed=st.integers(0, 2**31 - 1),
       sigma=st.sampled_from([0.0, 1.0, 2.5]), holes=st.sampled_from([0.0, 0.1, 0.3]), four=st.booleans(),
       grounded=st.booleans())
def test_random_rasters_give_a_sound_hierarchy(harness, nr, nc, seed, sigma, holes, four, grounded):
    """Whatever raster comes in (contrast, holes, 4/8 neighbours, singular or grounded): R = P^T,
    Galerkin coarse operators, a symmetric V-cycle, and PCG converging to the true solution."""
    rng = np.random.default_rng(seed)
    g = np.exp(rng.normal(0.0, sigma, (nr, nc))) if sigma > 0 else rng.uniform(0.1, 1.0, (nr, nc))
    g[rng.random((nr, nc)) < holes] = 0.0
    nm = graph.construct_node_map(g)
    if nm.max() < 2:
        return
    G = graph.laplacian(graph.construct_graph(g, nm, False, four))
    comp = max(graph.connected_components(G), key=len) - 1
    if len(comp) < 2:
        return
    A = G[comp][:, comp].tocsr()
    n = A.shape[0]
    if grounded:
        d = np.zeros(n); d[rng.integers(0, n)] = rng.uniform(0.1, 2.0)
        A = (A + sp.diags(d)).tocsr()
    levels, pinv = build(harness, A)
    for l in range(len(levels) - 1):
        L = levels[l]
        assert abs(L["R"] - L["P"].T).max() < 1e-15
        Ac = (L["R"] @ L["A"] @ L["P"]).tocsr()
        assert abs(Ac - levels[l + 1]["A"]).max() <= 1e-12 * max(1e-300, abs(Ac).max())
        # damped Jacobi must stay convergent on every level: omega * lambda_max(D^-1 A) < 2
        d = L["A"].diagonal()
        if d.min() > 0 and L["A"].shape[0] > 2:
            Dm = sp.diags(1.0 / np.sqrt(d))
            lam = spla.eigsh((Dm @ L["A"] @ Dm).asfptype(), k=1, which="LA", return_eigenvectors=False, tol=1e-4)[0]
            assert 0 < L["omega"] * lam < 2.0, (L["omega"], lam)
    M = (lambda r: vcycle(levels, r, pinv)) if len(levels) > 1 else None
    if M is not None:
        u, w = rng.standard_normal(n), rng.standard_normal(n)
        if not grounded:
            u -= u.mean(); w -= w.mean()
        assert abs(u @ M(w) - w @ M(u)) <= 1e-9 * (np.linalg.norm(u) * np.linalg.norm(M(w)) + 1e-300)
        assert u @ M(u) > 0
    b = np.zeros(n); b[0] += 1.0; b[n - 1] -= 1.0
    if grounded:
        b[0] += 0.5
    x, it = pcg(A, b, M if M is not None else (lambda r: r / A.diagonal()), rtol=1e-8, itmax=400)
    assert np.linalg.norm(A @ x - b) / np.linalg.norm(b) < 1e-5
    if M is not None:
        assert it <= 120, it


@settings(max_examples=40, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(n=st.integers(1, 700), ncols=st.integers(1, 900), seed=st.integers(0, 2**31 - 1),
       kind=st.sampled_from(["banded", "two-bands", "scattered", "long-rows", "empty-rows"]))
def test_windowed_form_random_rectangular(harness, n, ncols, seed, kind):
    """win_host.hpp on arbitrary rectangular CSR (the transfer operators are rectangular): segment
    windows, the direct-gather fallback for blocks that do not fit, rows longer than a block,
    empty rows -- the host emulation of the kernel's walk must reproduce y = A x."""
    harness.winh_spmv_rect.restype = C.c_long
    harness.winh_spmv_rect.argtypes = [C.c_long, C.c_long, C.c_long] + [C.c_void_p] * 7
    rng = np.random.default_rng(seed)
    rows, cols = [], []
    for i in range(n):
        c0 = int(i * ncols / max(n, 1))
        if kind == "banded":
            cs = c0 + rng.integers(-4, 5, size=rng.integers(1, 8))
        elif kind == "two-bands":
            cs = np.concatenate([c0 + rng.integers(-2, 3, 3), (c0 + ncols // 2) % ncols + rng.integers(-2, 3, 3)])
        elif kind == "scattered":
            cs = rng.integers(0, ncols, size=rng.integers(1, 12))
        elif kind == "long-rows":
            cs = rng.integers(0, ncols, size=1300 if i % 97 == 0 else 3)
        else:
            cs = c0 + rng.integers(-3, 4, size=0 if i % 3 == 0 else 4)
        cs = np.unique(np.clip(cs, 0, ncols - 1))
        rows += [i] * len(cs); cols += list(cs)
    A = sp.csr_matrix((rng.standard_normal(len(rows)), (rows, cols)), shape=(n, ncols))
    A.sort_indices()
    if A.nnz == 0:
        return
    x = rng.standard_normal(ncols)
    y = np.full(n, np.nan)
    ptr = A.indptr.astype(np.int32); idx = A.indices.astype(np.int32); val = A.data.astype(np.float64)
    nb, mw = C.c_long(), C.c_long()
    nwin = harness.winh_spmv_rect(n, ncols, A.nnz, ptr.ctypes.data, idx.ctypes.data, val.ctypes.data,
                                  x.ctypes.data, y.ctypes.data, C.byref(nb), C.byref(mw))
    assert nwin >= 0
    ref = A @ x
    assert np.all(np.isfinite(y))
    assert np.abs(y - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())
    assert mw.value <= 1024

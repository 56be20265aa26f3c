"""Network mode with its per-solve output work on the device: branch currents of a handle's stored strictly-lower
entries (cs_b200_branch_index, k_branch_cur), per-pair branch currents and their cumulative vector
(cs_b200_solve_pairs_branch, CUDASolver(branch_on_device=True)), and network advanced mode on one whole-graph
operator (cs_b200_solve_advanced_network, core.network_advanced) with one 1e-8 cut over the summed voltages.

CPU: the drivers on a SciPy double of the new handle methods (defined here) against the network goldens and the
oracle on random networks; no stack in any k_branch_cur instantiation; the new symbols and their argument
rejection without a device.
GPU: the branch order on random CSR inputs; per-pair branch currents against the host formula over every panel
width, precision and SpMM form, and at the 1e-8 cut; the cumulative branch vector; the other entries left as
they were; network_advanced against the oracle and the goldens, including the global cut."""

import ctypes

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla
from hypothesis import HealthCheck, given, settings, strategies as st

import circuitscape_b200 as cb
from circuitscape_b200 import _lib, graph
from circuitscape_b200 import core as core_mod
from circuitscape_b200 import solver as S
from oracle import circuitscape_oracle as co

from . import cases
from .fake_factor import FakeFactor
from .test_driver_vs_oracle import networks
from .test_transfer_kernels import _mangled, _resource_usage

POLICIES = ["keepall", "rmvsrc", "rmvgnd", "rmvall"]


# ---------------------------------------------------------------------------
# the handle's branch definitions restated in SciPy
# ---------------------------------------------------------------------------
def lower_branches(A):
    """(lo, hi, |a_hi,lo|) of the stored strictly-lower entries, ordered by hi, then lo."""
    low = sp.tril(sp.csr_matrix(A), k=-1).tocoo()
    order = np.lexsort((low.col, low.row))
    return low.col[order].astype(np.int64), low.row[order].astype(np.int64), np.abs(low.data[order])


def branch_columns(A, V):
    """Branch currents of every column of V (n, k): b = |a_hi,lo| (v_lo - v_hi), cut at 1e-8 of the column's
    maximum over the stored upper entries (k_cur_max), returned as |b| (nb, k)."""
    lo, hi, a = lower_branches(A)
    up = sp.triu(sp.csr_matrix(A), k=1).tocoo()
    out = np.zeros((len(lo), V.shape[1]))
    for c in range(V.shape[1]):
        v = V[:, c]
        d = a * (v[lo] - v[hi])
        mp = (np.abs(up.data) * (v[up.row] - v[up.col])).max(initial=-1e300)
        with np.errstate(divide="ignore", invalid="ignore"):
            out[:, c] = np.where(~(np.abs(d / mp) < 1e-8), np.abs(d), 0.0)
    return out


class NetworkDouble(FakeFactor):
    """CPU double of B200Factor.branch_index / solve_pairs(want_branch) / read_branch_currents /
    set_grounds + solve_advanced_network."""

    fg = None

    def reset_currents(self):
        super().reset_currents()
        self.cum_branch = np.zeros(len(lower_branches(self.A)[0]))

    def branch_index(self):
        return lower_branches(self.A)[:2]

    def read_branch_currents(self):
        return self.cum_branch.copy()

    def set_grounds(self, finite=None, dirichlet=None):
        super().set_grounds(finite, dirichlet)
        self.fg = None if finite is None else np.asarray(finite, dtype=np.float64).copy()

    def solve_pairs(self, src, dst, weight=None, want_volt=False, want_curr=False, accumulate=False,
                    want_branch=False, **kw):
        res = super().solve_pairs(src, dst, weight, want_volt=True, want_curr=want_curr, accumulate=accumulate)
        B = branch_columns(self.A, res["volt"]) if want_branch else None
        if want_branch and accumulate:
            w = np.ones(len(src)) if weight is None else np.asarray(weight, dtype=np.float64)
            self.cum_branch += B @ w
        res["branch"] = B
        if not want_volt:
            res["volt"] = None
        return res

    def solve_advanced_network(self, sets, gset, sources, owner, want_volt=False, want_curr=False,
                               want_branch=False, **kw):
        n, k = self.n, len(gset)
        owner = np.asarray(owner)
        assert len(owner) == n and owner.min(initial=-1) >= -1 and owner.max(initial=-1) < k
        assert all(s >= 0 for s in gset) or self.fg is not None
        v = np.zeros(n)
        for c in range(k):
            rows, vals = (np.asarray(x) for x in sources[c])
            g = np.asarray(sets[gset[c]]) if gset[c] >= 0 else np.zeros(0, dtype=np.int64)
            assert np.all(owner[rows] == c) and np.all(owner[g] == c)
            b = np.zeros(n)
            np.add.at(b, rows.astype(np.int64), vals.astype(np.float64))
            keep = np.nonzero((owner == c) & ~np.isin(np.arange(n), g))[0]
            v[keep] = spla.splu(self.A[keep][:, keep].tocsc()).solve(b[keep])
        return dict(volt=v if want_volt else None,
                    curr=co.get_node_currents(self.A, v, self.fg) if want_curr else None,
                    branch=branch_columns(self.A, v[:, None])[:, 0] if want_branch else None,
                    iters=np.zeros(k, dtype=np.int64), relres=np.zeros(k))


@pytest.fixture
def network_double(monkeypatch):
    monkeypatch.setattr(S, "construct_cholesky_factor", lambda m, s, **kw: NetworkDouble(m, s, **kw))
    monkeypatch.setattr(S, "multiple_solve", lambda s, m, b: FakeFactor(m, s).solve_rhs(np.asarray(b))[0])


def _check_cum_branch(prob, r, exp):
    v = exp["branch_currents_cum.txt"].copy()
    v[:, :2] += 1
    mine = np.column_stack([prob.coords[0], prob.coords[1], r.cum_branch])
    mine = mine[~np.isclose(mine[:, 2], 0.0, atol=1e-6)]
    assert mine.shape == v.shape
    assert np.sum((cases.sorted_rows(mine) - cases.sorted_rows(v)) ** 2) < 1e-6


def _pairwise_vs_oracle(raw, fp, solver):
    cfg = {"data_type": "network", "scenario": "pairwise", "habitat_map_is_resistances": "False",
           "write_cur_maps": "True", "write_volt_maps": "True"}
    inputs = {"habitat_file": ("txtlist", raw, np.zeros(0)), "point_file": ("txtlist", fp.reshape(-1, 1), np.zeros(0))}
    want = co.network_pairwise(cfg, inputs)
    i, j, v, _ = co.load_graph(raw, False)
    G, cc = co.network_graph(i, j, v)
    got = cb.single_ground_all_pairs(cb.GraphProblem(G, cc, fp, fp, set(), None, None, None, solver, (i, j)),
                                     cb.Flags.from_cfg(cfg))
    rel = lambda a, b: np.abs(a - b).max(initial=0.0) <= 1e-8 * max(1.0, np.abs(b).max(initial=0.0))
    assert rel(got.resistances, want.resistances)
    assert set(got.branch) == set(want.branch)
    srt = lambda t: (lambda m: m[np.lexsort(m.T[::-1])])(np.column_stack([np.asarray(x, dtype=float) for x in t]))
    for key in want.branch:
        gb, wb = srt(got.branch[key]), srt(want.branch[key])
        assert gb.shape == wb.shape and rel(gb, wb)
    assert rel(got.cum_node, want.cum_node)
    assert rel(got.cum_branch, want.cum_branch)


def _advanced_problem(raw, rng, kind):
    i, j, v, _ = co.load_graph(raw, False)
    G, cc = co.network_graph(i, j, v)
    n = G.shape[0]
    sources = np.where(rng.random(n) < 0.3, rng.uniform(0.5, 2.0, n), 0.0)
    grounds = np.where(rng.random(n) < 0.3, rng.uniform(0.5, 2.0, n), 0.0)
    if kind == "inf":
        grounds = np.where(grounds != 0, np.inf, 0.0)
    elif kind == "mixed":
        grounds = np.where((grounds != 0) & (rng.random(n) < 0.5), np.inf, grounds)
    return G, cc, sources, grounds


def _advanced_agree(got, want, rel=1e-8):
    close = lambda a, b: np.abs(a - b).max(initial=0.0) <= rel * max(1.0, np.abs(b).max(initial=0.0))
    assert close(got.voltages, want.voltages)
    assert close(got.node_currents, want.node_currents)
    wr, wc, wv = want.branch                                    # the oracle keeps 0-based rows
    assert np.array_equal(got.branch[0], np.asarray(wr) + 1) and np.array_equal(got.branch[1], np.asarray(wc) + 1)
    assert close(got.branch[2], wv)


# ---------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("i", range(1, 4))
def test_device_branch_pairwise_goldens_on_the_double(network_double, golden, i):
    prob, flags, exp = cases.network_pairwise_problem(golden, f"sgNetworkVerify{i}",
                                                      cb.CUDASolver(branch_on_device=True))
    r = cb.single_ground_all_pairs(prob, flags)
    cases.check_network_pairwise(r, exp)
    _check_cum_branch(prob, r, exp)


@pytest.mark.parametrize("i", range(1, 4))
def test_network_advanced_goldens_on_the_double(network_double, golden, i):
    prob, flags, exp = cases.advanced_problem(golden, f"mgNetworkVerify{i}", cb.CUDASolver())
    r = cb.network_advanced(prob, flags)
    cases.check_advanced(r, exp, flags)
    assert r.num_solves > 0


@settings(max_examples=60, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(p=networks(), device=st.booleans())
def test_pairwise_matches_oracle_with_and_without_device_branches(network_double, p, device):
    raw, fp = p
    _pairwise_vs_oracle(raw, fp, cb.CUDASolver(branch_on_device=device))


@settings(max_examples=80, deadline=None, derandomize=True, suppress_health_check=[HealthCheck.function_scoped_fixture])
@given(p=networks(), seed=st.integers(0, 2**31 - 1), policy=st.sampled_from(POLICIES),
       kind=st.sampled_from(["finite", "inf", "mixed"]))
def test_network_advanced_matches_oracle(network_double, p, seed, policy, kind):
    G, cc, sources, grounds = _advanced_problem(p[0], np.random.default_rng(seed), kind)
    s, g, f = co.resolve_conflicts(sources, grounds, policy)
    try:
        want = co.advanced_kernel(G, cc, s, g, f)
    except Exception:
        return
    got = cb.network_advanced(cb.AdvancedProblem(G, cc, *cb.resolve_conflicts(sources, grounds, policy),
                                                 solver=cb.CUDASolver()), cb.Flags(is_raster=False, is_advanced=True))
    _advanced_agree(got, want)


def test_network_advanced_solves_nothing_without_a_handle(network_double, monkeypatch):
    G, cc = co.network_graph(np.array([1., 2, 4]), np.array([2., 3, 5]), np.ones(3))
    n = G.shape[0]
    monkeypatch.setattr(S, "construct_cholesky_factor", lambda *a, **kw: pytest.fail("no handle expected"))
    s = np.zeros(n); s[0] = 1.0
    got = cb.network_advanced(cb.AdvancedProblem(G, cc, s, np.zeros(n), np.array([-9999.0])),
                              cb.Flags(is_raster=False, is_advanced=True))
    _advanced_agree(got, co.advanced_kernel(G, cc, s, np.zeros(n), np.array([-9999.0])))
    assert got.num_solves == 0 and not np.any(got.node_currents)


def test_device_branch_order_is_checked(network_double, golden, monkeypatch):
    prob, flags, _ = cases.network_pairwise_problem(golden, "sgNetworkVerify1", cb.CUDASolver(branch_on_device=True))
    monkeypatch.setattr(NetworkDouble, "branch_index", lambda self: tuple(a[::-1] for a in lower_branches(self.A)[:2]))
    with pytest.raises(RuntimeError, match="branch order"):
        cb.single_ground_all_pairs(prob, flags)


BRANCH_KERNELS = [("k_branch_cur", t, kt) for t in ("float", "double") for kt in (1, 2, 4, 8)]


@pytest.mark.parametrize("kernel", BRANCH_KERNELS, ids=lambda k: "-".join(map(str, k)))
def test_branch_kernels_do_not_spill(kernel):
    funcs = _resource_usage()
    key = _mangled(kernel[0], kernel[1:])
    hits = {f: s for f, s in funcs.items() if key in f}
    assert hits, f"{kernel} is not in the library"
    assert all(s == 0 for s in hits.values()), hits


def test_new_entries_are_exported_and_reject_bad_arguments_without_a_device():
    lib = _lib.load()
    for name in ("cs_b200_branch_index", "cs_b200_solve_pairs_branch", "cs_b200_read_branch_currents",
                 "cs_b200_solve_advanced_network"):
        assert name in _lib.EXPORTED_SYMBOLS and hasattr(ctypes.CDLL(_lib.LIB_PATH), name)
    assert lib.cs_b200_version() == 1008
    nb = ctypes.c_int64()
    assert lib.cs_b200_branch_index(None, ctypes.byref(nb), None, None) == _lib.ERR_ARG
    assert lib.cs_b200_read_branch_currents(None, None) == _lib.ERR_ARG
    i64 = lambda *v: np.array(v, dtype=np.int64)
    src, dst, R = i64(0, 1), i64(1, 2), np.zeros(2)
    rc = lib.cs_b200_solve_pairs_branch(None, 2, src.ctypes.data, dst.ctypes.data, None, 1e-6, 100, R.ctypes.data,
                                        None, None, 0, None, None, None)
    assert rc == _lib.ERR_ARG and b"solve_pairs_branch" in lib.cs_b200_last_error(None)
    vals = np.ones(8)

    def call(ptr, rows, gset, sptr, srows, owner):
        rc = lib.cs_b200_solve_advanced_network(None, len(ptr) - 1, ptr.ctypes.data, rows.ctypes.data, len(gset),
                                                gset.ctypes.data, sptr.ctypes.data, srows.ctypes.data,
                                                vals.ctypes.data, None if owner is None else owner.ctypes.data,
                                                1e-6, 100, None, None, None, None, None)
        return rc, lib.cs_b200_last_error(None).decode()

    ptr, rows = i64(0, 2, 3), i64(4, 7, 9)
    sptr, srows = i64(0, 1, 3), i64(5, 1, 2)
    owner = i64(*([0] * 10))
    rc, msg = call(ptr, rows, i64(0, 1), sptr, srows, None)
    assert rc == _lib.ERR_ARG and "owner" in msg
    rc, msg = call(ptr, rows, i64(0, -1), sptr, srows, owner)
    assert rc == _lib.ERR_ARG and "no direct grounds" in msg
    rc, msg = call(ptr, rows, i64(0, 1), sptr, i64(7, 1, 2), owner)
    assert rc == _lib.ERR_ARG and "on its ground set" in msg
    rc, msg = call(ptr, rows, i64(0, 1), sptr, srows, owner)    # well-formed: only the missing handle is left
    assert rc == _lib.ERR_ARG and "null handle" in msg


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
def _random_laplacian(n, seed, zeros=0):
    """A connected random graph's Laplacian; `zeros` symmetric pairs stored as explicit zeros."""
    rng = np.random.default_rng(seed)
    e = np.column_stack([np.arange(1, n), rng.integers(0, np.arange(1, n))])          # a random tree
    e = np.vstack([e, rng.integers(0, n, (2 * n, 2))])
    e = e[e[:, 0] != e[:, 1]]
    w = rng.uniform(0.1, 1.0, len(e))
    A = sp.coo_matrix((np.r_[w, w], (np.r_[e[:, 0], e[:, 1]], np.r_[e[:, 1], e[:, 0]])), shape=(n, n)).tocsr()
    L = graph.laplacian(A)
    if zeros:
        z = rng.integers(0, n, (zeros, 2))
        z = z[(z[:, 0] != z[:, 1]) & (np.asarray(L[z[:, 0], z[:, 1]]).ravel() == 0)]
        coo = L.tocoo()
        L = sp.csr_matrix((np.r_[coo.data, np.zeros(2 * len(z))],
                           (np.r_[coo.row, z[:, 0], z[:, 1]], np.r_[coo.col, z[:, 1], z[:, 0]])), shape=(n, n))
        L.sum_duplicates()
        L.sort_indices()
    return L


def _triu_order(A):
    coo = sp.triu(sp.csr_matrix(A), k=1).tocoo()
    order = np.lexsort((coo.row, coo.col))
    return coo.row[order], coo.col[order]


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_branch_index_is_the_upper_triangle_order(seed):
    L = _random_laplacian(500 + 300 * seed, seed, zeros=200)
    assert (L.data == 0).sum() > 0
    with cb.B200Factor(L, cb.CUDASolver()) as f:
        lo, hi = f.branch_index()
        row, col = _triu_order(L)
        assert np.array_equal(lo, row) and np.array_equal(hi, col)
        assert f.read_branch_currents().shape == (len(lo),) and not f.read_branch_currents().any()


@pytest.mark.gpu
def test_branch_index_rejects_rows_that_do_not_ascend():
    L = _random_laplacian(300, 5)
    ci = L.indices.copy()
    r = int(np.argmax(np.diff(L.indptr)))                    # a row with several entries, reversed
    ci[L.indptr[r]:L.indptr[r + 1]] = ci[L.indptr[r]:L.indptr[r + 1]][::-1].copy()
    vals = L.data.copy()
    vals[L.indptr[r]:L.indptr[r + 1]] = vals[L.indptr[r]:L.indptr[r + 1]][::-1].copy()
    lib = _lib.load()
    solver = cb.CUDASolver(precond="jacobi", window="off", setup="host")
    opts = cb.B200Factor._opts(solver)
    h = ctypes.c_void_p()
    rp = np.ascontiguousarray(L.indptr, dtype=np.int32)
    ci = np.ascontiguousarray(ci, dtype=np.int32)
    _lib.check(lib, None, lib.cs_b200_create(L.shape[0], L.nnz, _lib._ptr(rp), _lib._ptr(ci), _lib._ptr(vals), 32, 0,
                                             _lib.F64, 0, ctypes.byref(opts), ctypes.byref(h)))
    try:
        nb = ctypes.c_int64()
        assert lib.cs_b200_branch_index(h, ctypes.byref(nb), None, None) == _lib.ERR_ARG
        assert f"row {r}".encode() in lib.cs_b200_last_error(h)
    finally:
        lib.cs_b200_destroy(h)


def _solver(prec, window):
    return cb.CUDASolver(rtol=1e-6 if prec == "single" else 1e-12, mixed=prec == "mixed", window=window,
                         precision="single" if prec == "single" else "double", f32_compute=prec == "single")


@pytest.mark.gpu
@pytest.mark.parametrize("window", ["on", "off"])
@pytest.mark.parametrize("prec", ["fp64", "mixed", "single"])
def test_per_pair_branch_currents_match_the_host_formula(prec, window):
    # a raster graph with NODATA holes: large enough for the windowed SpMM form, and no stencil form
    rng = np.random.default_rng(3)
    g = 1.0 / rng.uniform(1.0, 10.0, size=(190, 130))
    g[rng.random(g.shape) < 0.04] = 0.0
    nm = graph.construct_node_map(g, None)
    G = graph.laplacian(graph.construct_graph(g, nm, False, False))
    big = max(graph.connected_components(G), key=len) - 1
    L = G[big][:, big].tocsr()
    rng = np.random.default_rng(9)
    with cb.B200Factor(L, _solver(prec, window)) as f:
        assert f.operator_form() == ("windowed" if window == "on" else "csr")
        comp = np.arange(1, L.shape[0] + 1)
        nb = len(f.branch_index()[0])
        tol = 1e-4 if prec == "single" else 1e-12
        for k in range(1, 18):                                     # every KT, partial panels
            src = rng.choice(L.shape[0], k)
            dst = (src + 1 + rng.integers(0, L.shape[0] - 1, k)) % L.shape[0]
            res = f.solve_pairs(src, dst, want_volt=True, want_branch=True, raise_on_residual=prec != "single")
            assert res["branch"].shape == (nb, k)
            for c in range(k):
                _, _, want = core_mod._branch_currents(L, np.asarray(res["volt"][:, c], dtype=np.float64), comp)
                got = np.asarray(res["branch"][:, c], dtype=np.float64)
                assert np.abs(got - want).max() <= tol * want.max(), (k, c)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp64", "mixed"])
def test_branch_cut_at_one_e_minus_8_of_the_maximum(prec):
    """1 A from node 0 to node 3 over the edge (0, 3) and two side routes of two edges each; the routes' series
    conductances are 2^-27 and 2^-26 of the direct edge's, so their branch currents sit at 7.5e-9 (cut) and
    1.5e-8 (kept) of the maximum."""
    e = [(0, 3, 1.0), (0, 1, 2.0 ** -26), (1, 3, 2.0 ** -26), (0, 2, 2.0 ** -25), (2, 3, 2.0 ** -25)]
    i, j, w = (np.array(x) for x in zip(*e))
    L = graph.laplacian(sp.coo_matrix((np.r_[w, w], (np.r_[i, j], np.r_[j, i])), shape=(4, 4)).tocsr())
    with cb.B200Factor(L, _solver(prec, "off")) as f:
        res = f.solve_pairs([3], [0], want_volt=True, want_branch=True)
        lo, hi = f.branch_index()
        got = dict(zip(zip(lo.tolist(), hi.tolist()), np.asarray(res["branch"][:, 0], dtype=np.float64)))
        _, _, want = core_mod._branch_currents(L, np.asarray(res["volt"][:, 0], dtype=np.float64), np.arange(1, 5))
    assert got[(0, 1)] == 0 and got[(1, 3)] == 0
    assert got[(0, 2)] > 0 and got[(2, 3)] > 0 and got[(0, 3)] > 0
    assert np.allclose([got[k] for k in zip(lo.tolist(), hi.tolist())], want, rtol=1e-12, atol=0)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp64", "single"])
def test_cumulative_branch_vector(prec):
    L = graph.power_law_laplacian(4000, m=3, seed=6)
    rng = np.random.default_rng(2)
    k = 11
    src = rng.choice(L.shape[0], k, replace=False)
    dst = (src + 7) % L.shape[0]
    w = rng.integers(1, 5, k).astype(np.float64)
    w[3] = 0.0
    with cb.B200Factor(L, _solver(prec, "off")) as f:
        f.reset_currents()
        res = f.solve_pairs(src, dst, w, accumulate=True, want_branch=True, raise_on_residual=prec != "single")
        cum = f.read_branch_currents()
        B = np.asarray(res["branch"], dtype=np.float64)
        want = B @ w
        assert np.abs(cum - want).max() <= (1e-6 if prec == "single" else 1e-12) * want.max()
        f.reset_currents()
        assert not f.read_branch_currents().any()
        again = f.solve_pairs(src, dst, w, accumulate=True, want_branch=True, raise_on_residual=prec != "single")
        assert np.array_equal(again["branch"], res["branch"]) and np.array_equal(f.read_branch_currents(), cum)
        f.solve_pairs(src, dst, w, accumulate=True, want_branch=True, raise_on_residual=prec != "single")
        assert np.abs(f.read_branch_currents() - 2 * cum).max() <= (1e-6 if prec == "single" else 1e-15) * cum.max()


@pytest.mark.gpu
def test_solve_pairs_is_unchanged_by_a_branch_call():
    L = graph.power_law_laplacian(5000, m=4, seed=8)
    rng = np.random.default_rng(4)
    src = rng.choice(L.shape[0], 9, replace=False)
    dst = (src + 13) % L.shape[0]
    w = rng.integers(1, 4, 9).astype(np.float64)
    with cb.B200Factor(L, cb.CUDASolver()) as f:
        def plain():
            f.reset_currents()
            r = f.solve_pairs(src, dst, w, want_volt=True, want_curr=True, accumulate=True)
            return (r["R"], r["volt"], r["curr"], *f.read_currents())
        before = plain()
        f.solve_pairs(src, dst, w, want_volt=True, want_curr=True, accumulate=True, want_branch=True)
        f.solve_pairs(src[:3], dst[:3], want_branch=True)          # the k_cur_max-only branch pass
        after = plain()
    for a, b in zip(before, after):
        assert np.array_equal(a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(1, 4))
def test_device_branch_pairwise_goldens_on_the_device(golden, i):
    prob, flags, exp = cases.network_pairwise_problem(golden, f"sgNetworkVerify{i}",
                                                      cb.CUDASolver(branch_on_device=True, rtol=1e-12))
    r = cb.single_ground_all_pairs(prob, flags)
    cases.check_network_pairwise(r, exp)
    _check_cum_branch(prob, r, exp)
    host, _, _ = cases.network_pairwise_problem(golden, f"sgNetworkVerify{i}", cb.CUDASolver(rtol=1e-12))
    h = cb.single_ground_all_pairs(host, flags)
    assert np.abs(r.cum_branch - h.cum_branch).max() <= 1e-10 * max(1.0, np.abs(h.cum_branch).max())


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(1, 4))
def test_network_advanced_goldens_on_the_device(golden, i):
    prob, flags, exp = cases.advanced_problem(golden, f"mgNetworkVerify{i}", cb.CUDASolver(rtol=1e-12))
    r = cb.network_advanced(prob, flags)
    cases.check_advanced(r, exp, flags)


def _disjoint(sizes, seed):
    """Laplacian of disjoint random components of the given sizes (0 = an isolated node) and their 1-based
    node lists; network_graph's component order."""
    blocks = [_random_laplacian(m, seed + c) if m > 1 else sp.csr_matrix((1, 1)) for c, m in enumerate(sizes)]
    G = sp.block_diag(blocks, format="csr")
    G.eliminate_zeros()
    G.sort_indices()
    return G, co.connected_components(G)


# the device stops each column at rtol or at the absolute sqrt(eps) of the reference's Krylov defaults, so its
# voltages agree with the oracle's direct solves to about 1e-8 of each column's scale
DEVICE_REL = 1e-7


def _run_advanced(G, cc, s, g, f):
    want = co.advanced_kernel(G, cc, s, g, f)
    got = cb.network_advanced(cb.AdvancedProblem(G, cc, s, g, f, solver=cb.CUDASolver(rtol=1e-12)),
                              cb.Flags(is_raster=False, is_advanced=True))
    return got, want


@pytest.mark.gpu
def test_network_advanced_global_cut():
    """Two components whose sources differ by 1e9: the reference takes one maximum over the whole graph, so the
    quiet component's branch currents are cut to 0 and its node currents keep only the ground currents."""
    G, cc = _disjoint([400, 300], 21)
    n = G.shape[0]
    s, g = np.zeros(n), np.zeros(n)
    s[5], s[420] = 1e9, 1.0
    g[100], g[500] = 2.0, np.inf
    g[101] = 0.5
    f = np.where(np.isfinite(g), g, 0.0)
    got, want = _run_advanced(G, cc, s, g, f)
    _advanced_agree(got, want, rel=DEVICE_REL)
    quiet = np.isin(got.branch[0], cc[1])
    assert quiet.sum() > 0 and not got.branch[2][quiet].any() and not np.asarray(want.branch[2])[quiet].any()
    q = np.asarray(cc[1]) - 1
    assert np.abs(got.voltages[q] - want.voltages[q]).max() <= DEVICE_REL * np.abs(want.voltages[q]).max()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["finite", "inf", "mixed"])
def test_network_advanced_many_components(kind):
    """More components than one panel holds, an isolated node with a finite ground and a source, components
    that are skipped."""
    sizes = [60 + 10 * c for c in range(19)] + [1] + [50]
    G, cc = _disjoint(sizes, 40)
    n = G.shape[0]
    rng = np.random.default_rng(5)
    s, g = np.zeros(n), np.zeros(n)
    for c, nodes in enumerate(cc):
        rows = np.asarray(nodes) - 1
        if len(rows) == 1:
            s[rows] = 2.0
            g[rows] = 0.25 if kind != "inf" else 0.0
            continue
        if c == len(cc) - 1:
            s[rows[0]] = 1.0                                 # no ground: skipped
            continue
        src = rng.choice(rows, 3, replace=False)
        s[src] = rng.uniform(0.5, 2.0, 3)
        gnd = rng.choice(np.setdiff1d(rows, src), 2, replace=False)
        g[gnd] = np.inf if kind == "inf" else rng.uniform(0.5, 2.0, 2)
        if kind == "mixed" and c % 2:
            g[gnd[0]] = np.inf
    s_, g_, f_ = cb.resolve_conflicts(s, g, "keepall")
    got, want = _run_advanced(G, cc, s_, g_, f_)
    _advanced_agree(got, want, rel=DEVICE_REL)
    assert got.stats["columns"] > 8
    iso = [c for c in cc if len(c) == 1][0][0] - 1
    if kind != "inf":
        assert abs(got.voltages[iso] - 8.0) <= DEVICE_REL * 8.0


@pytest.mark.gpu
def test_network_advanced_nothing_solved():
    G, cc = _disjoint([50, 40], 3)
    n = G.shape[0]
    got, want = _run_advanced(G, cc, np.zeros(n), np.zeros(n), np.array([-9999.0]))
    _advanced_agree(got, want)
    assert not got.voltages.any() and not got.node_currents.any() and not got.branch[2].any()


@pytest.mark.gpu
def test_solve_advanced_network_rejects_bad_owners():
    G, cc = _disjoint([30, 20], 7)
    n = G.shape[0]
    a, b = np.asarray(cc[0]) - 1, np.asarray(cc[1]) - 1
    owner = np.full(n, -1, dtype=np.int64)
    owner[a], owner[b] = 0, 1
    sets = [a[:1], b[:1]]
    sources = [(a[1:2], [1.0]), (b[1:2], [1.0])]
    with cb.B200Factor(G, cb.CUDASolver()) as f:
        def rejects(sets, gset, sources, owner, text):
            with pytest.raises(cb.B200Error, match=text) as e:
                f.solve_advanced_network(sets, gset, sources, owner, want_volt=True)
            assert e.value.code == _lib.ERR_ARG
        rejects(sets, [0, 1], sources, np.where(owner == 1, 2, owner), "not a column")
        rejects(sets, [0, 1], sources, np.where(owner == 1, -2, owner), "not a column")
        rejects(sets, [0, 1], [sources[0], (a[2:3], [1.0])], owner, "source row")
        rejects([a[:1], a[3:4]], [0, 1], sources, owner, "ground row")
        rejects(sets, [0, -1], sources, owner, "no direct grounds")
        ok = f.solve_advanced_network(sets, [0, 1], sources, owner, want_volt=True, want_curr=True, want_branch=True)
        assert np.all(ok["volt"][owner == -1] == 0) and ok["volt"][a[1]] > 0 and ok["volt"][b[1]] > 0

"""k_advanced_batch (csrc/advanced_batch.cu) stage by stage against tests/reference_ops.py
`advanced_window`, a float64 restatement of one moving window: component labels and the skip rule
(through what they decide), the Jacobi-PCG iterates and stop iterations, the reported residual and
status, the node currents with the 1e-8 cut, and shapes, types and batches.

The kernel is a second, self-contained solver: none of the handle-based kernels, and none of their
checks, are behind it.  CG hides mistakes in its recurrence (they cost iterations, not accuracy) and a
branch at 1e-8 of a maximum is invisible at the 1e-7 tolerance of tests/test_advanced_batch.py, so the
comparisons here are per stage and every bound comes from the reference, never from the device.

CPU: `advanced_window` reproduces the per-window specification (test_advanced_batch.reference).
GPU (`pytest -m gpu`): everything else, through solver.solve_advanced_batch."""
import re

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from circuitscape_b200 import _lib
from circuitscape_b200 import solver as S

from .reference_ops import (ATOL, NODATA, WIN_MAXITER, WIN_OK, WIN_RESIDUAL, advanced_window, node_currents, pcg,
                            true_relres, window_graph)
from .test_advanced_batch import _cfg, parity_windows, reference, split

ITMAX = 50_000
EPS = np.finfo(np.float64).eps
WORST = {}             # group -> largest measured / bound, and counts of what was excluded


def note(group, measured, bound):
    """measured <= bound, and remember the largest ratio of the group for the report"""
    measured, bound = np.asarray(measured, dtype=np.float64), np.asarray(bound, dtype=np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(measured > 0, measured / bound, 0.0)
    WORST[group] = max(WORST.get(group, 0.0), float(ratio.max(initial=0.0)))
    assert np.all(measured <= bound), (group, float(ratio.max()))


def count(key, k):
    WORST[key] = WORST.get(key, 0) + int(k)


@pytest.fixture(scope="module", autouse=True)
def report(request):
    yield
    tr = request.config.pluginmanager.get_plugin("terminalreporter")
    cap = request.config.pluginmanager.get_plugin("capturemanager")
    if tr is not None and cap is not None and WORST:
        with cap.global_and_fixture_disabled():
            tr.write_line("")
            tr.write_line("test_advanced_batch_kernel: largest measured / bound, and counts: " +
                          ", ".join(f"{k} = {v:.3g}" for k, v in sorted(WORST.items())))


def run(ws, four, rtol, itmax=ITMAX, want_volt=True, dtype=np.float64):
    g, s, n = (np.stack(a).astype(dtype) for a in split(ws))
    return S.solve_advanced_batch(g, s, n, four, 0, rtol, itmax, want_volt=want_volt)


def widen(w, dtype):
    """the values the kernel sees: the window rounded to `dtype`"""
    return tuple(np.asarray(a, dtype=np.float64).astype(dtype).astype(np.float64) for a in w)


def flat(a):
    return np.asarray(a).T.ravel()         # cell r + c nrows


def lognormal(rng, nr, nc, sigma=1.0):
    return np.exp(sigma * rng.normal(size=(nr, nc)))


def check_direct(group, w, ref, res, k=0, tol=1e-9):
    """The support of volt / cur is the union of the solved components, and every solved component
    agrees with a direct solve of its reduced system to `tol` of its max."""
    volt, cur = flat(res["volt"][k]), flat(res["cur"][k])
    assert np.array_equal(volt != 0, flat(ref["volt"]) != 0) and np.array_equal(cur != 0, flat(ref["cur"]) != 0)
    solved = np.isin(flat(ref["labels"]), ref["solved"])
    assert not volt[~solved].any() and not cur[~solved].any()
    for c in ref["comps"]:
        x = spla.spsolve(c["A_red"].tocsc(), c["b"]) if len(c["b"]) > 1 else c["b"] / c["A_red"].diagonal()
        assert np.any(x != 0)
        note(group, np.abs(volt[c["keep"]] - x).max(), tol * np.abs(x).max())
        gone = np.setdiff1d(c["cells"], c["keep"])
        assert not volt[gone].any()


def near_tie(c, rtol, itmax=ITMAX, rel=1e-9):
    """Is the reference's stop iteration sensitive to rounding?  sqrt(rho) at the stop or the iteration
    before lies within `rel` of tol, or within 10x the distance between two float64 restatements of the
    recurrence that differ in one rounding (z = r / d against z = r (1 / d)), or the two stop apart.
    After ~100 iterations on an 8-neighbour lognormal window that distance reaches 0.3 tol."""
    dinv = 1.0 / c["A_red"].diagonal()
    _, it, rho, _ = pcg(c["A_red"], c["b"], lambda R: R * dinv[:, None], rtol, itmax, stall_limit=0)
    if int(it[0]) != c["iters"]:
        return True
    mine, other = np.sqrt(c["rho"][-2:]), np.sqrt(rho[-2:, 0])
    return bool(np.any(np.abs(mine - c["tol"]) <= rel * c["tol"] + 10 * np.abs(mine - other).max()))


# ---------------------------------------------------------------------------
# windows
# ---------------------------------------------------------------------------
def corridor_ends(g, cells, strength=1e3):
    src, gnd = np.zeros_like(g), np.zeros_like(g)
    gnd[cells[0]] = np.inf
    src[cells[-1]] = strength
    return g, src, gnd


def square_spiral(n, seed=0):
    """one corridor wound into a square spiral, ground at the outer end, source at the centre"""
    rng = np.random.default_rng(seed)
    g = np.full((n, n), NODATA)
    r = c = 0
    path = [(0, 0)]
    lengths = [n - 1] * 3 + [k for k in range(n - 3, 0, -2) for _ in range(2)]
    for i, L in enumerate(lengths):
        dr, dc = [(0, 1), (1, 0), (0, -1), (-1, 0)][i % 4]
        for _ in range(L):
            r, c = r + dr, c + dc
            path.append((r, c))
    for p in path:
        g[p] = rng.uniform(0.5, 2.0)
    return corridor_ends(g, path)


def serpentine(n, seed=1):
    """every other column, joined alternately at the bottom and at the top"""
    rng = np.random.default_rng(seed)
    g = np.full((n, n), NODATA)
    g[:, 0::2] = rng.uniform(0.5, 2.0, size=g[:, 0::2].shape)
    for c in range(1, n, 2):
        g[n - 1 if (c // 2) % 2 == 0 else 0, c] = 1.0
    last = n - 1 if n % 2 else n - 2
    end = (n - 1, last) if (last // 2) % 2 == 0 else (0, last)
    return corridor_ends(g, [(0, 0), end])


def comb(n, seed=2):
    """a spine along row 0 with a full-height tooth on every other column, a source at every tooth's tip"""
    rng = np.random.default_rng(seed)
    g = np.full((n, n), NODATA)
    g[0, :] = rng.uniform(0.5, 2.0, n)
    g[:, 0::2] = rng.uniform(0.5, 2.0, size=g[:, 0::2].shape)
    src, gnd = np.zeros_like(g), np.zeros_like(g)
    src[n - 1, 0::2] = 100.0
    gnd[0, n - 1 if n % 2 == 0 else n - 2] = np.inf
    src[gnd != 0] = 0.0
    return g, src, gnd


def block_checkerboard(n, seed=3, b=4):
    """b x b blocks on the black squares of a checkerboard: separate components 4-connected, joined at
    their corners 8-connected.  A scattered third have a source and a ground (Inf or finite), the rest
    a source only, a ground only or neither."""
    rng = np.random.default_rng(seed)
    g = np.full((n, n), NODATA)
    src, gnd = np.zeros_like(g), np.zeros_like(g)
    nb = n // b
    for I in range(nb):
        for J in range(nb):
            if (I + J) % 2:
                continue
            r0, c0 = I * b, J * b
            g[r0:r0 + b, c0:c0 + b] = np.exp(rng.normal(size=(b, b)))
            kind = rng.integers(0, 6)                     # 0, 1: both; 2, 3: source; 4: ground; 5: neither
            if kind in (0, 1, 2, 3):
                src[r0 + rng.integers(0, b), c0 + rng.integers(0, 2)] = rng.uniform(50.0, 150.0)
            if kind in (0, 1, 4):
                gnd[r0 + rng.integers(0, b), c0 + 2 + rng.integers(0, 2)] = np.inf if kind == 0 else rng.uniform(0.5, 2)
    return g, src, gnd


def skip_edges():
    """name -> (window, number of components, number solved)"""
    rng = np.random.default_rng(11)
    base = lognormal(rng, 7, 6)
    z = np.zeros_like(base)
    out = {}

    def put(**kw):
        a = {"src": z.copy(), "gnd": z.copy(), "g": base.copy()}
        for name, cells in kw.items():
            for rc, v in cells.items():
                a[name][rc] = v
        return a["g"], 1e3 * a["src"], a["gnd"]         # strong sources: the absolute tolerance is far below

    out["sources_cancel"] = (put(src={(1, 1): 1.0, (5, 4): -1.0}, gnd={(3, 3): np.inf}), 1, 0)
    out["sources_almost_cancel"] = (put(src={(1, 1): 1.0, (5, 4): -0.5}, gnd={(3, 3): np.inf}), 1, 1)
    out["finite_ground_only"] = (put(gnd={(3, 3): 0.7}), 1, 0)
    out["source_on_inf_ground"] = (put(src={(3, 3): 2.0}, gnd={(3, 3): np.inf}), 1, 0)
    out["source_on_finite_ground_and_another"] = (put(src={(3, 3): 2.0, (0, 5): 1.0}, gnd={(3, 3): 0.4}), 1, 1)
    out["source_on_nodata"] = (put(g={(2, 2): NODATA}, src={(2, 2): 1.0}, gnd={(3, 3): np.inf}), 1, 0)
    # the finite ground of the component's first cell is the sentinel: the component's finite grounds
    # (the 0.9 too) stay out of the operator and of the currents
    out["sentinel_first_ground"] = (put(src={(4, 4): 1.0}, gnd={(0, 0): NODATA, (6, 5): np.inf, (2, 3): 0.9}), 1, 1)
    g = np.full_like(base, NODATA)
    g[6, 2] = g[0, 3] = 1.0                        # cells nr - 1 + 2 nr and 3 nr: adjacent in memory only
    out["no_wrap_between_columns"] = ((g, *put(src={(6, 2): 1.0}, gnd={(0, 3): np.inf})[1:]), 2, 0)
    return out


# ---------------------------------------------------------------------------
# CPU: the float64 restatement against the per-window specification
# ---------------------------------------------------------------------------
ANCHOR = parity_windows() + [w for w, _, _ in skip_edges().values()]


@pytest.mark.parametrize("four", [False, True])
@pytest.mark.parametrize("k", range(len(ANCHOR)))
def test_reference_reproduces_the_per_window_specification(k, four):
    """advanced_window solved to rtol 1e-12 (no absolute tolerance) equals compute_omniscape_current on a
    direct solver: the -9999 first-cell rule, a source on a grounded cell and the skip rule included."""
    w = ANCHOR[k]
    ref = advanced_window(*w, four, 1e-12, ITMAX, atol=0.0)
    cur, volt = reference(*w, _cfg(four))
    for mine, spec in ((ref["cur"], cur), (ref["volt"], volt)):
        assert np.array_equal(mine == 0, spec == 0)
        assert np.abs(mine - spec).max() <= 1e-10 * np.abs(spec).max()
    assert ref["status"] == WIN_OK and all(c["iters"] > 0 for c in ref["comps"])


def test_reference_skip_edges_have_their_property():
    for name, (w, ncomp, nsolved) in skip_edges().items():
        for four in (False, True):
            ref = advanced_window(*w, four, 1e-10, ITMAX)
            assert len(np.unique(ref["labels"][ref["labels"] >= 0])) == ncomp, name
            assert len(ref["solved"]) == nsolved, name
    # the sentinel keeps every finite ground of its component out of the operator: the reduced system is
    # the Laplacian with the Inf-ground row deleted
    w = skip_edges()["sentinel_first_ground"][0]
    c = advanced_window(*w, False, 1e-10, ITMAX)["comps"][0]
    sel = flat(w[2])[c["cells"]] != np.inf
    assert c["fin"] is None and abs(c["A_red"] - c["a_local"][sel][:, sel]).max() == 0
    c = advanced_window(*skip_edges()["source_on_finite_ground_and_another"][0], False, 1e-10, ITMAX)["comps"][0]
    assert abs((c["A_red"] - c["a_local"]).diagonal().sum() - 0.4) < 1e-12 and c["b"].sum() == 1e3


def test_reference_labels_are_the_smallest_cell_of_each_component():
    g, src, gnd = block_checkerboard(41)
    for four, many in ((True, True), (False, False)):
        lab = advanced_window(g, src, gnd, four, 1e-6, 5)["labels"]
        roots = np.unique(lab[lab >= 0])
        assert (len(roots) >= 40) == many
        for r in roots:
            cells = np.flatnonzero(flat(lab) == r)
            assert cells.min() == r and np.all(flat(g)[cells] > 0)
        assert np.array_equal(lab >= 0, g > 0)


def test_reference_weak_source_and_itmax_zero_fail_the_gate_without_iterating():
    """sqrt(rho0) <= tol at the start (the absolute tolerance decides) and itmax = 0 both leave x = 0,
    whose true relative residual is 1: the per-window path (src/core.jl:639-641) raises there too."""
    rng = np.random.default_rng(5)
    g = lognormal(rng, 6, 5)
    src, gnd = np.zeros_like(g), np.zeros_like(g)
    src[4, 3], gnd[0, 0] = 1e-9, np.inf
    for s, itmax in ((src, ITMAX), (src * 1e9, 0)):
        ref = advanced_window(g, s, gnd, False, 1e-6, itmax)
        assert ref["iters"] == 0 and ref["relres"] == 1.0 and ref["status"] == WIN_RESIDUAL
        assert not ref["volt"].any() and not ref["cur"].any() and ref["solved"] == [0]


# ---------------------------------------------------------------------------
# GPU (a): labels and the skip rule, through what they decide
# ---------------------------------------------------------------------------
def longest_path(w, four):
    W, _ = window_graph(w[0], four)
    start = int(np.flatnonzero(np.isinf(flat(w[2])))[0])
    d = sp.csgraph.shortest_path(W, unweighted=True, indices=start)
    return int(d[np.isfinite(d)].max())


HARD = {
    "spiral101": (lambda: square_spiral(101), True, dict(path=5000)),
    "spiral151_8": (lambda: square_spiral(151), False, dict(path=5000)),
    "serpentine101": (lambda: serpentine(101), True, dict(path=5000)),
    "serpentine151": (lambda: serpentine(151), True, dict(path=11000)),
    "comb101_8": (lambda: comb(101), False, dict(path=190, comps=1)),
    "comb151": (lambda: comb(151), True, dict(path=290, comps=1)),
    "blocks101_4": (lambda: block_checkerboard(101), True, dict(comps=300, solved=80)),
    "blocks151_4": (lambda: block_checkerboard(151), True, dict(comps=650, solved=180)),
    "blocks101_8": (lambda: block_checkerboard(101), False, dict(comps=1, solved=1)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(HARD))
def test_hard_shapes_label_and_solve_as_the_reference(name):
    make, four, prop = HARD[name]
    w = make()
    ref = advanced_window(*w, four, 1e-12, ITMAX)
    ncomp = len(np.unique(ref["labels"][ref["labels"] >= 0]))
    if "path" in prop:
        assert longest_path(w, four) >= prop["path"]
    if prop.get("comps") == 1:
        assert ncomp == 1
    elif "comps" in prop:
        assert ncomp >= prop["comps"]
        both = sum(1 for r in np.unique(ref["labels"][ref["labels"] >= 0])
                   if (flat(w[1])[flat(ref["labels"]) == r] != 0).any() and (flat(w[2])[flat(ref["labels"]) == r] != 0).any())
        assert ncomp // 4 <= len(ref["solved"]) == both <= ncomp // 2     # a third, scattered
        assert np.any(np.diff(np.isin(np.unique(ref["labels"][ref["labels"] >= 0]), ref["solved"]).astype(int)) != 0)
    assert len(ref["solved"]) >= prop.get("solved", 1) and ref["status"] == WIN_OK
    res = run([w], four, 1e-12)
    assert res["rc"] == _lib.OK and res["first_failed"] == -1
    longest = max(len(c["b"]) for c in ref["comps"])
    check_direct("a_direct", w, ref, res)
    ties = sum(near_tie(c, 1e-12) for c in ref["comps"])
    count("a_near_ties", ties)
    if longest < 3000 and not ties:
        assert res["iters"][0] == ref["iters"]
    else:            # thousands of iterations: rounding moves the stop by a few
        assert abs(int(res["iters"][0]) - ref["iters"]) <= 0.02 * ref["iters"]
    note("a_relres", res["relres"][0], 10 * ref["relres"])


@pytest.mark.gpu
@pytest.mark.parametrize("four", [False, True])
def test_skip_rule_edges(four):
    edges = skip_edges()
    ws = [w for w, _, _ in edges.values()]
    res = run(ws, four, 1e-12)
    assert res["rc"] == _lib.OK
    for k, (name, (w, _, nsolved)) in enumerate(edges.items()):
        ref = advanced_window(*w, four, 1e-12, ITMAX)
        assert len(ref["solved"]) == nsolved
        check_direct("a_direct", w, ref, res, k)
        assert res["iters"][k] == ref["iters"] and (nsolved or res["iters"][k] == 0), name
        cur, volt = reference(*w, _cfg(four))
        for dev, spec in ((res["cur"][k], cur), (res["volt"][k], volt)):
            assert np.array_equal(dev != 0, spec != 0), name
            note("a_spec", np.abs(dev - spec).max(), 1e-8 * np.abs(spec).max() if nsolved else 0.0)


# ---------------------------------------------------------------------------
# GPU (b): the recurrence
# ---------------------------------------------------------------------------
def recurrence_windows(nr=26, nc=22):
    """single-component windows: full and holey lognormal x Inf ground, finite grounds, both"""
    ws = []
    for seed, holes in ((0, 0.0), (1, 0.0), (2, 0.06), (3, 0.06)):
        for grounds in ("inf", "finite", "both"):
            rng = np.random.default_rng(100 * seed + len(grounds))
            g = lognormal(rng, nr, nc, 1.0 + 0.5 * seed)
            g[rng.random(g.shape) < holes] = NODATA
            src = np.where((g > 0) & (rng.random(g.shape) < 0.15), rng.uniform(0.5, 2.0, g.shape), 0.0)
            gnd = np.zeros_like(g)
            if grounds != "finite":
                gnd[nr // 2, nc // 2] = np.inf
            if grounds != "inf":
                sel = (rng.random(g.shape) < 0.03) & (src == 0)
                gnd[sel] = rng.uniform(0.05, 0.5, int(sel.sum()))
            g[gnd != 0] = np.abs(g[gnd != 0])
            ws.append((g, src, gnd))
    return ws


def one_component(ref, least=400):
    assert len(ref["comps"]) == 1 and len(ref["comps"][0]["b"]) > least
    return ref["comps"][0]


@pytest.mark.gpu
@pytest.mark.parametrize("four", [False, True])
@pytest.mark.parametrize("m", [1, 2, 3, 5, 8])
def test_mth_iterate(m, four):
    ws = recurrence_windows()
    res = run(ws, four, 1e-14, itmax=m)
    for k, w in enumerate(ws):
        ref = advanced_window(*w, four, 1e-14, m, iterates=True)
        c = one_component(ref)
        assert c["iters"] == m == len(c["x_hist"]) and np.array_equal(c["x_hist"][-1], c["x"])
        assert res["iters"][k] == m
        note("b_iterate", np.abs(res["volt"][k] - ref["volt"]).max(), 1e-12 * np.abs(ref["volt"]).max())
        note("b_relres", abs(res["relres"][k] - ref["relres"]), 1e-10 * ref["relres"])
        assert ref["relres"] > 1e-4 and ref["status"] == WIN_RESIDUAL
    assert res["rc"] == _lib.ERR_RESIDUAL and res["first_failed"] == 0


@pytest.mark.gpu
def test_stop_iterations():
    """The stop iteration equals the reference's wherever that is not sensitive to rounding: windows of
    572 cells (100 - 300 iterations) and of 90 cells (tens of iterations, before CG loses orthogonality)."""
    ties, checked = {False: 0, True: 0}, {False: 0, True: 0}
    for ws, most in ((recurrence_windows(), 2000), (recurrence_windows(10, 9), 100)):
        for four in (False, True):
            for rtol in (1e-6, 1e-10):
                res = run(ws, four, rtol)
                assert res["rc"] == _lib.OK
                for k, w in enumerate(ws):
                    c = one_component(advanced_window(*w, four, rtol, ITMAX), 60)
                    assert 10 < c["iters"] < most
                    if near_tie(c, rtol):
                        ties[four] += 1
                        continue
                    checked[four] += 1
                    assert res["iters"][k] == c["iters"], (four, rtol, k)
    count("b_stop_checked", sum(checked.values()))
    count("b_stop_rounding_sensitive", sum(ties.values()))
    assert ties[True] <= 4 and checked[False] >= 24, (ties, checked)


@pytest.mark.gpu
@pytest.mark.parametrize("four", [False, True])
def test_itmax_zero_and_a_source_below_the_absolute_tolerance(four):
    ws = recurrence_windows()[:3]
    res = run(ws, four, 1e-6, itmax=0)
    assert res["rc"] == _lib.ERR_RESIDUAL and res["first_failed"] == 0
    assert not res["volt"].any() and not res["cur"].any() and not res["iters"].any()
    assert np.all(res["relres"] == 1.0)
    # sqrt(rho0) <= tol from the start: no iteration, x = 0, relative residual 1 -- as the reference
    weak = []
    for g, src, gnd in ws:
        s = np.zeros_like(src)
        s[np.nonzero(src)[0][0], np.nonzero(src)[1][0]] = 1e-9
        weak.append((g, s, gnd))
    mixed = [weak[0], ws[1], weak[2]]
    res = run(mixed, four, 1e-6)
    for k, w in enumerate(mixed):
        ref = advanced_window(*w, four, 1e-6, ITMAX)
        if k != 1:
            c = ref["comps"][0]
            assert np.sqrt(c["rho"][0]) <= ATOL and ref["iters"] == 0 and ref["status"] == WIN_RESIDUAL
            assert not res["volt"][k].any() and not res["cur"][k].any()
            assert res["iters"][k] == 0 and res["relres"][k] == ref["relres"] == 1.0
        else:               # the ordinary window between them is untouched by its neighbours' early exit
            assert ref["status"] == WIN_OK and 0 < res["relres"][k] < 1e-4 and res["volt"][k].any()
            assert abs(int(res["iters"][k]) - ref["iters"]) <= 2
    assert res["rc"] == _lib.ERR_RESIDUAL and res["first_failed"] == 0 and "(0 iterations)" in res["msg"]


@pytest.mark.gpu
@pytest.mark.parametrize("four", [False, True])
def test_power_of_two_scalings_are_exact(four):
    """After m iterations (no stop before: asserted on the reference) a source scaled by 2^k scales the
    voltages and currents exactly; conductances and grounds scaled by 2^k scale the voltages by 2^-k
    exactly and leave the currents bit-identical."""
    ws = recurrence_windows()[:6]
    m = 6
    base = run(ws, four, 1e-14, itmax=m)
    for k in (20, -20):
        f = 2.0 ** k
        scaled = [(g, s * f, n) for g, s, n in ws]
        assert all(advanced_window(*w, four, 1e-14, m)["iters"] == m for w in scaled)
        res = run(scaled, four, 1e-14, itmax=m)
        assert np.array_equal(res["volt"], base["volt"] * f) and np.array_equal(res["cur"], base["cur"] * f)
        assert np.array_equal(res["relres"], base["relres"])
    for k in (10, -10):
        f = 2.0 ** k
        scaled = [(np.where(g > 0, g * f, g), s, n * f) for g, s, n in ws]
        assert all(advanced_window(*w, four, 1e-14, m)["iters"] == m for w in scaled)
        res = run(scaled, four, 1e-14, itmax=m)
        assert np.array_equal(res["volt"], base["volt"] / f) and np.array_equal(res["cur"], base["cur"])


# ---------------------------------------------------------------------------
# GPU (c): gate and status
# ---------------------------------------------------------------------------
def regions(seed, nr=20, ncols=(9, 7, 11)):
    """side-by-side regions behind NODATA walls, each with its own sources and an Inf ground"""
    rng = np.random.default_rng(seed)
    nc = sum(ncols) + len(ncols) - 1
    g = lognormal(rng, nr, nc, 1.5)
    src, gnd = np.zeros_like(g), np.zeros_like(g)
    c0 = 0
    for k, w in enumerate(ncols):
        blk = (slice(None), slice(c0, c0 + w))
        s = np.where(rng.random((nr, w)) < 0.1, rng.uniform(500.0, 2000.0, (nr, w)), 0.0)
        s[0, 0] = 1000.0
        src[blk] = s
        gnd[nr - 1, c0 + w - 1] = np.inf
        src[nr - 1, c0 + w - 1] = 0.0
        if k < len(ncols) - 1:
            g[:, c0 + w] = NODATA
        c0 += w + 1
    src[g <= 0] = 0.0
    return g, src, gnd


def relres_of(ref, volt):
    return [float(true_relres(c["A_red"], flat(volt)[c["keep"]], c["b"])[0]) for c in ref["comps"]]


@pytest.mark.gpu
@pytest.mark.parametrize("four", [False, True])
@pytest.mark.parametrize("itmax", [2, 5, 20])
def test_reported_residual_is_the_true_residual_of_the_returned_voltages(itmax, four):
    ws = [regions(1, ncols=(9, 12)), regions(2, ncols=(12, 9)), regions(3), regions(4, ncols=(11, 9, 7)),
          regions(5, ncols=(7, 11, 9))]
    ws = [tuple(a[:, :29] if a.shape[1] > 29 else np.pad(a, ((0, 0), (0, 29 - a.shape[1]))) for a in w) for w in ws]
    res = run(ws, four, 1e-13, itmax=itmax)
    not_last = 0
    for k, w in enumerate(ws):
        ref = advanced_window(*w, four, 1e-13, itmax)
        assert len(ref["comps"]) == (2 if k < 2 else 3) and ref["iters"] == itmax * len(ref["comps"])
        mine = relres_of(ref, res["volt"][k])
        assert min(c["relres"] for c in ref["comps"]) > 1e-6
        assert max(mine) > 1.005 * sorted(mine)[-2]                  # the max is not a tie
        not_last += int(np.argmax(mine)) < len(mine) - 1
        note("c_relres", abs(res["relres"][k] - max(mine)), 1e-10 * max(mine))
        note("c_relres_ref", abs(res["relres"][k] - ref["relres"]), 1e-9 * ref["relres"])
        assert res["iters"][k] == ref["iters"]
    assert 0 < not_last < len(ws)                   # the largest is the last component's in some windows only
    assert res["rc"] == _lib.ERR_RESIDUAL and res["first_failed"] == 0


def status_batch():
    """converged | itmax reached with a residual under the gate | no node | second component fails the
    gate while the first converges | converged; all at rtol 1e-13, itmax 14"""
    shape = (20, 21)

    def tiny(seed):
        rng = np.random.default_rng(seed)
        g = np.full(shape, NODATA)
        g[:2, :3] = lognormal(rng, 2, 3)
        src, gnd = np.zeros(shape), np.zeros(shape)
        src[0, 0], gnd[1, 2] = 1.0, np.inf
        return g, src, gnd

    rng = np.random.default_rng(7)           # strong finite grounds everywhere: converges geometrically
    src = np.where(rng.random(shape) < 0.1, 1e3, 0.0)
    well = (lognormal(rng, *shape, 0.1), src, np.where(src == 0, 4.0, 0.0))
    nothing = (np.full(shape, NODATA), np.ones(shape), np.zeros(shape))
    second = regions(8, ncols=(1, 19))
    second = tuple(a.copy() for a in second)
    second[0][:, 0], second[1][:, 0], second[2][:, 0] = NODATA, 0.0, 0.0
    second[0][:3, 0], second[1][0, 0], second[2][2, 0] = 1.0, 1.0, np.inf       # a 3-cell first component
    return [tiny(1), well, nothing, second, tiny(2)], 1e-13, 14


def message_numbers(msg):
    return [float(x) for x in re.findall(r"[-+]?\d+\.?\d*(?:[eE][-+]?\d+)?", msg)]


@pytest.mark.gpu
@pytest.mark.parametrize("four", [False, True])
def test_status_precedence_first_failed_and_message(four):
    ws, rtol, itmax = status_batch()
    refs = [advanced_window(*w, four, rtol, itmax) for w in ws]
    assert [r["status"] for r in refs] == [WIN_OK, WIN_MAXITER, WIN_OK, WIN_RESIDUAL, WIN_OK]
    assert refs[1]["relres"] < 1e-4 and refs[1]["iters"] == itmax and not refs[2]["solved"]
    assert [c["status"] for c in refs[3]["comps"]] == [WIN_OK, WIN_RESIDUAL] and refs[3]["comps"][0]["iters"] < itmax
    alone = [run([w], four, rtol, itmax=itmax) for w in ws]

    def same_as_alone(res, keep):
        for j, k in enumerate(keep):
            for key in ("cur", "volt", "iters", "relres"):
                assert np.array_equal(res[key][j], alone[k][key][0]), (key, k)
            assert res["iters"][j] == refs[k]["iters"]
            note("c_status_volt", np.abs(res["volt"][j] - refs[k]["volt"]).max(),
                 1e-11 * max(np.abs(refs[k]["volt"]).max(), 1e-300))

    res = run(ws, four, rtol, itmax=itmax)
    same_as_alone(res, range(5))
    assert res["rc"] == _lib.ERR_RESIDUAL and res["first_failed"] == 3
    _, relres, iters = refs[3]["fail"]
    nums = message_numbers(res["msg"])
    assert f"for window 3 ({iters} iterations)" in res["msg"] and iters == itmax
    assert abs(nums[0] - relres) <= 1e-5 * relres and relres > 1e-4
    assert abs(res["relres"][3] - relres) <= 1e-9 * relres

    keep = [0, 1, 2, 4]
    res = run([ws[k] for k in keep], four, rtol, itmax=itmax)
    same_as_alone(res, keep)
    assert res["rc"] == _lib.ERR_MAXITER and res["first_failed"] == 1
    assert f"reached itmax = {itmax} before rtol for window 1 " in res["msg"]
    assert abs(message_numbers(res["msg"])[-1] - refs[1]["relres"]) <= 1e-5 * refs[1]["relres"]
    assert [a["rc"] for a in alone] == [_lib.OK, _lib.ERR_MAXITER, _lib.OK, _lib.ERR_RESIDUAL, _lib.OK]


# ---------------------------------------------------------------------------
# GPU (d): node currents of the returned voltages
# ---------------------------------------------------------------------------
def pockets(seed=8, nr=64, nc=56):
    """lognormal sigma = 3 with two corner pockets behind two-cell walls of conductance 1e-7 and 1e-5;
    the pockets' only sources are weak, so their branch currents straddle the 1e-8 cut"""
    rng = np.random.default_rng(seed)
    g = lognormal(rng, nr, nc, 3.0)
    g[14:16, 0:16] = g[0:16, 14:16] = 1e-7
    g[48:50, 40:] = g[48:, 40:42] = 1e-5
    src = np.where(rng.random(g.shape) < 0.05, rng.uniform(0.5, 2.0, g.shape), 0.0)
    src[:16, :16] = src[48:, 40:] = 0.0
    src[3, 4], src[60, 50] = 2e-7, 3e-6
    gnd = np.zeros_like(g)
    gnd[30, 28], src[30, 28] = np.inf, 0.0
    return g, src, gnd


def dead_end(seed=9, nr=60, nc=50):
    """a one-cell corridor that leads nowhere: zero current in exact arithmetic, exactly zero after the cut"""
    rng = np.random.default_rng(seed)
    g = lognormal(rng, nr, nc, 1.0)
    g[24:31, 0:31] = NODATA
    g[27, 0:31] = 1.0
    g[27, 0] = NODATA
    g[26:29, 30] = NODATA
    g[27, 30] = 1.0
    src = np.where((g > 0) & (rng.random(g.shape) < 0.05), 1e3, 0.0)
    src[24:31, 0:32] = 0.0
    gnd = np.zeros_like(g)
    gnd[50, 40], src[50, 40] = np.inf, 0.0
    return g, src, gnd


def strong_and_weak(seed=10, nr=40, nc=41):
    """two solved components whose largest branch currents differ by >= 1e9"""
    rng = np.random.default_rng(seed)
    g = lognormal(rng, nr, nc, 1.0)
    g[:, 20] = NODATA
    src, gnd = np.zeros_like(g), np.zeros_like(g)
    src[5, 3], src[30, 15], gnd[20, 10] = 4e3, 2e3, np.inf
    src[7, 25], src[33, 38], gnd[18, 30] = 1e-6, 2e-6, np.inf
    return g, src, gnd


def in_and_out(seed=12, nc=160):
    """one row, an Inf ground in the middle: strong sources left of it (every current runs towards larger
    cells), weak ones right of it (towards smaller cells), 1e9 apart"""
    rng = np.random.default_rng(seed)
    g = lognormal(rng, 1, nc, 0.5)
    src, gnd = np.zeros_like(g), np.zeros_like(g)
    gnd[0, nc // 2] = np.inf
    src[0, :nc // 2:7] = 1e4
    src[0, nc // 2 + 3::7] = 1e-5
    return g, src, gnd


def negative_sources(seed=13, nr=30, nc=33):
    rng = np.random.default_rng(seed)
    g = lognormal(rng, nr, nc, 1.0)
    g[rng.random(g.shape) < 0.04] = NODATA
    src = np.where((g > 0) & (rng.random(g.shape) < 0.1), -rng.uniform(50.0, 200.0, g.shape), 0.0)
    gnd = np.where((g > 0) & (src == 0) & (rng.random(g.shape) < 0.05), rng.uniform(0.1, 1.0, g.shape), 0.0)
    return g, src, gnd


def branches(c, v):
    """(positive, negative) branch currents of a component, as the node currents see them"""
    coo = sp.triu(c["a_local"], k=1).tocoo()
    d = np.abs(coo.data) * (v[coo.row] - v[coo.col])
    return d, -d


def check_currents(w, ref, res, k=0):
    """device currents against node_currents of the device's own voltages, component by component"""
    volt, cur = flat(res["volt"][k]), flat(res["cur"][k])
    zeros = 0
    for c in ref["comps"]:
        v = volt[c["cells"]]
        dv = 4 * EPS * np.abs(v).max()
        want, mask = node_currents(c["a_local"], v, dv=dv, finitegrounds=c["fin"])
        arow = np.asarray(abs(c["a_local"]).sum(axis=1)).ravel() - np.abs(c["a_local"].diagonal())
        fin = 0.0 if c["fin"] is None else np.abs(c["fin"])
        note("d_currents", np.abs(cur[c["cells"]] - want)[~mask], (1e-12 * want + (arow + fin) * dv)[~mask])
        count("d_masked_nodes", mask.sum())
        zeros += int(((want == 0) & ~mask).sum())
    return zeros


@pytest.mark.gpu
@pytest.mark.parametrize("four", [False, True])
def test_node_currents_and_the_cut(four):
    rtol = 1e-12
    # pockets: branch currents over >= 10 decades, some on each side of the cut
    w = pockets()
    ref = advanced_window(*w, four, rtol, ITMAX)
    d, _ = branches(ref["comps"][0], flat(ref["volt"])[ref["comps"][0]["cells"]])
    ratio = np.abs(d) / np.abs(d).max()
    assert np.sum((ratio > 1e-10) & (ratio < 1e-8)) > 20 and np.sum((ratio >= 1e-8) & (ratio < 1e-6)) > 20
    check_currents(w, ref, run([w], four, rtol))

    w = dead_end()
    ref = advanced_window(*w, four, rtol, ITMAX)
    assert len(ref["solved"]) == 1 and not ref["cur"][27, 3:28].any()
    res = run([w], four, rtol)
    assert check_currents(w, ref, res) >= 25 and not res["cur"][0][27, 3:28].any() and res["volt"][0][27, 3:28].all()

    # a window-wide cut would zero the weak component
    w = strong_and_weak()
    ref = advanced_window(*w, four, rtol, ITMAX)
    big, small = (np.abs(branches(c, flat(ref["volt"])[c["cells"]])[0]).max() for c in ref["comps"])
    assert len(ref["comps"]) == 2 and big >= 1e9 * small and ref["comps"][1]["iters"] > 10
    res = run([w], four, rtol)
    check_currents(w, ref, res)
    weak = ref["comps"][1]["cells"]
    assert np.all(flat(ref["cur"])[weak] > 0)
    note("d_weak_component", np.abs(flat(res["cur"][0])[weak] - flat(ref["cur"])[weak]), 1e-6 * flat(ref["cur"])[weak].max())
    assert res["iters"][0] == ref["iters"] or any(near_tie(c, rtol) for c in ref["comps"])

    # inflow and outflow are cut against their own maxima
    w = in_and_out()
    ref = advanced_window(*w, four, rtol, ITMAX)
    c = ref["comps"][0]
    p, q = branches(c, flat(ref["volt"])[c["cells"]])
    between = (q > 1e-8 * q.max()) & (q < 1e-8 * p.max())
    assert len(ref["comps"]) == 1 and p.max() >= 1e8 * q.max() and between.sum() > 50
    res = run([w], four, rtol)
    check_currents(w, ref, res)
    right = ref["cur"][:, 81:-2]
    assert np.all(right > 0)
    # the weak side is solved to the absolute tolerance, 1.5e-8 against sources of 1e-5
    note("d_outflow_side", np.abs(res["cur"][0][:, 81:-2] - right), 1e-3 * right.max())

    # finite grounds under negative sources: the ground current joins the inflow
    w = negative_sources()
    ref = advanced_window(*w, four, rtol, ITMAX)
    big = max(ref["comps"], key=lambda c: len(c["b"]))
    fg = big["fin"] * flat(ref["volt"])[big["cells"]]
    assert np.sum(fg < 0) > 10 and not np.any(fg > 0)
    res = run([w], four, rtol)
    check_currents(w, ref, res)
    note("d_currents_ref", np.abs(res["cur"][0] - ref["cur"]).max(), 1e-8 * ref["cur"].max())

    # everything injected leaves through the only Inf ground (sources far above the absolute tolerance)
    for w in (strong_and_weak(), dead_end()):
        res = run([w], four, rtol)
        ref = advanced_window(*w, four, rtol, ITMAX)
        for c in ref["comps"][:1]:
            at = np.setdiff1d(c["cells"], c["keep"])
            assert len(at) == 1 and c["b"].sum() > 1e3
            note("d_ground_current", abs(flat(res["cur"][0])[at[0]] - c["b"].sum()), 1e-8 * c["b"].sum())


# ---------------------------------------------------------------------------
# GPU (e): shapes, types, batches
# ---------------------------------------------------------------------------
def shaped(nr, nc, seed, holes=0.0):
    rng = np.random.default_rng(seed)
    g = lognormal(rng, nr, nc, 1.0)
    g[rng.random(g.shape) < holes] = NODATA
    g[nr // 2, nc // 2] = 1.0
    src = np.where(g > 0, rng.uniform(100.0, 200.0, g.shape), 0.0)
    gnd = np.zeros_like(g)
    gnd[nr // 2, nc // 2] = np.inf
    if nr * nc > 1:
        gnd[-1, -1] = 0.3 if g[-1, -1] > 0 else 0.0
    return g, src, gnd


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
@pytest.mark.parametrize("shape", [(1, 1), (1, 257), (255, 1), (256, 1), (16, 16), (37, 211), (301, 301)])
def test_shapes_and_input_types(shape, dtype):
    if shape == (301, 301) and dtype == np.float32:
        pytest.skip("the largest window runs once, in float64")
    w = shaped(*shape, seed=shape[0] + shape[1], holes=0.03 if shape[0] == 301 else 0.0)
    seen = widen(w, dtype)
    for four in (False, True):
        ref = advanced_window(*seen, four, 1e-12, ITMAX)
        res = run([w], four, 1e-12, dtype=dtype)
        if shape == (1, 1):                   # its only cell is the ground: nothing to solve
            assert not ref["solved"] and res["rc"] == _lib.OK and not res["cur"].any() and res["iters"][0] == 0
            one = (np.ones((1, 1)), np.ones((1, 1)), np.zeros((1, 1)))
            assert not run([one], four, 1e-12, dtype=dtype)["cur"].any()
            continue
        assert res["rc"] == _lib.OK and len(ref["solved"]) >= 1
        check_direct("e_direct", seen, ref, res)
        check_currents(seen, ref, res)
        note("e_relres", res["relres"][0], 10 * ref["relres"])


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_a_window_does_not_see_its_batch(dtype):
    """720 windows (more CTAs than the device holds at once) of 6 distinct ones in shuffled order: every
    copy equals the window run alone bit for bit, whatever its neighbours are; want_volt=False returns
    the same currents."""
    distinct = recurrence_windows()[:4] + [regions(21, nr=26, ncols=(9, 12)),
                                           tuple(np.pad(a, ((0, 19), (0, 16)), constant_values=NODATA if j == 0 else 0.0)
                                                 for j, a in enumerate(skip_edges()["sentinel_first_ground"][0]))]
    assert len({w[0].shape for w in distinct}) == 1
    alone = [run([w], False, 1e-8, dtype=dtype) for w in distinct]
    for a, w in zip(alone, distinct):
        ref = advanced_window(*widen(w, dtype), False, 1e-8, ITMAX)
        assert a["rc"] == _lib.OK and a["iters"][0] == ref["iters"] > 0
        note("e_batch_volt", np.abs(a["volt"][0] - ref["volt"]).max(), 1e-9 * np.abs(ref["volt"]).max())
    order = np.random.default_rng(0).permutation(np.repeat(np.arange(6), 120))
    res = run([distinct[k] for k in order], False, 1e-8, dtype=dtype)
    cur_only = run([distinct[k] for k in order], False, 1e-8, dtype=dtype, want_volt=False)
    assert cur_only["volt"] is None and np.array_equal(cur_only["cur"], res["cur"])
    for j, k in enumerate(order):
        for key in ("cur", "volt", "iters", "relres"):
            assert np.array_equal(res[key][j], alone[k][key][0]), (j, k, key)
    # neighbours with conductances 1e6 times larger
    loud = [(np.where(w[0] > 0, w[0] * 1e6, w[0]), w[1] * 1e6, w[2] * 1e6) for w in distinct]
    for k in range(6):
        batch = [loud[(k + 1) % 6], loud[(k + 2) % 6], distinct[k], loud[(k + 3) % 6], loud[(k + 4) % 6]]
        res = run(batch, False, 1e-8, dtype=dtype)
        for key in ("cur", "volt", "iters", "relres"):
            assert np.array_equal(res[key][2], alone[k][key][0]), (k, key)

"""compute_omniscape_currents: many moving-window advanced-mode solves in one device call
(cs_b200_solve_advanced_batch).  The specification is the per-window compute_omniscape_current
(src/utils.jl:145-257), run here on FakeFactor, a direct solve.

CPU tests replace the C call with that per-window reference and check the host side: padding,
cropping, batch splitting, output order and argument checks.  GPU tests run the kernel."""
import ctypes
import itertools

import numpy as np
import pytest

import circuitscape_b200 as cb
from circuitscape_b200 import _lib, core, graph
from circuitscape_b200 import solver as S

from .fake_factor import FakeFactor


def _cfg(four, **kw):
    return {"connect_four_neighbors_only": "True" if four else "False", **kw}


def reference(g, src, gnd, cfg):
    """compute_omniscape_current on FakeFactor, returning (currents, voltages).  A window without a
    single node has nothing to solve: zeros (the per-window function has no graph to label there)."""
    if not np.any(np.asarray(g, dtype=np.float64) > 0):
        return np.zeros(np.shape(g)), np.zeros(np.shape(g))
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(S, "multiple_solve", lambda sol, m, b: FakeFactor(m, sol).solve_rhs(np.asarray(b))[0])
        cellmap = np.array(g, dtype=np.float64)
        cellmap[cellmap == core.NODATA] = 0.0
        nodemap = graph.construct_node_map(cellmap, None)
        four = core._flag(cfg, "connect_four_neighbors_only")
        G = graph.laplacian(graph.construct_graph(cellmap, nodemap, False, four))
        s, n, f = core.sources_and_grounds_from_maps(np.asarray(src, dtype=np.float64),
                                                     np.asarray(gnd, dtype=np.float64), nodemap, G.shape[0], "rmvsrc")
        prob = core.AdvancedProblem(G, graph.connected_components(G), s, n, f, nodemap, None, cellmap, S.CUDASolver())
        out = core.advanced_kernel(prob, core.Flags(is_raster=True, is_advanced=True), cfg)
        cur = cb.compute_omniscape_current(g, src, gnd, cfg)
        assert np.array_equal(cur, out.curmap)
        return out.curmap, out.voltmap


# ---------------------------------------------------------------------------
# windows
# ---------------------------------------------------------------------------
def example_window():
    """test/internal.jl:5-43"""
    g = np.array([[1, 5, 1.], [2, 1, 1], [9, 1, 6]])
    src = np.array([[1, 0, 0.], [0, 0, 0], [0, 1, 0]])
    gnd = np.array([[0, 0, 1.], [0, 0, 0], [0, 0, 0]])
    return g, src, gnd


def lognormal(rng, nr, nc, holes):
    g = np.exp(rng.normal(size=(nr, nc)))
    g[rng.random(g.shape) < holes] = core.NODATA
    return g


def mixed_grounds(seed):
    """finite and Inf grounds, a source cell that is also grounded, NODATA holes"""
    rng = np.random.default_rng(seed)
    g = lognormal(rng, 23, 17, 0.08)
    src = np.where(rng.random(g.shape) < 0.2, rng.uniform(0.5, 2.0, g.shape), 0.0)
    gnd = np.zeros_like(g)
    gnd[3, 4], gnd[15, 12], gnd[20, 2] = np.inf, 0.7, 2.5
    g[[3, 15, 20, 8], [4, 12, 2, 9]] = 1.0
    src[8, 9] = gnd[8, 9] = 1.5                      # a source on a grounded cell: rmvsrc drops it
    return g, src, gnd


def four_regions(seed):
    """NODATA walls split the window: sources + Inf ground | sources + finite ground |
    sources without ground | ground without sources"""
    rng = np.random.default_rng(seed)
    g = lognormal(rng, 10, 16, 0.05)
    g[:, [4, 8, 12]] = core.NODATA
    g[[2, 6, 1, 7, 9], [1, 6, 10, 14, 3]] = 1.0
    src = np.zeros_like(g)
    gnd = np.zeros_like(g)
    src[2, 1], gnd[8, 3] = 1.0, np.inf
    g[8, 3] = 1.0
    src[6, 6], gnd[0, 5] = 2.0, 0.8
    g[0, 5] = 1.0
    src[1, 10] = 1.0
    gnd[7, 14] = np.inf
    return g, src, gnd


def spiral(seed, n=21):
    """one corridor wound into a square spiral: a long path for the component labelling"""
    rng = np.random.default_rng(seed)
    g = np.full((n, n), core.NODATA)
    r = c = 0
    g[0, 0] = 1.0
    lengths = [n - 1] * 3 + [k for k in range(n - 3, 0, -2) for _ in range(2)]
    for L, (dr, dc) in zip(lengths, itertools.cycle([(0, 1), (1, 0), (0, -1), (-1, 0)])):
        for _ in range(L):
            r, c = r + dr, c + dc
            g[r, c] = rng.uniform(0.5, 2.0)
    src = np.zeros_like(g)
    gnd = np.zeros_like(g)
    src[r, c] = 1.0
    gnd[0, 0] = np.inf
    return g, src, gnd


def all_nodata():
    g = np.full((6, 5), core.NODATA)
    return g, np.ones_like(g), np.where(np.arange(30).reshape(6, 5) == 7, np.inf, 0.0)


def moving_window(rng, size=101, holes=0.03):
    """Omniscape's shape: unit sources on the valid cells, a direct ground at the target"""
    g = lognormal(rng, size, size, holes)
    t = size // 2
    g[t, t] = np.exp(rng.normal())
    src = np.where(g > 0, 1.0, 0.0)
    gnd = np.zeros_like(g)
    gnd[t, t] = np.inf
    return g, src, gnd


def parity_windows():
    ws = [example_window(), mixed_grounds(1), mixed_grounds(2), four_regions(3), spiral(4), all_nodata()]
    rng = np.random.default_rng(9)
    for nr, nc in ((1, 13), (11, 1), (17, 29)):
        g = lognormal(rng, nr, nc, 0.1)
        g[0, 0] = 1.0
        src = np.where(g > 0, rng.uniform(0, 1, g.shape), 0.0)
        gnd = np.zeros_like(g)
        gnd[0, 0] = np.inf
        gnd[-1, -1] = 0.3 if g[-1, -1] > 0 else 0.0
        ws.append((g, src, gnd))
    return ws


def split(ws):
    return [w[0] for w in ws], [w[1] for w in ws], [w[2] for w in ws]


# ---------------------------------------------------------------------------
# CPU: the C call replaced by the per-window reference
# ---------------------------------------------------------------------------
@pytest.fixture
def fake_batch(monkeypatch):
    calls = []

    def fake(g, src, gnd, four, device, rtol, itmax, want_volt=False):
        calls.append(g.shape)
        cfg = _cfg(four)
        res = [reference(g[w], src[w], gnd[w], cfg) for w in range(g.shape[0])]
        return dict(cur=np.stack([c for c, _ in res]), volt=np.stack([v for _, v in res]) if want_volt else None,
                    iters=np.arange(g.shape[0]), relres=np.zeros(g.shape[0]), rc=_lib.OK, first_failed=-1, msg="")

    monkeypatch.setattr(S, "solve_advanced_batch", fake)
    return calls


@pytest.mark.parametrize("four", [False, True])
def test_padding_cropping_batches_and_order(fake_batch, four):
    ws = parity_windows()
    g, s, n = split(ws)
    pad = (max(w.shape[0] for w in g), max(w.shape[1] for w in g))
    one = S.advanced_batch_bytes(pad[0] * pad[1], 8, True)
    out = cb.compute_omniscape_currents(g, s, n, _cfg(four), want_voltages=True, max_batch_bytes=3 * one + 1)
    assert fake_batch == [(3,) + pad] * 3
    assert [c.shape for c in out.currents] == [w.shape for w in g] == [v.shape for v in out.voltages]
    assert list(out.iterations) == [0, 1, 2, 0, 1, 2, 0, 1, 2]
    for k, (gw, sw, nw) in enumerate(ws):
        cur, volt = reference(gw, sw, nw, _cfg(four))
        assert np.array_equal(out.currents[k], cur), k
        assert np.array_equal(out.voltages[k], volt), k


def test_stack_input_and_single_batch(fake_batch):
    rng = np.random.default_rng(0)
    ws = [moving_window(rng, 9) for _ in range(4)]
    g, s, n = (np.stack(a) for a in split(ws))
    out = cb.compute_omniscape_currents(g, s, n, {})
    assert fake_batch == [(4, 9, 9)] and out.voltages is None
    for k in range(4):
        assert np.array_equal(out.currents[k], reference(g[k], s[k], n[k], {})[0])


@pytest.mark.parametrize("bad", ["count", "shape", "ndim", "empty", "dtype", "stack2d", "budget"])
def test_malformed_input_is_rejected_before_the_device(fake_batch, bad):
    g, s, n = split([example_window(), example_window()])
    kw = {}
    if bad == "count":
        n = n[:1]
    elif bad == "shape":
        s[1] = s[1][:2]
    elif bad == "ndim":
        g[0] = g[0].ravel()
    elif bad == "empty":
        g[1], s[1], n[1] = (np.zeros((0, 3)),) * 3
    elif bad == "dtype":
        g[0] = np.array([["a", "b"], ["c", "d"]])
    elif bad == "stack2d":
        g = g[0]
    else:
        kw["max_batch_bytes"] = 0
    with pytest.raises(ValueError):
        cb.compute_omniscape_currents(g, s, n, {}, **kw)
    assert fake_batch == []


def test_bad_arguments_are_rejected_without_a_device():
    lib = _lib.load()
    g = np.ones((1, 3, 3))
    p = g.ctypes.data_as(ctypes.c_void_p)
    bad = ctypes.c_int64(5)
    calls = [(1, 0, 3, p, p, p, 1), (1, 3, 3, p, p, p, 7), (1, 3, 3, None, p, p, 1), (-1, 3, 3, p, p, p, 1),
             (1, 1 << 20, 1 << 20, p, p, p, 1)]
    for nwin, nr, nc, a, b, c, dt in calls:
        rc = lib.cs_b200_solve_advanced_batch(nwin, nr, nc, a, b, c, dt, 0, 0, 1e-6, 100, p, None, None, None,
                                              ctypes.byref(bad))
        assert rc == _lib.ERR_ARG and bad.value == -1
        assert lib.cs_b200_last_error(None)
    with pytest.raises(cb.B200Error):
        S.solve_advanced_batch(np.zeros((1, 0, 3)), np.zeros((1, 0, 3)), np.zeros((1, 0, 3)), False, 0, 1e-6, 10)


def test_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    g, s, n = split([example_window()])
    with pytest.raises(cb.B200Unavailable):
        cb.compute_omniscape_currents(g, s, n, {})


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
@pytest.mark.gpu
def test_reference_example_on_device():
    g, s, n = split([example_window()])
    out = cb.compute_omniscape_currents(g, s, n, {"connect_four_neighbors_only": "False", "solver": "cuda"})
    assert abs(out.currents[0][0, 2] - 2.0) < 1e-9


@pytest.mark.gpu
@pytest.mark.parametrize("four", [False, True])
@pytest.mark.parametrize("f32", [False, True])
def test_parity_with_the_per_window_reference(four, f32):
    ws = parity_windows()
    if f32:
        ws = [tuple(a.astype(np.float32) for a in w) for w in ws]
    g, s, n = split(ws)
    cfg = _cfg(four, gpu_rtol="1e-10")
    out = cb.compute_omniscape_currents(g, s, n, cfg, want_voltages=True)
    for k, (gw, sw, nw) in enumerate(ws):
        cur, volt = reference(gw, sw, nw, cfg)
        assert np.abs(out.currents[k] - cur).max() <= 1e-7 * np.abs(cur).max(), k
        assert np.abs(out.voltages[k] - volt).max() <= 1e-7 * np.abs(volt).max(), k
        assert np.all(out.relres[k] < 1e-4)
    # skipped components stay 0: four_regions has a source-only and a ground-only region
    fr = out.currents[3]
    assert np.all(fr[:, 9:] == 0) and np.any(fr[:, :4] > 0) and np.any(fr[:, 5:8] > 0)
    assert np.all(out.currents[5] == 0) and out.iterations[5] == 0


def moving_windows(count, seed=42):
    rng = np.random.default_rng(seed)
    return [moving_window(rng) for _ in range(count)]


@pytest.mark.gpu
def test_default_settings_meet_the_reference_map_bar():
    ws = moving_windows(6)
    g, s, n = split(ws)
    out = cb.compute_omniscape_currents(g, s, n, {})
    for k, (gw, sw, nw) in enumerate(ws):
        cur, _ = reference(gw, sw, nw, {})
        d = out.currents[k] - cur
        assert (d ** 2).sum() < 1e-6, k                       # test/test_utils.jl:196
        assert np.abs(d).max() <= 1e-5 * cur.max(), k


@pytest.mark.gpu
def test_agrees_with_the_per_window_device_path():
    """The batched path at default settings against the per-window device path at rtol 1e-10: at the
    default rtol the per-window AMG-PCG stops with a true residual of ~1.2e-4 on these windows (unit
    sources on every cell) and fails its own 1e-4 gate, with the fp32 or the fp64 V-cycle."""
    ws = moving_windows(3, seed=7)
    g, s, n = split(ws)
    out = cb.compute_omniscape_currents(g, s, n, {})
    for k, (gw, sw, nw) in enumerate(ws):
        cur = cb.compute_omniscape_current(gw, sw, nw, {}, solver=cb.CUDASolver(rtol=1e-10))
        assert np.abs(out.currents[k] - cur).max() <= 1e-5 * cur.max(), k


@pytest.mark.gpu
def test_bit_identical_repeats_and_batch_splits():
    ws = moving_windows(5, seed=3) + parity_windows()
    g, s, n = split(ws)
    a = cb.compute_omniscape_currents(g, s, n, {}, want_voltages=True)
    b = cb.compute_omniscape_currents(g, s, n, {}, want_voltages=True)
    one = S.advanced_batch_bytes(101 * 101, 8, True)
    c = cb.compute_omniscape_currents(g, s, n, {}, want_voltages=True, max_batch_bytes=2 * one)
    for other in (b, c):
        assert all(np.array_equal(x, y) for x, y in zip(a.currents, other.currents))
        assert all(np.array_equal(x, y) for x, y in zip(a.voltages, other.voltages))
        assert np.array_equal(a.iterations, other.iterations) and np.array_equal(a.relres, other.relres)


@pytest.mark.gpu
def test_itmax_fails_the_gate_and_still_writes_outputs():
    ws = [all_nodata(), all_nodata()] + moving_windows(2)
    g, s, n = split(ws)
    two = 2 * S.advanced_batch_bytes(101 * 101, 8, False)
    with pytest.raises(cb.SolverResidualError, match=r"exceeds tolerance 0.0001 for window 2 ") as e:
        cb.compute_omniscape_currents(g, s, n, {}, solver=cb.CUDASolver(itmax=2), max_batch_bytes=two)
    assert e.value.window == 2
    res = S.solve_advanced_batch(*[np.stack(x) for x in (g[2:], s[2:], n[2:])], False, 0, 1e-6, 2, want_volt=True)
    assert res["rc"] == _lib.ERR_RESIDUAL and res["first_failed"] == 0 and "window 0" in res["msg"]
    assert np.all(res["iters"] == 2) and np.all(res["relres"] > 1e-4)
    assert np.all(np.isfinite(res["cur"])) and res["cur"].max() > 0 and res["volt"].max() > 0
    with pytest.raises(cb.B200Error):
        S.solve_advanced_batch(np.ones((1, 3, 3)), np.ones((1, 3, 3)), np.ones((1, 3, 3)), False, 10_000, 1e-6, 10)

"""moving_window_current_map: Omniscape's moving-window loop over one landscape, with the windows cut and
their currents summed on the device (cs_b200_solve_moving_windows).

The specification is a composition of existing pieces: window w is the (2R+1)^2 square around its target
(cells off the landscape, off the disc or without conductance get g = 0), solved as
compute_omniscape_current solves it, and placed into the landscape map in window order in float64.  The
CPU tests anchor that square-window definition to the reference function on the landscape's clipped
windows and check the argument rules; the GPU tests hold the device map bit for bit to the same
composition built on the host from compute_omniscape_currents."""
import ctypes

import numpy as np
import pytest

import circuitscape_b200 as cb
from circuitscape_b200 import _lib, core
from circuitscape_b200 import solver as S

from .test_advanced_batch import reference

NODATA = core.NODATA


def _cfg(four, **kw):
    return {"connect_four_neighbors_only": "True" if four else "False", **kw}


# ---------------------------------------------------------------------------
# the host composition
# ---------------------------------------------------------------------------
def in_disc(R, circular):
    d = np.arange(-R, R + 1)
    return (d[:, None] ** 2 + d[None, :] ** 2 <= R * R) if circular else np.ones((2 * R + 1,) * 2, dtype=bool)


def square_window(G, Sr, t, R, circular, scale=1.0, gnd=np.inf, dtype=np.float64):
    """window (g, src, gnd) around target t as the device cuts it: dtype arrays of (2R+1)^2 cells"""
    W = 2 * R + 1
    g, s, n = (np.zeros((W, W), dtype=dtype) for _ in range(3))
    r0, c0 = t[0] - R, t[1] - R
    rr, cc = np.meshgrid(np.arange(W) + r0, np.arange(W) + c0, indexing="ij")
    inside = (rr >= 0) & (rr < G.shape[0]) & (cc >= 0) & (cc < G.shape[1]) & in_disc(R, circular)
    gl = np.zeros((W, W), dtype=G.dtype)
    gl[inside] = G[rr[inside], cc[inside]]
    node = inside & (gl.astype(np.float64) > 0)
    g[node] = gl[node]
    s[node] = (float(scale) * Sr[rr[node], cc[node]].astype(np.float64)).astype(dtype)
    if node[R, R]:
        n[R, R] = dtype(gnd)
    return g, s, n


def clipped_window(G, Sr, t, R, circular, scale=1.0, gnd=np.inf):
    """the reference's form of the same window: the landscape slice around t, NODATA off the disc;
    returns (g, src, gnd, (row, col) of the slice's origin)"""
    r0, r1 = max(t[0] - R, 0), min(t[0] + R + 1, G.shape[0])
    c0, c1 = max(t[1] - R, 0), min(t[1] + R + 1, G.shape[1])
    g = np.array(G[r0:r1, c0:c1], dtype=np.float64)
    disc = in_disc(R, circular)[r0 - (t[0] - R):r1 - (t[0] - R), c0 - (t[1] - R):c1 - (t[1] - R)]
    g[~disc] = NODATA
    s = scale * np.array(Sr[r0:r1, c0:c1], dtype=np.float64)
    n = np.zeros_like(g)
    if g[t[0] - r0, t[1] - c0] > 0:
        n[t[0] - r0, t[1] - c0] = gnd
    return g, s, n, (r0, c0)


def place_sum(curs, origins, shape):
    """sum windows into one float64 map in window order; origins may lie off the map (clipped)"""
    cum = np.zeros(shape)
    for cur, (r0, c0) in zip(curs, origins):
        h, w = cur.shape
        a, b = max(r0, 0), max(c0, 0)
        e, f = min(r0 + h, shape[0]), min(c0 + w, shape[1])
        if a < e and b < f:
            cum[a:e, b:f] += cur[a - r0:e - r0, b - c0:f - c0]
    return cum


def host_composition(G, Sr, targets, R, cfg, circular=True, scale=None, gnd=None, dtype=np.float64, solver=None):
    """square windows through compute_omniscape_currents (one stack), placed and summed on the host"""
    nwin = len(targets)
    scale = np.ones(nwin) if scale is None else scale
    gnd = np.full(nwin, np.inf) if gnd is None else gnd
    ws = [square_window(G, Sr, t, R, circular, scale[w], gnd[w], dtype) for w, t in enumerate(targets)]
    stacks = [np.stack([w[k] for w in ws]) for k in range(3)]
    out = cb.compute_omniscape_currents(*stacks, cfg, solver=solver, max_batch_bytes=1 << 40)
    return place_sum(out.currents, [(t[0] - R, t[1] - R) for t in targets], G.shape), out


def landscape(seed, nr, nc, holes=0.08):
    rng = np.random.default_rng(seed)
    G = np.exp(rng.normal(size=(nr, nc)))
    G[rng.random(G.shape) < holes] = NODATA
    G[rng.random(G.shape) < 0.01] = 0.0
    Sr = rng.uniform(0.2, 1.5, size=(nr, nc))
    return G, Sr


def edge_targets(nr, nc):
    return np.array([(0, 0), (0, nc - 1), (nr - 1, 0), (nr - 1, nc - 1), (0, nc // 2), (nr // 2, 0),
                     (nr - 1, nc // 3), (nr // 3, nc - 1), (nr // 2, nc // 2), (2, 3)])


# ---------------------------------------------------------------------------
# CPU: the square-window definition against the reference's clipped windows
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("circular", [False, True])
@pytest.mark.parametrize("four", [False, True])
def test_square_windows_agree_with_the_reference_clipped_windows(circular, four):
    G, Sr = landscape(1, 19, 23)
    targets = edge_targets(*G.shape)
    G[tuple(targets[-1])] = 1.3                       # grounded target with a source under it: rmvsrc
    R = 4
    scale = np.linspace(0.5, 2.0, len(targets))
    gnd = np.where(np.arange(len(targets)) % 3 == 1, 0.8, np.inf)
    cfg = _cfg(four)
    clipped, square = [], []
    for w, t in enumerate(targets):
        g, s, n, org = clipped_window(G, Sr, t, R, circular, scale[w], gnd[w])
        clipped.append((reference(g, s, n, cfg)[0], org))
        sg, ss, sn = square_window(G, Sr, t, R, circular, scale[w], gnd[w])
        square.append((reference(sg, ss, sn, cfg)[0], (t[0] - R, t[1] - R)))
    a = place_sum([c for c, _ in clipped], [o for _, o in clipped], G.shape)
    b = place_sum([c for c, _ in square], [o for _, o in square], G.shape)
    assert a.max() > 0
    assert np.abs(a - b).max() <= 1e-10 * np.abs(a).max()


def test_core_passes_targets_settings_and_defaults_through(monkeypatch):
    seen = {}

    def fake(g, src, tr, tc, radius, circular, scale, gnd, four, device, rtol, itmax, budget):
        seen.update(dtype=g.dtype, tr=tr.copy(), tc=tc.copy(), radius=radius, circular=circular, scale=scale,
                    gnd=gnd.copy(), four=four, device=device, rtol=rtol, itmax=itmax, budget=budget)
        return dict(cum=np.zeros(g.shape), iters=np.arange(len(tr)), relres=np.zeros(len(tr)), rc=_lib.OK,
                    first_failed=-1, msg="")

    monkeypatch.setattr(S, "solve_moving_windows", fake)
    G, Sr = landscape(2, 9, 7)
    out = cb.moving_window_current_map(G.astype(np.float32), Sr.astype(np.float32), [(1, 2), (8, 6)], 3,
                                       _cfg(True), solver=cb.CUDASolver(rtol=1e-8, itmax=77), max_batch_bytes=123)
    assert out.current.shape == G.shape and list(out.iterations) == [0, 1]
    assert seen["dtype"] == np.float32 and list(seen["tr"]) == [1, 8] and list(seen["tc"]) == [2, 6]
    assert seen["radius"] == 3 and seen["circular"] and seen["scale"] is None and np.all(np.isinf(seen["gnd"]))
    assert seen["four"] and (seen["rtol"], seen["itmax"], seen["budget"]) == (1e-8, 77, 123)
    cb.moving_window_current_map(G, Sr.astype(np.float32), np.zeros((2, 2), dtype=int), 0, {}, source_scale=2.0,
                                 ground=[1.0, 2.0], circular=False, max_batch_bytes=5)
    assert seen["dtype"] == np.float64 and not seen["circular"] and list(seen["scale"]) == [2.0, 2.0]
    assert list(seen["gnd"]) == [1.0, 2.0]


@pytest.mark.parametrize("bad", ["ndim", "shape", "dtype", "targets_shape", "targets_float", "scale_len",
                                 "ground_len", "budget"])
def test_malformed_python_arguments_are_rejected_before_the_device(monkeypatch, bad):
    monkeypatch.setattr(S, "solve_moving_windows", lambda *a: pytest.fail("reached the device call"))
    G, Sr = landscape(3, 6, 5)
    t, kw = np.array([(1, 1), (2, 3)]), {}
    if bad == "ndim":
        G = G.ravel()
    elif bad == "shape":
        Sr = Sr[:4]
    elif bad == "dtype":
        G = np.full(G.shape, "a")
    elif bad == "targets_shape":
        t = np.array([1, 2, 3])
    elif bad == "targets_float":
        t = t.astype(float)
    elif bad == "scale_len":
        kw["source_scale"] = [1.0, 2.0, 3.0]
    elif bad == "ground_len":
        kw["ground"] = np.ones((2, 1))
    else:
        kw["max_batch_bytes"] = 0
    with pytest.raises(ValueError):
        cb.moving_window_current_map(G, Sr, t, 2, {}, **kw)


def _call(lib, nr=5, nc=4, g=True, src=True, dtype=1, nwin=2, tr=(0, 4), tc=(0, 3), radius=2, scale=None,
          gnd=None, rtol=1e-6, itmax=100, budget=1 << 20, cum=True, null_targets=False):
    a = np.ones(max(nr * nc, 1) if 0 < nr < 1 << 16 and 0 < nc < 1 << 16 else 1)
    out = np.full(a.shape, 7.0)
    p = a.ctypes.data_as(ctypes.c_void_p)
    tr_ = np.array(tr, dtype=np.int64)
    tc_ = np.array(tc, dtype=np.int64)
    sc_ = None if scale is None else np.array(scale, dtype=np.float64)
    gn_ = None if gnd is None else np.array(gnd, dtype=np.float64)
    bad = ctypes.c_int64(5)
    rc = lib.cs_b200_solve_moving_windows(nr, nc, p if g else None, p if src else None, dtype, nwin,
                                          None if null_targets else _lib._ptr(tr_),
                                          None if null_targets else _lib._ptr(tc_), radius, 1, _lib._ptr(sc_),
                                          _lib._ptr(gn_), 0, 0, rtol, itmax, budget,
                                          _lib._ptr(out) if cum else None, None, None, ctypes.byref(bad))
    return rc, bad.value, out


BAD_ABI = {
    "rows0": dict(nr=0), "cols_negative": dict(nc=-1), "landscape_over_int_max": dict(nr=1 << 20, nc=1 << 20),
    "radius_negative": dict(radius=-1), "window_over_int_max": dict(radius=30000), "nwin_negative": dict(nwin=-1),
    "target_row_high": dict(tr=(0, 5)), "target_row_negative": dict(tr=(-1, 0)), "target_col_high": dict(tc=(0, 4)),
    "ground_zero": dict(gnd=(1.0, 0.0)), "ground_negative": dict(gnd=(-1.0, 1.0)),
    "ground_nan": dict(gnd=(np.nan, 1.0)), "scale_nan": dict(scale=(1.0, np.nan)),
    "scale_inf": dict(scale=(np.inf, 1.0)), "scale_minus_inf": dict(scale=(1.0, -np.inf)),
    "null_g": dict(g=False), "null_src": dict(src=False), "null_cum": dict(cum=False),
    "null_targets": dict(null_targets=True), "dtype": dict(dtype=7), "budget": dict(budget=0),
    "rtol": dict(rtol=float("nan")), "itmax": dict(itmax=-1),
}


@pytest.mark.parametrize("case", sorted(BAD_ABI))
def test_bad_abi_arguments_are_rejected_without_a_device(case):
    lib = _lib.load()
    rc, first_failed, _ = _call(lib, **BAD_ABI[case])
    assert rc == _lib.ERR_ARG and first_failed == -1
    assert lib.cs_b200_last_error(None)


def test_bad_values_raise_through_python():
    G, Sr = landscape(4, 6, 5)
    for kw in (dict(targets=[(6, 0)]), dict(targets=[(0, -1)]), dict(radius=-2), dict(ground=0.0),
               dict(ground=np.nan), dict(source_scale=np.inf)):
        args = dict(targets=[(1, 1)], radius=2) | kw
        with pytest.raises(cb.B200Error) as e:
            cb.moving_window_current_map(G, Sr, args.pop("targets"), args.pop("radius"), {}, **args)
        assert e.value.code == _lib.ERR_ARG


def test_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    G, Sr = landscape(5, 6, 5)
    with pytest.raises(cb.B200Unavailable):
        cb.moving_window_current_map(G, Sr, [(1, 1)], 2, {})
    with pytest.raises(cb.B200Unavailable):
        cb.moving_window_current_map(G, Sr, np.zeros((0, 2), dtype=int), 2, {})


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
def job(seed, nr=37, nc=53):
    """a non-square landscape with NODATA holes; targets on corners and edges, one on a NODATA cell,
    a repeated target; non-unit scales; Inf and finite target grounds"""
    G, Sr = landscape(seed, nr, nc)
    rng = np.random.default_rng(seed + 100)
    t = np.concatenate([edge_targets(nr, nc), np.stack([rng.integers(0, nr, 20), rng.integers(0, nc, 20)], 1)])
    t = np.concatenate([t, t[[3, 12]]])
    for k in (0, 1, 7, 12):
        G[tuple(t[k])] = 1.0
    G[tuple(t[5])] = NODATA
    scale = rng.uniform(0.25, 3.0, len(t))
    gnd = np.where(rng.random(len(t)) < 0.4, rng.uniform(0.3, 4.0, len(t)), np.inf)
    return G, Sr, t, scale, gnd


@pytest.mark.gpu
@pytest.mark.parametrize("R", [0, 3, 7])
@pytest.mark.parametrize("circular", [False, True])
@pytest.mark.parametrize("four", [False, True])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_bit_identical_to_the_host_composition(dtype, four, circular, R):
    G, Sr, t, scale, gnd = job(11)
    G, Sr = G.astype(dtype), Sr.astype(dtype)
    cfg = _cfg(four)
    out = cb.moving_window_current_map(G, Sr, t, R, cfg, source_scale=scale, ground=gnd, circular=circular)
    ref, batch = host_composition(G, Sr, t, R, cfg, circular, scale, gnd, dtype)
    assert out.current.shape == G.shape and out.current.dtype == np.float64
    assert np.array_equal(out.current, ref)
    assert np.array_equal(out.iterations, batch.iterations) and np.array_equal(out.relres, batch.relres)
    if R > 0:
        assert out.current.max() > 0 and out.iterations[5] == 0      # target on NODATA: nothing grounded


@pytest.mark.gpu
def test_a_disc_that_splits_a_component():
    """a U-shaped corridor whose bend lies in the square's corners: the disc cuts it into a grounded arm
    (with the target) and an ungrounded arm, which is skipped"""
    G = np.full((21, 21), NODATA)
    G[8:13, 8] = G[8:13, 12] = G[7, 8:13] = 1.0       # arms at dc = -2 and +2, bend at dr = -3
    G[10, 10:12] = 1.0                                # the target, joined to the right arm
    Sr = np.ones_like(G)
    t = np.array([(10, 10)])
    for circular in (False, True):
        out = cb.moving_window_current_map(G, Sr, t, 3, {}, circular=circular)
        ref, _ = host_composition(G, Sr, t, 3, {}, circular)
        assert np.array_equal(out.current, ref)
        left = out.current[8:13, 8]
        assert np.all(left == 0) if circular else np.all(left > 0)
        assert np.all(out.current[8:13, 12] > 0)


@pytest.mark.gpu
def test_agrees_with_the_per_window_device_path():
    """one target per call against compute_omniscape_current on the clipped window, per-window device
    path at rtol 1e-10, the bar of test_advanced_batch.py::test_agrees_with_the_per_window_device_path"""
    G, Sr = landscape(21, 90, 80, holes=0.03)
    R = 20
    for t in [(45, 40), (3, 70), (88, 2)]:
        G[t] = 1.0
        out = cb.moving_window_current_map(G, Sr, [t], R, {})
        g, s, n, org = clipped_window(G, Sr, t, R, True)
        cur = cb.compute_omniscape_current(g, s, n, {}, solver=cb.CUDASolver(rtol=1e-10))
        ref = place_sum([cur], [org], G.shape)
        assert np.abs(out.current - ref).max() <= 1e-5 * cur.max(), t


@pytest.mark.gpu
def test_batch_splits_and_repeats_are_bit_identical():
    G, Sr, t, scale, gnd = job(12, 60, 45)
    R = 6
    kw = dict(source_scale=scale, ground=gnd)
    whole = cb.moving_window_current_map(G, Sr, t, R, {}, max_batch_bytes=1 << 40, **kw)
    for budget in (1, 3 * S.advanced_batch_bytes((2 * R + 1) ** 2, 8, False), 1 << 40):
        other = cb.moving_window_current_map(G, Sr, t, R, {}, max_batch_bytes=budget, **kw)
        assert np.array_equal(whole.current, other.current), budget
        assert np.array_equal(whole.iterations, other.iterations) and np.array_equal(whole.relres, other.relres)


@pytest.mark.gpu
def test_every_cell_of_a_landscape_in_several_batches():
    G, Sr = landscape(13, 120, 120, holes=0.05)
    R = 8
    rr, cc = np.meshgrid(np.arange(120), np.arange(120), indexing="ij")
    t = np.stack([rr.ravel(), cc.ravel()], 1)
    assert len(t) >= 10_000
    budget = 4000 * S.advanced_batch_bytes((2 * R + 1) ** 2, 8, False)     # four batches
    out = cb.moving_window_current_map(G, Sr, t, R, {}, max_batch_bytes=budget)
    ref, batch = host_composition(G, Sr, t, R, {})
    assert np.array_equal(out.current, ref)
    assert np.array_equal(out.iterations, batch.iterations)
    assert np.all(out.relres < 1e-4)


@pytest.mark.gpu
def test_no_windows_leave_the_map_at_zero():
    G, Sr = landscape(14, 8, 9)
    out = cb.moving_window_current_map(G, Sr, np.zeros((0, 2), dtype=np.int64), 3, {})
    assert out.current.shape == (8, 9) and np.all(out.current == 0) and len(out.iterations) == 0


@pytest.mark.gpu
def test_itmax_fails_the_gate_with_the_global_window_index():
    G, Sr = landscape(15, 40, 40, holes=0.0)
    t = np.array([(5, 5), (6, 6), (20, 20), (30, 12)])
    G[5, 5] = G[6, 6] = NODATA                        # no ground: nothing solved, nothing fails
    one = S.advanced_batch_bytes(21 * 21, 8, False)
    with pytest.raises(cb.SolverResidualError, match=r"exceeds tolerance 0.0001 for window 2 ") as e:
        cb.moving_window_current_map(G, Sr, t, 10, {}, solver=cb.CUDASolver(itmax=2), max_batch_bytes=one)
    assert e.value.window == 2
    res = S.solve_moving_windows(G, Sr, t[:, 0], t[:, 1], 10, True, None, None, False, 0, 1e-6, 2, one)
    assert res["rc"] == _lib.ERR_RESIDUAL and res["first_failed"] == 2 and "window 2 " in res["msg"]
    assert list(res["iters"]) == [0, 0, 2, 2] and np.all(res["relres"][2:] > 1e-4)
    assert np.all(np.isfinite(res["cum"])) and res["cum"].max() > 0

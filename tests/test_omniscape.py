"""omniscape_current_maps: a whole Omniscape job on the device (cs_b200_solve_omniscape) -- block targets,
per-window source normalisation, the moving-window solves, flow potential and the normalised map.

The specification is restated below in float64 on the host (targets, amps, window sums, scales, both
window kinds, normalisation and the NODATA mask).  The CPU tests anchor that restatement to the
reference function on Omniscape's clipped windows and check the argument rules; the GPU tests hold the
device to it: targets and amps bit for bit, scales to summation order, and the maps bit for bit to the
same windows solved by compute_omniscape_currents and placed on the host."""
import ctypes

import numpy as np
import pytest

import circuitscape_b200 as cb
from circuitscape_b200 import _lib, core
from circuitscape_b200 import solver as S

from .test_advanced_batch import reference
from .test_moving_windows import clipped_window, in_disc, place_sum, square_window
from .test_symmetric_stencil import _registers_and_stack

NODATA = core.NODATA


def _cfg(four):
    return {"connect_four_neighbors_only": "True" if four else "False"}


# ---------------------------------------------------------------------------
# the host restatement
# ---------------------------------------------------------------------------
def effective(G, Sr, theta):
    """s': the strength where it is finite, above theta and on a node (g > 0), else 0 (Sr's dtype)"""
    g, s = np.asarray(G, dtype=np.float64), np.asarray(Sr, dtype=np.float64)
    with np.errstate(invalid="ignore"):
        ok = (s > theta) & np.isfinite(s) & (g > 0)
    return np.where(ok, Sr, 0).astype(Sr.dtype)


def host_targets(G, Sr, bs, theta):
    """block centres in block-column-major order, amps summed sequentially in float64 from +0.0 (column
    outer, row inner); the ones with amps > 0"""
    sp = effective(G, Sr, theta).astype(np.float64)
    h, (nr, nc) = (bs - 1) // 2, G.shape
    t, amps = [], []
    for tc in range(h, nc, bs):
        for tr in range(h, nr, bs):
            a = 0.0
            for c in range(tc - h, min(tc + h, nc - 1) + 1):
                for r in range(tr - h, min(tr + h, nr - 1) + 1):
                    a += float(sp[r, c])
            if a > 0:
                t.append((tr, tc))
                amps.append(a)
    return np.array(t, dtype=np.int64).reshape(-1, 2), np.array(amps)


def outside_block(R, h):
    d = np.abs(np.arange(-R, R + 1))
    return (d[:, None] > h) | (d[None, :] > h)


def in_landscape(shape, t, R):
    W = 2 * R + 1
    rr, cc = np.meshgrid(np.arange(W) + t[0] - R, np.arange(W) + t[1] - R, indexing="ij")
    inside = (rr >= 0) & (rr < shape[0]) & (cc >= 0) & (cc < shape[1])
    return inside, rr, cc


def window_sums(sp, targets, R, h):
    """float64 sum of s' over each target's landscape cells in the disc and outside its block"""
    out = []
    keep = in_disc(R, True) & outside_block(R, h)
    for t in targets:
        inside, rr, cc = in_landscape(sp.shape, t, R)
        m = inside & keep
        out.append(float(np.sum(sp[rr[m], cc[m]].astype(np.float64))))
    return np.array(out)


def scales(amps, sums):
    return np.where(sums > 0, amps / np.where(sums > 0, sums, 1.0), 0.0)


def omni_window(G, sp, t, R, h, scale, dtype, flow):
    """the conductance (flow False) or flow-potential (flow True) window of target t, square form"""
    g, s, n = square_window(G, sp, t, R, True, scale, np.inf, dtype)
    s[~outside_block(R, h)] = 0
    if flow:
        inside, _, _ = in_landscape(G.shape, t, R)
        g = np.where(inside & in_disc(R, True), 1, 0).astype(dtype)
        n = np.zeros_like(g)
        n[R, R] = np.inf
    return g, s, n


def finish(cum, fp, G):
    """normalized = fp > 0 ? cum / fp : 0, then -9999 where g is NaN or -9999 in every map"""
    g = np.asarray(G, dtype=np.float64)
    mask = np.isnan(g) | (g == NODATA)
    norm = None
    if fp is not None:
        norm = np.where(fp > 0, cum / np.where(fp > 0, fp, 1.0), 0.0)
        fp, norm = np.where(mask, NODATA, fp), np.where(mask, NODATA, norm)
    return np.where(mask, NODATA, cum), fp, norm


def host_maps(G, Sr, targets, scale, R, bs, theta, cfg, dtype, flow):
    """every window through compute_omniscape_currents (one stack per kind), placed and summed on the
    host, then finished; returns (cum, fp, normalized, batch, fp_batch)"""
    sp = effective(G, Sr, theta)
    h = (bs - 1) // 2
    origins = [(t[0] - R, t[1] - R) for t in targets]
    maps, batches = [], []
    for kind in ((False, True) if flow else (False,)):
        if len(targets) == 0:
            maps.append(np.zeros(G.shape))
            batches.append(None)
            continue
        ws = [omni_window(G, sp, t, R, h, scale[w], dtype, kind) for w, t in enumerate(targets)]
        out = cb.compute_omniscape_currents(*[np.stack([w[k] for w in ws]) for k in range(3)], cfg,
                                            max_batch_bytes=1 << 40)
        maps.append(place_sum(out.currents, origins, G.shape))
        batches.append(out)
    cum, fp, norm = finish(maps[0], maps[1] if flow else None, G)
    return cum, fp, norm, batches[0], batches[1] if flow else None


def landscape(seed, nr, nc, holes=0.08):
    rng = np.random.default_rng(seed)
    G = np.exp(rng.normal(size=(nr, nc)))
    G[rng.random(G.shape) < holes] = NODATA
    G[rng.random(G.shape) < 0.01] = 0.0
    G[rng.random(G.shape) < 0.01] = np.nan
    Sr = rng.uniform(0.0, 1.5, size=(nr, nc))
    Sr[rng.random(G.shape) < 0.3] = 0.0
    return G, Sr


# ---------------------------------------------------------------------------
# CPU: the restatement against the reference's clipped windows
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("bs,R", [(1, 3), (3, 3), (5, 4), (5, 3), (7, 2)])
@pytest.mark.parametrize("four", [False, True])
def test_square_windows_agree_with_omniscapes_clipped_windows(four, bs, R):
    """Omniscape's windows (the landscape slice around the target, NODATA off the disc, the block's
    sources zeroed, sources normalised; flow potential: conductance 1 on the slice's disc) through the
    reference function, against the restatement's square windows through the same function.  Targets
    lie on edges and corners; (5, 3) has block corners outside the disc and (7, 2) a block larger than
    the disc (every window sum 0, nothing injected)."""
    G, Sr = landscape(1, 17, 22)
    G[np.isnan(G)] = NODATA                       # the reference's cellmap reads NaN as a conductance
    theta = 0.2
    targets, amps = host_targets(G, Sr, bs, theta)
    sp = effective(G, Sr, theta)
    h = (bs - 1) // 2
    scale = scales(amps, window_sums(sp, targets, R, h))
    assert len(targets) > 0 and (bs < 7 or np.all(scale == 0))
    cfg = _cfg(four)
    for flow in (False, True):
        clipped, square = [], []
        for w, t in enumerate(targets):
            g, s, n, org = clipped_window(G, sp, t, R, True, scale[w])
            rr, cc = np.meshgrid(np.arange(g.shape[0]) + org[0], np.arange(g.shape[1]) + org[1], indexing="ij")
            s[(np.abs(rr - t[0]) <= h) & (np.abs(cc - t[1]) <= h)] = 0.0
            if flow:
                g = np.where((rr - t[0]) ** 2 + (cc - t[1]) ** 2 <= R * R, 1.0, NODATA)
                n = np.zeros_like(g)
                n[t[0] - org[0], t[1] - org[1]] = np.inf
            clipped.append((reference(g, s, n, cfg)[0], org))
            sg, ss, sn = omni_window(G, sp, t, R, h, scale[w], np.float64, flow)
            square.append((reference(sg, ss, sn, cfg)[0], (t[0] - R, t[1] - R)))
        a = place_sum([c for c, _ in clipped], [o for _, o in clipped], G.shape)
        b = place_sum([c for c, _ in square], [o for _, o in square], G.shape)
        assert np.abs(a - b).max() <= 1e-10 * max(np.abs(a).max(), 1e-300)
        assert (a.max() > 0) == (bs < 7)


def test_flow_potential_windows_have_conductance_one_on_nodata():
    """the clipped flow-potential window above sets every slice cell in the disc to 1: the square form
    does the same for NODATA, 0 and NaN cells, and keeps their (zero) sources"""
    G = np.full((5, 5), 2.0)
    G[1, 1], G[1, 3], G[3, 1] = NODATA, 0.0, np.nan
    Sr = np.ones((5, 5))
    sp = effective(G, Sr, 0.0)
    g, s, n = omni_window(G, sp, (2, 2), 2, 0, 0.5, np.float64, True)
    assert np.array_equal(g, in_disc(2, True).astype(float))
    assert s[1, 1] == s[1, 3] == s[3, 1] == 0 and s[0, 2] == 0.5 and s[2, 2] == 0
    assert n[2, 2] == np.inf and np.count_nonzero(n) == 1


def test_restated_targets_amps_and_the_finish_rules():
    """the sequential amps equal block sums of s' (threshold, NaN, Inf, negative, off-node strengths
    dropped); clipped blocks at the far edges; the finish rules on a hand-made map"""
    G, Sr = landscape(2, 11, 13)
    Sr[0, 0], Sr[4, 4], Sr[7, 2] = np.inf, -3.0, np.nan
    for bs in (1, 3, 5):
        t, amps = host_targets(G, Sr, bs, 0.25)
        sp = effective(G, Sr, 0.25)
        assert np.all(np.isfinite(sp)) and sp.min() == 0 and not np.any((sp > 0) & ~(G > 0))
        h = (bs - 1) // 2
        blocks = {(r, c): sp[r - h:r + h + 1, c - h:c + h + 1].sum() for r in range(h, 11, bs) for c in range(h, 13, bs)}
        assert [tuple(x) for x in t] == sorted((k for k, v in blocks.items() if v > 0), key=lambda k: (k[1], k[0]))
        assert np.allclose(amps, [blocks[tuple(x)] for x in t], rtol=1e-14)
    cum = np.array([[1.0, 2.0, 3.0], [4.0, 0.0, 6.0]])
    fp = np.array([[2.0, 0.0, 1.5], [0.0, 0.0, 3.0]])
    G = np.array([[1.0, 1.0, NODATA], [np.nan, 0.0, 1.0]])
    c, f, n = finish(cum, fp, G)
    assert np.array_equal(n, [[0.5, 0.0, NODATA], [NODATA, 0.0, 2.0]])
    assert np.array_equal(c, [[1.0, 2.0, NODATA], [NODATA, 0.0, 6.0]]) and f[0, 2] == f[1, 0] == NODATA


def test_core_passes_settings_and_defaults_through(monkeypatch):
    seen = {}

    def fake(g, src, radius, bs, theta, flow, four, device, rtol, itmax, budget):
        seen.update(dtype=g.dtype, radius=radius, bs=bs, theta=theta, flow=flow, four=four, device=device,
                    rtol=rtol, itmax=itmax, budget=budget)
        z = np.zeros(g.shape)
        return dict(cum=z, fp=z if flow else None, normalized=z if flow else None,
                    targets=np.zeros((1, 2), dtype=np.int64), amps=np.ones(1), scale=np.ones(1),
                    iters=np.arange(1), relres=np.zeros(1), fp_iters=np.arange(1) if flow else None,
                    fp_relres=np.zeros(1) if flow else None, rc=_lib.OK, first_failed=-1, msg="")

    monkeypatch.setattr(S, "solve_omniscape", fake)
    G, Sr = landscape(3, 9, 7)
    out = cb.omniscape_current_maps(G.astype(np.float32), Sr.astype(np.float32), 3, _cfg(True), block_size=3,
                                    source_threshold=0.5, flow_potential=True,
                                    solver=cb.CUDASolver(rtol=1e-8, itmax=77), max_batch_bytes=123)
    assert out.cum_currmap.shape == G.shape and out.flow_potential is not None
    assert seen == dict(dtype=np.float32, radius=3, bs=3, theta=0.5, flow=True, four=True, device=0, rtol=1e-8,
                        itmax=77, budget=123)
    out = cb.omniscape_current_maps(G, Sr.astype(np.float32), 0, {})
    assert out.flow_potential is None and out.normalized_cum_currmap is None and out.fp_iterations is None
    assert seen["dtype"] == np.float64 and (seen["bs"], seen["theta"], seen["flow"]) == (1, 0.0, False)
    assert not seen["four"] and seen["budget"] == 1 << 30


@pytest.mark.parametrize("bad", ["ndim", "shape", "dtype", "radius_negative", "radius_float", "block_even",
                                 "block_zero", "block_float", "theta_negative", "theta_nan", "budget"])
def test_malformed_python_arguments_are_rejected_before_the_library(monkeypatch, bad):
    monkeypatch.setattr(S, "solve_omniscape", lambda *a: pytest.fail("reached the library call"))
    monkeypatch.setattr(_lib, "load", lambda: pytest.fail("loaded the library"))
    G, Sr = landscape(4, 6, 5)
    args, kw = [G, Sr, 2, {}], {}
    if bad == "ndim":
        args[0] = G.ravel()
    elif bad == "shape":
        args[1] = Sr[:4]
    elif bad == "dtype":
        args[0] = np.full(G.shape, "a")
    elif bad == "radius_negative":
        args[2] = -1
    elif bad == "radius_float":
        args[2] = 2.5
    elif bad == "block_even":
        kw["block_size"] = 4
    elif bad == "block_zero":
        kw["block_size"] = 0
    elif bad == "block_float":
        kw["block_size"] = 3.0
    elif bad == "theta_negative":
        kw["source_threshold"] = -0.1
    elif bad == "theta_nan":
        kw["source_threshold"] = np.nan
    else:
        kw["max_batch_bytes"] = 0
    with pytest.raises(ValueError):
        cb.omniscape_current_maps(*args, **kw)


def _call(lib, nr=5, nc=4, g=True, src=True, dtype=1, radius=2, bs=1, theta=0.0, flow=1, fp=True, norm=True,
          cap=None, rtol=1e-6, itmax=100, budget=1 << 20, cum=True, nt=True, targets=True):
    n = max(nr * nc, 1) if 0 < nr < 1 << 16 and 0 < nc < 1 << 16 else 1
    a = np.ones(n)
    maps = [np.full(n, 7.0) for _ in range(3)]
    cap = n if cap is None else cap
    vec = [np.zeros(max(cap, 1), dtype=np.int64) for _ in range(2)] + [np.zeros(max(cap, 1)) for _ in range(2)]
    p = a.ctypes.data_as(ctypes.c_void_p)
    cnt, bad = ctypes.c_int64(3), ctypes.c_int64(5)
    rc = lib.cs_b200_solve_omniscape(nr, nc, p if g else None, p if src else None, dtype, radius, bs, theta, flow, 0,
                                     0, rtol, itmax, budget, _lib._ptr(maps[0]) if cum else None,
                                     _lib._ptr(maps[1]) if fp else None, _lib._ptr(maps[2]) if norm else None, cap,
                                     ctypes.byref(cnt) if nt else None, *[_lib._ptr(v) if targets else None for v in vec],
                                     None, None, None, None, ctypes.byref(bad))
    return rc, bad.value


BAD_ABI = {
    "rows0": dict(nr=0), "cols_negative": dict(nc=-1), "landscape_over_int_max": dict(nr=1 << 20, nc=1 << 20),
    "radius_negative": dict(radius=-1), "window_over_int_max": dict(radius=30000), "block_even": dict(bs=2),
    "block_zero": dict(bs=0), "block_negative": dict(bs=-3), "theta_negative": dict(theta=-0.5),
    "theta_nan": dict(theta=float("nan")), "capacity": dict(cap=19), "capacity_blocks": dict(bs=3, cap=1),
    "null_fp": dict(fp=False), "null_normalized": dict(norm=False), "null_g": dict(g=False),
    "null_src": dict(src=False), "null_cum": dict(cum=False), "null_ntargets": dict(nt=False),
    "null_targets": dict(targets=False), "dtype": dict(dtype=7), "budget": dict(budget=0),
    "rtol": dict(rtol=float("nan")), "itmax": dict(itmax=-1),
}


@pytest.mark.parametrize("case", sorted(BAD_ABI))
def test_bad_abi_arguments_are_rejected_without_a_device(case):
    lib = _lib.load()
    rc, first_failed = _call(lib, **BAD_ABI[case])
    assert rc == _lib.ERR_ARG and first_failed == -1
    assert lib.cs_b200_last_error(None)


def test_no_flow_potential_needs_no_fp_buffers_and_fails_loudly_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    rc, _ = _call(_lib.load(), flow=0, fp=False, norm=False)
    assert rc == _lib.ERR_CUDA
    G, Sr = landscape(5, 6, 5)
    with pytest.raises(cb.B200Unavailable):
        cb.omniscape_current_maps(G, Sr, 2, {}, flow_potential=True)


@pytest.mark.parametrize("kernel", ["k_window_cut", "k_block_targets", "k_omniscape_finish"])
def test_new_instantiations_keep_no_stack(kernel):
    hits = {f: v for f, v in _registers_and_stack().items() if kernel in f}
    assert len(hits) == (6 if kernel == "k_window_cut" else 2)
    for f, (reg, stack) in hits.items():
        assert stack == 0, (f, stack)


# ---------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------
def _check_targets(out, G, Sr, R, bs, theta):
    t, amps = host_targets(G, Sr, bs, theta)
    assert np.array_equal(out.targets, t) and out.targets.dtype == np.int64
    assert np.array_equal(out.amps, amps)                                  # bit for bit
    sums = window_sums(effective(G, Sr, theta), t, R, (bs - 1) // 2)
    ref = scales(amps, sums)
    assert np.array_equal(out.scale == 0, ref == 0)
    assert np.all(np.abs(out.scale - ref) <= 1e-12 * np.abs(ref))
    zero = sums == 0
    assert np.all(out.iterations[zero] == 0)
    return t


TARGET_CASES = {
    "bs1": (37, 53, 1, 0.0), "bs3": (37, 53, 3, 0.0), "bs5": (37, 53, 5, 0.0), "bs7": (37, 53, 7, 0.0),
    "multiple_of_bs3": (30, 45, 3, 0.0), "multiple_of_bs5": (30, 45, 5, 0.0), "threshold": (37, 53, 3, 0.9),
    "one_cell": (1, 1, 1, 0.0), "one_cell_bs3": (1, 1, 3, 0.0), "smaller_than_half_block": (2, 9, 5, 0.0),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(TARGET_CASES))
def test_targets_amps_and_scales_against_the_restatement(case):
    nr, nc, bs, theta = TARGET_CASES[case]
    G, Sr = landscape(7, nr, nc)
    Sr = np.where(Sr > 0, Sr + 0.25, Sr)      # no near-zero amps: those right-hand sides stop on atol, not rtol
    G[-1, -1] = NODATA if nr > 1 else G[-1, -1]
    if nr > 2:
        Sr[0, 0], Sr[5, 5], Sr[10, 7], Sr[12, 30] = np.nan, -2.0, np.inf, 4.0
        G[12, 30] = NODATA                                 # a source on NODATA is never injected
    R = 3
    out = cb.omniscape_current_maps(G, Sr, R, {}, block_size=bs, source_threshold=theta)
    t = _check_targets(out, G, Sr, R, bs, theta)
    if case == "smaller_than_half_block":
        assert len(t) == 0 and len(out.iterations) == 0
        c, _, _ = finish(np.zeros(G.shape), None, G)
        assert np.array_equal(out.cum_currmap, c) and np.any(c == NODATA)
    if case == "one_cell" and G[0, 0] > 0 and Sr[0, 0] > 0:
        assert len(t) == 1 and out.scale[0] == 0 and np.all(out.cum_currmap[G > 0] == 0)


@pytest.mark.gpu
@pytest.mark.parametrize("bs", [1, 3, 5])
@pytest.mark.parametrize("four", [False, True])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_maps_bit_identical_to_the_host_composition(dtype, four, bs):
    G, Sr = landscape(11, 41, 36)
    G, Sr = G.astype(dtype), Sr.astype(dtype)
    R, theta, cfg = 5, 0.1, _cfg(four)
    out = cb.omniscape_current_maps(G, Sr, R, cfg, block_size=bs, source_threshold=theta, flow_potential=True)
    t = _check_targets(out, G, Sr, R, bs, theta)
    cum, fp, norm, batch, fp_batch = host_maps(G, Sr, t, out.scale, R, bs, theta, cfg, dtype, True)
    assert out.cum_currmap.max() > 0 and out.flow_potential.max() > 0
    assert np.array_equal(out.cum_currmap, cum)
    assert np.array_equal(out.flow_potential, fp)
    assert np.array_equal(out.normalized_cum_currmap, norm)
    assert np.array_equal(out.iterations, batch.iterations) and np.array_equal(out.relres, batch.relres)
    assert np.array_equal(out.fp_iterations, fp_batch.iterations) and np.array_equal(out.fp_relres, fp_batch.relres)
    mask = np.isnan(G.astype(np.float64)) | (G == NODATA)
    assert mask.any() and np.all(out.cum_currmap[mask] == NODATA) and np.all(out.cum_currmap[~mask] >= 0)
    bare = cb.omniscape_current_maps(G, Sr, R, cfg, block_size=bs, source_threshold=theta)
    assert np.array_equal(bare.cum_currmap, cum) and bare.flow_potential is None


@pytest.mark.gpu
@pytest.mark.parametrize("four", [False, True])
def test_block_size_one_is_the_moving_window_map_of_the_effective_strengths(four):
    G, Sr = landscape(12, 33, 29)
    R, theta, cfg = 4, 0.3, _cfg(four)
    out = cb.omniscape_current_maps(G, Sr, R, cfg, source_threshold=theta, flow_potential=True)
    sp = effective(G, Sr, theta)
    mw = cb.moving_window_current_map(G, sp, out.targets, R, cfg, source_scale=out.scale)
    ones = cb.moving_window_current_map(np.ones_like(G), sp, out.targets, R, cfg, source_scale=out.scale)
    cum, fp, _ = finish(mw.current, ones.current, G)
    assert np.array_equal(out.cum_currmap, cum) and np.array_equal(out.flow_potential, fp)
    assert np.array_equal(out.iterations, mw.iterations) and np.array_equal(out.fp_iterations, ones.iterations)


@pytest.mark.gpu
def test_windows_without_sources_outside_the_block_add_nothing():
    """sources only in isolated 5 x 5 blocks with radius 2: every disc lies in its block, so every window
    sum is 0 -- scale 0, no iterations, zero maps except the mask"""
    G, _ = landscape(13, 25, 30)
    Sr = np.zeros_like(G)
    Sr[0:5, 0:5] = Sr[10:15, 20:25] = 1.0
    G[2, 2] = G[12, 22] = 1.0
    out = cb.omniscape_current_maps(G, Sr, 2, {}, block_size=5, flow_potential=True)
    assert [tuple(t) for t in out.targets] == [(2, 2), (12, 22)]
    assert np.all(out.scale == 0) and np.all(out.iterations == 0) and np.all(out.fp_iterations == 0)
    c, f, n = finish(np.zeros(G.shape), np.zeros(G.shape), G)
    assert np.array_equal(out.cum_currmap, c) and np.array_equal(out.flow_potential, f)
    assert np.array_equal(out.normalized_cum_currmap, n)


@pytest.mark.gpu
def test_batch_splits_and_repeats_are_bit_identical():
    G, Sr = landscape(14, 60, 45)
    R, bs = 6, 3
    kw = dict(block_size=bs, flow_potential=True)
    whole = cb.omniscape_current_maps(G, Sr, R, {}, max_batch_bytes=1 << 40, **kw)
    assert len(whole.targets) > 100
    one = S.advanced_batch_bytes((2 * R + 1) ** 2, 8, False)
    for budget in (1, 2 * one, 7 * 2 * one, 1 << 40):
        other = cb.omniscape_current_maps(G, Sr, R, {}, max_batch_bytes=budget, **kw)
        for a in ("cum_currmap", "flow_potential", "normalized_cum_currmap", "targets", "amps", "scale",
                  "iterations", "relres", "fp_iterations", "fp_relres"):
            assert np.array_equal(getattr(whole, a), getattr(other, a)), (budget, a)


@pytest.mark.gpu
def test_itmax_fails_the_gate_naming_the_target_and_the_window_kind():
    G, Sr = landscape(15, 40, 40, holes=0.0)
    G[np.isnan(G) | (G <= 0)] = 1.0
    Sr[:] = 1.0
    G[2, 2] = NODATA                                  # target 0 has no ground; its flow-potential window does
    solver = cb.CUDASolver(itmax=2)
    with pytest.raises(cb.SolverResidualError, match=r"for target 0, flow-potential window") as e:
        cb.omniscape_current_maps(G, Sr, 10, {}, block_size=5, flow_potential=True, solver=solver)
    assert e.value.window == 0
    with pytest.raises(cb.SolverResidualError, match=r"for target 1, conductance window") as e:
        cb.omniscape_current_maps(G, Sr, 10, {}, block_size=5, solver=solver)
    assert e.value.window == 1
    res = S.solve_omniscape(G, Sr, 10, 5, 0.0, True, False, 0, 1e-6, 2, 1 << 30)
    assert res["rc"] == _lib.ERR_RESIDUAL and res["first_failed"] == 0
    assert res["iters"][0] == 0 and np.all(res["iters"][1:] == 2) and np.all(res["fp_iters"] == 2)
    assert np.all(np.isfinite(res["cum"])) and res["cum"].max() > 0 and res["fp"].max() > 0

"""A whole Omniscape job through omniscape_current_maps (cs_b200_solve_omniscape): block targets, window
sources normalised, conductance and flow-potential windows cut, solved and summed on the device.  Prints
one JSON line.

(a) The landscape of run_moving_windows.py -- 1200 x 1200, resistance exp(N(0, 1)) (seed 42), 3 % NODATA
    (seed 44) -- with source strength = conductance on the valid cells, threshold 0, radius 50, block sizes
    5 and 9, flow potential off and on: targets, end-to-end seconds, windows/s.
(b) The 3163 x 3163 bench raster (R ~ U[1, 10], seed 42), sources = conductance, radius 50, block 15, flow
    potential on.
(c) Block 9 on (a) with flow potential, through the host stack path: numpy targets, amps and window
    scales, host-cut windows with the block zeroed, one compute_omniscape_currents call per map, host
    placement, normalisation and mask.  Its time and its largest relative difference from the device maps
    (the host sums amps and window sums in another order, so its scales differ in the last bits).
(d) Device time per kernel of the block-9 flow-potential call (torch.profiler, a run of its own)."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import circuitscape_b200 as cb

from run_moving_windows import gpu_info, landscape   # noqa: E402

RADIUS, BENCH = 50, 3163
KERNELS = ("k_advanced_batch", "k_window_cut", "k_block_targets", "k_omniscape_finish", "k_window_accumulate",
           "k_window_tiles", "k_tile_bounds", "DeviceRadixSort", "DeviceSelect")


def timed(f):
    t0 = time.perf_counter()
    res = f()
    return time.perf_counter() - t0, res


def stack_path(g, src, bs):
    """the same job with the host doing Omniscape's work and compute_omniscape_currents the solves"""
    nr, nc = g.shape
    h, W = (bs - 1) // 2, 2 * RADIUS + 1
    sp = np.where((g > 0) & (src > 0) & np.isfinite(src), src, 0.0)
    ni, nj = (nr - 1 - h) // bs + 1, (nc - 1 - h) // bs + 1
    blk = np.zeros((ni * bs, nj * bs))
    blk[:min(nr, ni * bs), :min(nc, nj * bs)] = sp[:ni * bs, :nj * bs]
    amps = blk.reshape(ni, bs, nj, bs).sum(axis=(1, 3)).T.ravel()          # j outer, i inner
    jj, ii = np.meshgrid(np.arange(nj), np.arange(ni), indexing="ij")
    t = np.stack([h + ii.ravel() * bs, h + jj.ravel() * bs], 1)[amps > 0]
    amps = amps[amps > 0]
    d = np.arange(-RADIUS, RADIUS + 1)
    disc = d[:, None] ** 2 + d[None, :] ** 2 <= RADIUS ** 2
    out_blk = (np.abs(d)[:, None] > h) | (np.abs(d)[None, :] > h)
    pad = lambda a: np.pad(a, RADIUS)
    view = lambda a: np.lib.stride_tricks.sliding_window_view(a, (W, W))[t[:, 0], t[:, 1]]
    ss = view(pad(sp)) * (disc & out_blk)
    sums = ss.sum(axis=(1, 2))
    scale = np.where(sums > 0, amps / np.where(sums > 0, sums, 1.0), 0.0)
    ss *= scale[:, None, None]
    maps = []
    for flow in (False, True):
        if flow:
            gs = view(pad(np.ones_like(g))) * disc
        else:
            gs = view(pad(np.where(g > 0, g, 0.0))) * disc
        ns = np.zeros_like(gs)
        ns[:, RADIUS, RADIUS] = np.where(gs[:, RADIUS, RADIUS] > 0, np.inf, 0.0)
        cur = cb.compute_omniscape_currents(gs, ss, ns, {}).currents
        del gs, ns
        m = np.zeros((nr + 2 * RADIUS, nc + 2 * RADIUS))
        for c, (r, q) in zip(cur, t):
            m[r:r + W, q:q + W] += c
        maps.append(m[RADIUS:-RADIUS, RADIUS:-RADIUS])
    cum, fp = maps
    norm = np.where(fp > 0, cum / np.where(fp > 0, fp, 1.0), 0.0)
    mask = np.isnan(g) | (g == -9999.0)
    return [np.where(mask, -9999.0, a) for a in (cum, fp, norm)], t


def kernel_ms(g, src, bs):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        cb.omniscape_current_maps(g, src, RADIUS, {}, block_size=bs, flow_potential=True)
    ms = {k: 0.0 for k in KERNELS}
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key:
                ms[k] += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
    return {k: round(v, 3) for k, v in ms.items()}


def main():
    name, power = gpu_info()
    res = {"gpu": name, "power_limit_w": power, "radius": RADIUS}
    g = landscape()
    src = np.where(g > 0, g, 0.0)
    cb.omniscape_current_maps(g[:200, :200], src[:200, :200], RADIUS, {}, block_size=25, flow_potential=True)
    for bs in (5, 9):
        for flow in (False, True):
            s, out = timed(lambda: cb.omniscape_current_maps(g, src, RADIUS, {}, block_size=bs, flow_potential=flow))
            nt = len(out.targets)
            res[f"a_bs{bs}_fp{int(flow)}"] = {"targets": nt, "s": round(s, 3),
                                             "windows_per_s": round(nt * (2 if flow else 1) / s, 1),
                                             "iters_p50": float(np.percentile(out.iterations, 50)),
                                             "relres_max": float(out.relres.max())}
            if bs == 9 and flow:
                dev9 = out
    gb = 1.0 / np.random.default_rng(42).uniform(1.0, 10.0, size=(BENCH, BENCH))
    s, big = timed(lambda: cb.omniscape_current_maps(gb, gb, RADIUS, {}, block_size=15, flow_potential=True,
                                                     max_batch_bytes=4 << 30))
    res["b_bench_bs15_fp1"] = {"targets": len(big.targets), "s": round(s, 3),
                               "windows_per_s": round(2 * len(big.targets) / s, 1),
                               "iters_p50": float(np.percentile(big.iterations, 50)),
                               "fp_iters_p50": float(np.percentile(big.fp_iterations, 50))}
    s, (host, t) = timed(lambda: stack_path(g, src, 9))
    dev = (dev9.cum_currmap, dev9.flow_potential, dev9.normalized_cum_currmap)
    res["c_stack_bs9_fp1"] = {
        "s": round(s, 3), "device_s": res["a_bs9_fp1"]["s"], "speedup": round(s / res["a_bs9_fp1"]["s"], 2),
        "same_targets": bool(np.array_equal(t, dev9.targets)),
        "max_rel_diff": [float(np.abs(a - b).max() / np.abs(b).max()) for a, b in zip(host, dev)],
        "bit_identical": [bool(np.array_equal(a, b)) for a, b in zip(host, dev)]}
    kms = kernel_ms(g, src, 9)
    base = kms["k_advanced_batch"]
    res["d_kernel_ms_bs9_fp1"] = kms
    res["d_share_of_k_advanced_batch"] = {k: round(v / base, 5) for k, v in kms.items() if base > 0}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()

"""Omniscape's moving-window loop over one landscape through moving_window_current_map (windows cut and
currents summed on the device, cs_b200_solve_moving_windows) and through the stack path
(compute_omniscape_currents on host-cut square windows, then host placement).  Prints one JSON line.

(a) The landscape and targets of run_advanced_batch.py -- 1200 x 1200, resistance exp(N(0, 1)) (seed 42),
    3 % NODATA (seed 44), 2048 interior targets and 64 within 50 cells of the edge drawn from the valid cells
    (seed 45) -- with centred square windows of radius 50 (101 x 101, no disc), unit sources on every valid
    cell, a direct (Inf) ground at the target, default settings, fp64.  Both paths end to end (median of 3),
    the device time of the new path's kernels (torch.profiler, a run of its own) and max |cum difference|.
(b) Capacity: the 3163 x 3163 bench raster (R ~ U[1, 10], seed 42), radius 50 with the disc, one target
    every 8th cell in each direction, unit sources, Inf ground at the target, through the new path only:
    time, windows/s and peak host RSS."""
import json
import os
import resource
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

import circuitscape_b200 as cb
from circuitscape_b200 import solver as S

SIZE, RADIUS, N_INNER, N_EDGE = 1200, 50, 2048, 64
BENCH, STRIDE = 3163, 8
KERNELS = ("k_advanced_batch", "k_window_cut", "k_window_accumulate", "k_window_tiles", "k_tile_bounds",
           "DeviceRadixSort")


def landscape():
    r = np.exp(np.random.default_rng(42).normal(size=(SIZE, SIZE)))
    g = 1.0 / r
    g[np.random.default_rng(44).random(g.shape) < 0.03] = -9999.0
    return g


def targets(g):
    rng = np.random.default_rng(45)
    rows, cols = np.nonzero(g > 0)
    inner = (rows >= RADIUS) & (rows < SIZE - RADIUS) & (cols >= RADIUS) & (cols < SIZE - RADIUS)
    pick = np.concatenate([rng.choice(np.nonzero(inner)[0], N_INNER, replace=False),
                           rng.choice(np.nonzero(~inner)[0], N_EDGE, replace=False)])
    return np.stack([rows[pick], cols[pick]], 1)


def gpu_info():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        power = None
    return name, power


def stack_path(g, src, t, budget):
    """square windows cut on the host, one compute_omniscape_currents call, placement on the host"""
    W = 2 * RADIUS + 1
    gp = np.pad(np.where(g > 0, g, 0.0), RADIUS)
    sp = np.pad(src, RADIUS)
    gs = np.lib.stride_tricks.sliding_window_view(gp, (W, W))[t[:, 0], t[:, 1]]
    ss = np.lib.stride_tricks.sliding_window_view(sp, (W, W))[t[:, 0], t[:, 1]]
    ns = np.zeros_like(gs)
    ns[:, RADIUS, RADIUS] = np.where(gs[:, RADIUS, RADIUS] > 0, np.inf, 0.0)
    out = cb.compute_omniscape_currents(gs, ss, ns, {}, max_batch_bytes=budget)
    cum = np.zeros(np.add(g.shape, 2 * RADIUS))
    for cur, (r, c) in zip(out.currents, t):
        cum[r:r + W, c:c + W] += cur
    return cum[RADIUS:-RADIUS, RADIUS:-RADIUS]


def median_time(f, reps=3):
    ts, res = [], None
    for _ in range(reps):
        t0 = time.perf_counter()
        res = f()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), res


def kernel_ms(g, src, t, budget):
    """device time per kernel of one moving_window_current_map call, from torch.profiler's CUDA activities"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        cb.moving_window_current_map(g, src, t, RADIUS, {}, circular=False, max_batch_bytes=budget)
    ms = {k: 0.0 for k in KERNELS}
    for e in prof.key_averages():
        for k in KERNELS:
            if k in e.key:
                ms[k] += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3
    return {k: round(v, 3) for k, v in ms.items()}


def rss_mb():
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024.0


def main():
    name, power = gpu_info()
    # (b) capacity, first, so that the peak RSS is this call's and not the stack path's of (a)
    gb = 1.0 / np.random.default_rng(42).uniform(1.0, 10.0, size=(BENCH, BENCH))
    sb = np.ones_like(gb)
    rr, cc = np.meshgrid(np.arange(0, BENCH, STRIDE), np.arange(0, BENCH, STRIDE), indexing="ij")
    tb = np.stack([rr.ravel(), cc.ravel()], 1)
    budget_b = 4 << 30
    cb.moving_window_current_map(gb[:200, :200], sb[:200, :200], tb[:4], RADIUS, {})      # module load
    rss0 = rss_mb()
    t0 = time.perf_counter()
    big = cb.moving_window_current_map(gb, sb, tb, RADIUS, {}, circular=True, max_batch_bytes=budget_b)
    t_big = time.perf_counter() - t0
    rss_b = rss_mb()

    # (a)
    g = landscape()
    src = np.where(g > 0, 1.0, 0.0)
    t = targets(g)
    nwin = len(t)
    budget = S.advanced_batch_bytes((2 * RADIUS + 1) ** 2, 8, False) * nwin      # the whole job in one batch
    cb.moving_window_current_map(g, src, t[:8], RADIUS, {}, circular=False)       # module load
    stack_path(g, src, t[:8], budget)
    t_new, new = median_time(lambda: cb.moving_window_current_map(g, src, t, RADIUS, {}, circular=False,
                                                                   max_batch_bytes=budget))
    t_old, old = median_time(lambda: stack_path(g, src, t, budget))
    kms = kernel_ms(g, src, t, budget)

    print(json.dumps({
        "gpu": name, "power_limit_w": power,
        "a_windows": nwin, "a_window_cells": (2 * RADIUS + 1) ** 2,
        "a_device_s": round(t_new, 4), "a_device_windows_per_s": round(nwin / t_new, 1),
        "a_stack_s": round(t_old, 4), "a_stack_windows_per_s": round(nwin / t_old, 1),
        "a_speedup": round(t_old / t_new, 2),
        "a_max_abs_cum_diff": float(np.abs(new.current - old).max()),
        "a_cum_max": float(new.current.max()),
        "a_kernel_ms": kms,
        "a_iters_p50": float(np.percentile(new.iterations, 50)), "a_relres_max": float(new.relres.max()),
        "b_landscape": [BENCH, BENCH], "b_windows": len(tb), "b_budget_bytes": budget_b,
        "b_s": round(t_big, 3), "b_windows_per_s": round(len(tb) / t_big, 1),
        "b_peak_rss_mb": round(rss_b, 1), "b_peak_rss_before_call_mb": round(rss0, 1),
        "b_iters_p50": float(np.percentile(big.iterations, 50)), "b_relres_max": float(big.relres.max()),
        "b_cum_max": float(big.current.max()),
    }), flush=True)


if __name__ == "__main__":
    main()

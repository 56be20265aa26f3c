#!/usr/bin/env python
"""Where one AMG-PCG iteration of the bench workload goes, kernel by kernel.

Runs `bench_cg_iter(8, reps)` on the `bench.py` operator (3163 x 3163 synthetic raster, seed 42, default
CUDASolver: fp64 CG, mixed fp32 V-cycle) under torch.profiler with CUDA activities and prints one JSON line:
per kernel launch slot of the iteration (name + "#i/m" when a kernel is launched m times per iteration, in
launch order), the launches, the average device time, the share of the iteration and -- for the finest-level
kernels -- the bytes the kernel moves, computed from the level shapes by the formulas below, the rate and the
fraction of the HBM peak.  The card name and power limit are read with a read-only nvidia-smi query.

  python profiles/run_iteration_breakdown.py [--reps 20] [--prolong-form strip|tile] [--out FILE]

--prolong-form tile: byte formula of the 128 x 8-tile fused prolongation kernel (x1 rebuilt on a 130 x 10 halo
tile, b and 1/diag read in both phases); strip: the streaming kernel (x1 built once per row, 2 halo rows per
strip of RPS rows, b and 1/diag read once).
"""
import argparse
import ctypes as C
import json
import os
import re
import subprocess
import sys
from collections import defaultdict

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

PEAK_GBS = 3350.0          # H100 SXM data sheet, HBM3
KT = 8


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, pl = [s.strip() for s in out[0].split(",")]
        return {"name": name, "power_limit": pl}
    except Exception as e:  # noqa: BLE001
        return {"name": None, "power_limit": None, "error": str(e)}


def level_dims(f):
    """(rows, cols, nnz) of A, P, R per level through the C ABI (no download)."""
    out = []
    for l in range(64):
        lev = {}
        for name, which in (("A", 0), ("P", 1), ("R", 2)):
            nr, nc, nnz = C.c_int64(), C.c_int64(), C.c_int64()
            om, win = C.c_double(), C.c_int()
            rc = f._lib.cs_b200_level_info(f._h, l, which, C.byref(nr), C.byref(nc), C.byref(nnz),
                                           C.byref(om), C.byref(win))
            lev[name] = (nr.value, nc.value, nnz.value, win.value) if rc == 0 else None
        if lev["A"] is None:
            break
        slots = C.c_int()
        f._lib.cs_b200_level_stencil(f._h, l, C.byref(slots))
        lev["A_stencil_slots"] = slots.value
        out.append(lev)
    return out


def short(name):
    """'void csb::(anonymous namespace)::k_x<float, 8, 5, 3>(args...)' -> 'k_x<float,8,5,3>'"""
    name = name.replace("(anonymous namespace)::", "").replace("csb::", "")
    name = re.sub(r"^void ", "", name)
    depth, cut = 0, len(name)
    for i, ch in enumerate(name):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0:
            cut = i
            break
    return name[:cut].replace(" ", "")


def finest_bytes(levels, prolong_form):
    """Bytes moved per launch by the finest-level kernels of one mixed-cycle iteration, k = 8.
    Panels: n x 8 of fp64 (64 B per row) or fp32 (32 B per row).  Diagonals: 9 per row (stencil form), or with
    the half form (level 0 reports 5 slots) 5 per row (3 more for the column left of each tile) plus the 2-row halo
    of each panel slot (RPP + 2 rows for RPP, RPP = 64 in fp64, 128 in fp32) or prolongation strip.  Level 0 reports the fp32 copy the V-cycle runs on; the
    fp64 operator of the CG step is the same matrix before rounding, so it takes the form the fp32 copy takes
    (rounding keeps bit-equal entries bit-equal; the reverse is not guaranteed).
    Restriction records: nnz(R) (4 B value + 2 B local column) + 2 B row offsets per coarse row,
    reading the fp32 residual panel and writing the coarse right-hand side."""
    n = levels[0]["A"][0]
    n1 = levels[1]["A"][0] if len(levels) > 1 else 0
    nnz_r = levels[0]["R"][2] if levels[0]["R"] else 0
    d64, d32 = 8 * KT, 4 * KT
    rps = 256 // 2 - 2                                   # fp32, k = 8: 128-row strips less the 2 halo rows
    half = levels[0].get("A_stencil_slots") == 5
    # diagonals per row streamed by the pipelined kernels; half: 5 runs per computed column and 3 for the column
    # left of each 16-column tile
    dg64 = (5 + 3 / 16) * 66 / 64 if half else 9
    dg32 = (5 + 3 / 16) * 130 / 128 if half else 9
    if prolong_form == "tile":
        halo = (130 * 10) / (128 * 8)                     # phase-1 streams of a 128 x 8 tile with its 1-cell halo
        # phase 1 (halo-inflated): b, 1/diag, ELL-4 (4 x (4 + 4) B), y gathers; phase 2: 9 diagonals, b, 1/diag, z
        prol = n * (halo * (d32 + 4 + 32 + d32) + 9 * 4 + d32 + 4 + d32)
    else:
        halo = (rps + 2) / rps
        prol = n * (halo * (d32 + 4 + 32 + d32) + (5 * halo if half else 9) * 4 + d32)
    # the stencil kernels under either name: k_stencil[_cg]_pipe (shared-memory pipeline) or the register-gather
    # form (CS_B200_NO_STENCIL_PIPE)
    # (the pipelined ones carry a last template argument: the half form or not)
    cg_step = n * (dg64 * 8 + d32 + 3 * d64 + 1.5 * d64)
    cg_step_no_ap = cg_step - n * d64
    res0 = n * (dg32 * 4 + d32 + 4 + d32)
    # fused residual sweep (strips of 62 rows): p and the 5 fp64 upper runs on rows -2 ... 63, r and the fp32 1/diag
    # on rows -1 ... 62 in; r, R32, T32 out (the fp32 diagonals are the fp64 ones rounded on chip)
    ru = n * ((d64 + 5 * 8) * 66 / 62 + (d64 + 4) * 64 / 62 + d64 + d32 + d32)
    return {
        "k_stencil<double,8,1>": n * (9 * 8 + d64 + d64),               # CG SpMM: diagonals, P, AP
        "k_stencil_pipe<double,8,1,*>": n * (dg64 * 8 + d64 + d64),
        # residual gate: diagonals, X, B in, residual out
        "k_stencil<double,8,2>": n * (9 * 8 + 3 * d64),
        "k_stencil_pipe<double,8,2,*>": n * (dg64 * 8 + 3 * d64),
        # fused CG step: diagonals, Z32, p_{it-1} in, AP, p_it out; X in/out + p_{it-2} in every other step
        "k_stencil_cg<double,8,float>": cg_step,
        "k_stencil_cg_pipe<double,8,float,*,true>": cg_step,
        "k_stencil_cg_pipe<double,8,float,*,false>": cg_step_no_ap,                # A p not stored
        "k_stencil_res_update<double,float,8>": ru,
        "k_cg_update_r0<double,8,float>": n * (d64 + 8 + 2 * d64 + d32),  # AP, 1/diag, R in/out, R32
        "k_stencil<float,8,7>#1": res0,                                 # residual with implicit x0: diagonals, b, 1/diag, t
        "k_stencil_pipe<float,8,7,*>#1": res0,
        "k_spmm_win<float,8,0,*>#1": nnz_r * 6 + n1 * 2 + n * d32 + n1 * d32,
        "k_stencil_prolong_jacobi<float,8,5,*>": prol,
        "k_cg_update_xp2<double,8,float>": n * (d32 + 4 * d64),         # Z32, X in/out, P in/out
    }, {"n": n, "n1": n1, "nnz_R0": nnz_r, "prolong_halo_factor": halo,
        "level0_stencil_slots": levels[0].get("A_stencil_slots")}


def match_bytes(key, table):
    for pat, b in table.items():
        base, _, occ = pat.partition("#")
        rx = "^" + re.escape(base).replace(r"\*", r"[^,>]+") + "$"
        name, _, slot = key.partition("#")
        if re.match(rx, name) and (not occ or (slot or "1").split("/")[0] == occ):
            return b
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=3163)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--prolong-form", default="strip", choices=["strip", "tile"])
    ap.add_argument("--out", default="")
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import circuitscape_b200 as cb
    from circuitscape_b200 import graph
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    L, _ = graph.synthetic_raster_laplacian(a.rows, a.rows, seed=42)
    with cb.construct_cholesky_factor(L, cb.CUDASolver()) as f:
        levels = level_dims(f)
        f.bench_cg_iter(KT, reps=5)                                    # warm-up
        ms_iter = f.bench_cg_iter(KT, reps=a.reps)                      # un-instrumented, CUDA events
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            f.bench_cg_iter(KT, reps=a.reps)
            torch.cuda.synchronize()
    evs = [e for e in prof.events() if e.device_type.name == "CUDA" and "memcpy" not in e.name.lower()
           and "memset" not in e.name.lower()]
    evs.sort(key=lambda e: e.time_range.start)
    # one iteration starts with the fp64 CG SpMM (or the fused CG step); the bench call runs 3 warm-up iterations +
    # reps, plus set-up kernels
    starts = [i for i, e in enumerate(evs) if short(e.name).startswith(("k_stencil<double,8,1>", "k_stencil_cg<double,8,",
                                                                        "k_stencil_pipe<double,8,1,",
                                                                        "k_stencil_cg_pipe<double,8,",
                                                                        "k_spmm_win<double,8,1,"))]
    iters = [evs[starts[j]:starts[j + 1]] for j in range(len(starts) - 1)]
    iters = iters[3:] if len(iters) > a.reps else iters             # drop the warm-up iterations
    if len(starts) > 1:
        last = evs[starts[-1]:]
        iters.append(last[:len(iters[0])] if iters else last)
    agg = defaultdict(lambda: [0, 0.0])
    for it in iters:
        names = [short(e.name) for e in it]
        tot = defaultdict(int)
        for nm in names:
            tot[nm] += 1
        seen = defaultdict(int)
        for e, nm in zip(it, names):
            seen[nm] += 1
            key = nm if tot[nm] == 1 else f"{nm}#{seen[nm]}/{tot[nm]}"
            agg[key][0] += 1
            agg[key][1] += e.time_range.elapsed_us()
    niter = max(1, len(iters))
    table, shape = finest_bytes(levels, a.prolong_form)
    if any(k.startswith("k_stencil_res_update<") for k in agg):
        # the fused sweep forms the level-0 residual: the first SP_RES0 launch of the iteration is level 1's
        table = {k: v for k, v in table.items() if not k.startswith(("k_stencil<float,8,7>", "k_stencil_pipe<float,8,7,"))}
    sum_us = sum(v[1] for v in agg.values()) / niter
    rows = {}
    for key, (cnt, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        avg = us / cnt
        r = {"launches_per_iter": cnt / niter, "avg_us": avg, "share": (us / niter) / sum_us}
        b = match_bytes(key, table)
        if b is not None:
            r.update({"bytes": b, "GB/s": b / (avg * 1e-6) / 1e9, "frac_of_peak": b / (avg * 1e-6) / 1e9 / PEAK_GBS})
        rows[key] = r
    res = {"card": card(), "rows": a.rows, "k": KT, "iterations_profiled": niter,
           "iter_ms_events": ms_iter, "iter_ms_kernel_sum": sum_us / 1e3, "peak_GBs": PEAK_GBS,
           "peak_source": "H100 SXM data sheet (HBM3)", "prolong_form": a.prolong_form, "shape": shape,
           "levels": [{k: v for k, v in lev.items()} for lev in levels], "kernels": rows}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

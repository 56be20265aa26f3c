#!/usr/bin/env python
"""What a panel of the bench workload spends outside its PCG loop, pass by pass, with the panel-end passes of
`panel_ends` (cs_b200.cu) on and off (CS_B200_NO_FUSED_PANEL_ENDS).

Runs one `solve_pairs` of 16 columns (two panels of 8, accumulate on, as `bench.py` runs them) on the `bench.py`
operator (3163 x 3163 synthetic raster, seed 42, default CUDASolver: fp64 CG, mixed fp32 V-cycle) under
torch.profiler with CUDA activities, once per setting of the switch, each in a child process of its own, after one
un-profiled warm-up call of the same shape.  From the device trace it reports, per panel:
  start  every device pass (kernel, memset, copy) from the panel's first one to the WHILE-loop condition kernel
         that opens its PCG loop -- the right-hand side, the fills, r / r32 and the start-up V-cycle;
  end    every pass after the loop's last condition kernel up to the end of k_cur_acc_dia -- the pending x
         update, the residual gate, the pair extraction and the two node-current passes;
with device time per pass and the per-panel sums (busy time: the sum of the pass durations).  The card name and
power limit are read in the same run with a read-only nvidia-smi query.

  python profiles/run_panel_ends.py [--rows 3163] [--pairs 16] [--out FILE]
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SWITCH = "CS_B200_NO_FUSED_PANEL_ENDS"


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, pl = [s.strip() for s in out[0].split(",")]
        return {"name": name, "power_limit": pl}
    except Exception as e:  # noqa: BLE001
        return {"name": None, "power_limit": None, "error": str(e)}


def short(name):
    """'void csb::k_x<double, 8, 2, true>(args...)' -> 'k_x<double,8,2,true>'; memsets and copies as named."""
    name = name.replace("(anonymous namespace)::", "").replace("csb::", "")
    name = re.sub(r"^void ", "", name)
    depth, cut = 0, len(name)
    for i, ch in enumerate(name):
        if ch == "<":
            depth += 1
        elif ch == ">":
            depth -= 1
        elif ch == "(" and depth == 0 and i > 0:
            cut = i
            break
    return name[:cut].replace(" ", "")


def child(rows, npairs, trace_path):
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import circuitscape_b200 as cb
    from circuitscape_b200 import graph

    L, _ = graph.synthetic_raster_laplacian(rows, rows, seed=42)
    npts = 2
    while npts * (npts - 1) // 2 < 128:                # bench.py's 128 pairs; the first npairs of them
        npts += 1
    src, dst = graph.all_pairs(graph.focal_nodes(L.shape[0], npts, seed=7), limit=128)
    src, dst = src[:npairs], dst[:npairs]
    with cb.construct_cholesky_factor(L, cb.CUDASolver()) as f:
        f.reset_currents()
        f.solve_pairs(src, dst, accumulate=True)           # warm-up: modules, graphs, smem attributes
        torch.cuda.synchronize()
        f.reset_currents()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            out = f.solve_pairs(src, dst, accumulate=True)
            torch.cuda.synchronize()
        prof.export_chrome_trace(trace_path)
        np.save(trace_path + ".R.npy", np.asarray(out["R"]))


def panels(trace_path):
    with open(trace_path) as fh:
        ev = json.load(fh)["traceEvents"]
    dev = sorted((e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memset", "gpu_memcpy")),
                 key=lambda e: e["ts"])
    out, cur = [], []
    for e in dev:                                           # a panel ends with its k_cur_acc_dia
        cur.append(e)
        if short(e["name"]).startswith("k_cur_acc_dia"):
            out.append(cur)
            cur = []
    res = []
    for p in out:
        conds = [i for i, e in enumerate(p) if short(e["name"]).startswith("k_loop_cond")]
        if not conds:
            raise SystemExit("no k_loop_cond in a panel: the device WHILE loop did not run")
        start, end = p[:conds[0]], p[conds[-1] + 1:]

        def passes(seg):
            agg = defaultdict(lambda: [0, 0.0])
            for e in seg:
                k = short(e["name"])
                agg[k][0] += 1
                agg[k][1] += e["dur"] / 1000.0
            return [{"pass": k, "launches": n, "ms": round(ms, 4)} for k, (n, ms) in agg.items()]

        res.append({"start_ms": round(sum(e["dur"] for e in start) / 1000.0, 4),
                    "end_ms": round(sum(e["dur"] for e in end) / 1000.0, 4),
                    "loop_cond_kernels": len(conds),
                    "start": passes(start), "end": passes(end)})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=3163)
    ap.add_argument("--pairs", type=int, default=16)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        child(a.rows, a.pairs, a.child)
        return
    import numpy as np
    result = {"card": card(), "rows": a.rows, "pairs": a.pairs, "settings": {}}
    with tempfile.TemporaryDirectory() as tmp:
        R = {}
        for name, off in (("on", False), ("off", True)):
            env = dict(os.environ)
            env.pop(SWITCH, None)
            if off:
                env[SWITCH] = "1"
            trace = os.path.join(tmp, f"{name}.json")
            subprocess.run([sys.executable, os.path.abspath(__file__), "--rows", str(a.rows), "--pairs", str(a.pairs),
                            "--child", trace], env=env, check=True, cwd=ROOT)
            ps = panels(trace)
            R[name] = np.load(trace + ".R.npy")
            result["settings"][name] = {
                "start_ms_per_panel": round(sum(p["start_ms"] for p in ps) / len(ps), 4),
                "end_ms_per_panel": round(sum(p["end_ms"] for p in ps) / len(ps), 4),
                "panels": ps}
        result["R_identical"] = bool(np.array_equal(R["on"], R["off"]))
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

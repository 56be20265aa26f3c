"""The host front end against CUDASolver(front_end_on_device=True) on the 3163 x 3163 bench raster: raster advanced
mode (run_advanced_raster.py's finite / direct / walls32 inputs), one-to-all and all-to-one at P = 16 and 64
(run_onetoall.py's points, cumulative map only) and 16 focal regions of 10 x 10 (run_focal_regions.py's regions).

Every case runs the switch off, on, off, on (`--rounds N`: N pairs), each in a child process of its own, so that
each run's peak host RSS is its own.  Per run: end-to-end host-clock seconds, split into setup (handle creates,
set_grounds), plan (components and plan_advanced, the device front end's own calls), solve (the column entries
and the current read-back) and host (the rest: node map, graph, labels, node values, output maps); ru_maxrss of the child; and whether every output array is bit-identical to the first
switch-off run.  Prints one JSON line per case, with the card's name and power limit read in the same run.
Arguments: optional comma-separated case names; `--size N` shrinks the raster for a dry run."""
import json
import os
import pickle
import resource
import subprocess
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import numpy as np

CASES = ["finite", "direct", "walls32", "one-to-all-16", "one-to-all-64", "all-to-one-16", "all-to-one-64",
         "regions-16x10"]
SETUP = ("set_grounds",)
PLAN = ("plan_advanced", "components")
SOLVE = ("solve_advanced", "solve_grounded", "solve_sources", "solve_region_pairs", "read_currents")


def run_one(name, on, size, out_path):
    """one case in this process -> (outputs as a dict of arrays, timings)"""
    import circuitscape_b200 as cb
    from circuitscape_b200 import solver as S
    import run_advanced_raster as adv
    import run_focal_regions as reg
    import run_onetoall as ota
    ota.SIZE = reg.SIZE = size
    spent = {"setup": 0.0, "plan": 0.0, "solve": 0.0}

    def timed(obj, attr, bucket):
        orig = getattr(obj, attr)

        def wrapper(*a, **kw):
            t0 = time.perf_counter()
            try:
                return orig(*a, **kw)
            finally:
                spent[bucket] += time.perf_counter() - t0
        setattr(obj, attr, wrapper)
    timed(S, "construct_raster_factor", "setup")
    for m in SETUP:
        timed(cb.B200Factor, m, "setup")
    for m in PLAN:
        timed(cb.B200Factor, m, "plan")
    for m in SOLVE:
        timed(cb.B200Factor, m, "solve")
    kw = dict(front_end_on_device=True) if on else {}
    t0 = time.perf_counter()
    if name in ("finite", "direct", "walls32"):
        g, src, gnd = adv.inputs(name, size)
        r = cb.raster_advanced(cb.RasterData(g, None, None, source_map=src, ground_map=gnd), adv.FLAGS,
                               {"remove_src_or_gnd": "keepall"}, solver=cb.CUDASolver(**kw))
        outs = dict(voltmap=r.voltmap, curmap=r.curmap, voltages=r.voltages, result=r.result,
                    num_solves=np.array(r.num_solves), iterations=np.array(r.iterations))
    elif name.startswith(("one-to-all", "all-to-one")):
        P = int(name.rsplit("-", 1)[1])
        g = ota.raster()
        r = cb.onetoall_kernel(cb.RasterData(g, None, ota.points(P)), ota.flags(False), {}, one_to_all=name[0] == "o",
                               solver=cb.CUDASolver(onetoall_raster=True, **kw))
        outs = dict(resistances=r.resistances, cum=r.cum_curmap, num_solves=np.array(r.num_solves))
        outs.update({f"cur_{k}": v for k, v in r.curmaps.items()})
    else:
        g = reg.raster()
        r = cb.raster_pairwise(cb.RasterData(g, None, reg.regions(16, 10)), reg.FLAGS, {}, solver=cb.CUDASolver(**kw))
        outs = dict(resistances=r.resistances, cum=r.cum_curmap, num_solves=np.array(r.num_solves))
    e2e = time.perf_counter() - t0
    with open(out_path, "wb") as fh:
        pickle.dump(outs, fh)
    return {"e2e_s": round(e2e, 2), "host_s": round(e2e - sum(spent.values()), 2),
            "setup_s": round(spent["setup"], 2), "plan_s": round(spent["plan"], 3), "solve_s": round(spent["solve"], 2),
            "peak_rss_mb": round(resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024.0)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    args = sys.argv[1:]
    if args and args[0] == "--child":
        name, on, size, path = args[1], args[2] == "1", int(args[3]), args[4]
        print(json.dumps(run_one(name, on, size, path)))
        return
    size = 3163
    if "--size" in args:
        i = args.index("--size")
        size = int(args[i + 1])
        del args[i:i + 2]
    rounds = 2
    if "--rounds" in args:
        i = args.index("--rounds")
        rounds = int(args[i + 1])
        del args[i:i + 2]
    names = args[0].split(",") if args else CASES
    gpu = card()
    with tempfile.TemporaryDirectory() as tmp:
        for name in names:
            runs, ref, same = [], None, True
            for rep, on in enumerate((False, True) * rounds):
                path = os.path.join(tmp, f"{rep}.pkl")
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", name, str(int(on)),
                                    str(size), path], capture_output=True, text=True)
                if p.returncode != 0:
                    raise RuntimeError(f"{name} (switch {'on' if on else 'off'}) failed:\n{p.stderr[-4000:]}")
                rec = json.loads(p.stdout.strip().splitlines()[-1])
                rec["switch"] = "on" if on else "off"
                runs.append(rec)
                with open(path, "rb") as fh:
                    outs = pickle.load(fh)
                if ref is None:
                    ref = outs
                else:
                    same = same and set(outs) == set(ref) and all(
                        np.asarray(outs[k]).tobytes() == np.asarray(ref[k]).tobytes() for k in ref)
            print(json.dumps({"case": name, "size": size, "card": gpu, "runs": runs, "outputs_bit_identical": same}),
                  flush=True)


if __name__ == "__main__":
    main()

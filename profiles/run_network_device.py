"""Network mode: host branch currents against the device ones, end to end.

    python profiles/run_network_device.py                       # both legs at the default sizes
    python profiles/run_network_device.py --only pairwise --nodes 5e5 --focal 8

pairwise: a power-law graph (graph.power_law_laplacian, the C5 graph of run_network.py) with `--focal` focal
nodes through core.solve and a sink that discards the per-pair output, once with the host branch path
(_branch_currents and _BranchIndex per pair) and once with CUDASolver(branch_on_device=True), alternated
`--reps` times; wall time per pair and the largest difference of the cumulative vectors.
advanced: `--components` disjoint power-law components of `--size` nodes plus `--isolated` nodes without
edges, one source, one finite ground and (every other component) one Inf ground each, through
advanced_kernel (one handle per component, node and branch currents in SciPy) and network_advanced (one
handle, cs_b200_solve_advanced_network), alternated; end-to-end wall time and the largest differences.
Prints the card name and power limit with one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as sp

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


class NullSink:
    def network(self, *a):
        pass

    voltmap = curmap = network


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
        name, power = (x.strip() for x in out.split(","))
        return name, power
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max(initial=0.0) / max(np.abs(np.asarray(b)).max(initial=0.0), 1e-300))


def pairwise(args):
    import circuitscape_b200 as cb
    from circuitscape_b200 import graph
    n = int(args.nodes)
    t0 = time.perf_counter()
    L = graph.power_law_laplacian(n, m=args.m, seed=11)
    print(f"pairwise graph: {time.perf_counter() - t0:.1f} s", file=sys.stderr, flush=True)
    up = sp.triu(L, k=1).tocoo()
    coords = (up.row.astype(np.int64) + 1, up.col.astype(np.int64) + 1)
    focal = graph.focal_nodes(n, args.focal, seed=7) + 1
    flags = cb.Flags(is_raster=False, outputflags=cb.OutputFlags(write_cur_maps=True))
    npairs = args.focal * (args.focal - 1) // 2
    times = {"host": [], "device": []}
    outs = {}
    for _ in range(args.reps):
        for leg in ("host", "device"):
            solver = cb.CUDASolver(precond=args.precond, branch_on_device=leg == "device")
            prob = cb.GraphProblem(L, [np.arange(1, n + 1)], focal, focal, set(), None, None, None, solver, coords)
            t0 = time.perf_counter()
            outs[leg] = cb.single_ground_all_pairs(prob, flags, sink=NullSink())
            times[leg].append((time.perf_counter() - t0) / npairs)
            print(f"pairwise {leg}: {times[leg][-1]:.3f} s per pair", file=sys.stderr, flush=True)
    h, d = outs["host"], outs["device"]
    return dict(nodes=n, edges=int(up.nnz), focal=args.focal, pairs=npairs, precond=args.precond,
                host_s_per_pair=min(times["host"]), device_s_per_pair=min(times["device"]),
                host_all=times["host"], device_all=times["device"],
                cum_branch_rel_diff=rel(d.cum_branch, h.cum_branch), cum_node_rel_diff=rel(d.cum_node, h.cum_node),
                resistance_rel_diff=rel(d.resistances, h.resistances))


def advanced(args):
    import circuitscape_b200 as cb
    from circuitscape_b200 import graph
    size = int(args.size)
    blocks = [graph.power_law_laplacian(size, m=args.m, seed=100 + c) for c in range(args.components)]
    half = args.components // 2
    G = sp.block_diag(blocks[:half] + [sp.csr_matrix((args.isolated, args.isolated))] + blocks[half:], format="csr")
    G.sort_indices()
    cc = graph.connected_components(G)
    n = G.shape[0]
    rng = np.random.default_rng(3)
    s, g = np.zeros(n), np.zeros(n)
    for c, nodes in enumerate(c for c in cc if len(c) > 1):
        rows = np.asarray(nodes) - 1
        pick = rng.choice(rows, 3, replace=False)
        s[pick[0]] = 1.0
        g[pick[1]] = 1.0
        if c % 2:
            g[pick[2]] = np.inf
    s, g, f = cb.resolve_conflicts(s, g, "keepall")
    flags = cb.Flags(is_raster=False, is_advanced=True)
    times = {"advanced_kernel": [], "network_advanced": []}
    outs = {}
    for _ in range(args.reps):
        for leg in times:
            prob = cb.AdvancedProblem(G, cc, s, g, f, solver=cb.CUDASolver(precond=args.precond))
            t0 = time.perf_counter()
            outs[leg] = (cb.advanced_kernel if leg == "advanced_kernel" else cb.network_advanced)(prob, flags)
            times[leg].append(time.perf_counter() - t0)
            print(f"advanced {leg}: {times[leg][-1]:.3f} s", file=sys.stderr, flush=True)
    a, b = outs["advanced_kernel"], outs["network_advanced"]
    assert np.array_equal(a.branch[0], b.branch[0]) and np.array_equal(a.branch[1], b.branch[1])
    return dict(nodes=n, edges=int(G.nnz - n + args.isolated) // 2, components=args.components, size=size,
                isolated=args.isolated, precond=args.precond, columns=b.stats["columns"],
                advanced_kernel_s=min(times["advanced_kernel"]), network_advanced_s=min(times["network_advanced"]),
                advanced_kernel_all=times["advanced_kernel"], network_advanced_all=times["network_advanced"],
                network_advanced_setup_s=b.stats["setup_s"], network_advanced_solve_s=b.stats["solve_s"],
                iterations=b.iterations, voltage_rel_diff=rel(b.voltages, a.voltages),
                node_current_rel_diff=rel(b.node_currents, a.node_currents),
                branch_rel_diff=rel(b.branch[2], a.branch[2]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", choices=["pairwise", "advanced"], default=None)
    ap.add_argument("--nodes", type=float, default=2e6)
    ap.add_argument("--m", type=int, default=5)
    ap.add_argument("--focal", type=int, default=16)
    ap.add_argument("--components", type=int, default=64)
    ap.add_argument("--size", type=float, default=3e4)
    ap.add_argument("--isolated", type=int, default=1000)
    ap.add_argument("--precond", default="amg", choices=["amg", "jacobi"])
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("run_network_device.py measures on a GPU; none is visible")
    name, power = card()
    res = dict(gpu=name, power_limit=power)
    if args.only in (None, "pairwise"):
        res["pairwise"] = pairwise(args)
    if args.only in (None, "advanced"):
        res["advanced"] = advanced(args)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

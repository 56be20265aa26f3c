"""Drivers of the hot path on the CUDA solver -- the host-side mirror of
src/core.jl (pairwise) and src/raster/advanced.jl:151-333 (advanced).

Public names follow the reference:
    get_solver(cfg)                         src/core.jl:74-94
    single_ground_all_pairs(prob, flags, cfg)  src/core.jl:70-72  -> solve(...)
    advanced_kernel(prob, flags, cfg)       src/raster/advanced.jl:151-271
    multiple_solver(cfg, solver, a, s, g, f)   src/raster/advanced.jl:274-305
`solve(prob, ::CUDASolver)` is the batched direct-style driver (src/core.jl:312-515)
re-thought for a device-resident solver: the pair list of a component is handed to
ONE `cs_b200_solve_pairs` call; voltages, node currents and the cumulative/max
accumulation stay on the GPU and only resistances (plus whatever per-pair maps the
flags ask for) come back.
"""
from __future__ import annotations

import time
from dataclasses import dataclass, field

import numpy as np
import scipy.sparse as sp

from . import _lib
from . import solver as S

NODATA = -9999.0
RESISTANCE_INVALID = -777.0   # src/consts.jl:45


# ---------------------------------------------------------------------------
# config / selection  (src/config.jl:68-73, src/consts.jl:12-15, src/core.jl:74-94)
# ---------------------------------------------------------------------------
def _parse_solver(s):
    """Unknown names fall back to cg+amg in the reference; here the only product
    solver is the CUDA one, so anything outside the CUDA table is refused loudly."""
    if s in S.CUDAB200:
        return "st_cuda"
    raise ValueError(f"solver = {s!r} is not served by circuitscape_b200 "
                     f"(use one of {S.CUDAB200}; cg+amg/cholmod stay in Circuitscape.jl)")


def get_solver(cfg):
    _parse_solver(cfg.get("solver", "cuda"))
    return S.CUDASolver(
        bs=int(cfg.get("cholmod_batch_size", "1000")),
        precision=cfg.get("precision", "double"),
        device=int(cfg.get("gpu_device", "0")),
        rtol=float(cfg.get("gpu_rtol", "1e-6")),
        precond=cfg.get("gpu_preconditioner", "amg"),
    )


def _flag(cfg, key, default="false"):
    return cfg.get(key, default) in ("True", "true", "1")   # src/config.jl:55-57


@dataclass
class OutputFlags:
    """src/out.jl:1-10."""
    write_volt_maps: bool = False
    write_cur_maps: bool = False
    write_cum_cur_map_only: bool = False
    write_max_cur_maps: bool = False
    set_null_currents_to_nodata: bool = False
    set_null_voltages_to_nodata: bool = False
    compress_grids: bool = False
    log_transform_maps: bool = False

    @classmethod
    def from_cfg(cls, cfg):
        return cls(**{k: _flag(cfg, k) for k in cls.__dataclass_fields__})


@dataclass
class Flags:
    """RasterFlags / NetworkFlags (src/raster/pairwise.jl:1-12, src/network/pairwise.jl:84-92)."""
    is_raster: bool = True
    is_advanced: bool = False
    outputflags: OutputFlags = field(default_factory=OutputFlags)

    @classmethod
    def from_cfg(cls, cfg):
        return cls(is_raster=cfg.get("data_type", "raster") in ("raster", "Raster"),
                   is_advanced=cfg.get("scenario", "pairwise") in ("advanced", "Advanced"),
                   outputflags=OutputFlags.from_cfg(cfg))


@dataclass
class GraphProblem:
    """src/core.jl:10-22 (hbmeta dropped: file metadata is not on the path)."""
    G: sp.csr_matrix
    cc: list                      # list of 1-based node-id arrays
    points: np.ndarray            # graph node per focal point (1-based, 0 = none)
    user_points: np.ndarray       # user ids
    exclude_pairs: set = field(default_factory=set)
    nodemap: np.ndarray | None = None
    polymap: np.ndarray | None = None
    cellmap: np.ndarray | None = None
    solver: S.CUDASolver = field(default_factory=S.CUDASolver)
    coords: tuple | None = None   # network mode: (i, j) 1-based edge list (Cumulative.coords)


@dataclass
class PairwiseOutput:
    resistances: np.ndarray
    voltmaps: dict = field(default_factory=dict)
    curmaps: dict = field(default_factory=dict)
    branch: dict = field(default_factory=dict)
    cum_curmap: np.ndarray | None = None
    max_curmap: np.ndarray | None = None
    cum_node: np.ndarray | None = None
    cum_branch: np.ndarray | None = None
    num_solves: int = 0
    iterations: int = 0
    stats: list = field(default_factory=list)


# ---------------------------------------------------------------------------
# pair enumeration  (src/core.jl:386-424, 537-603)
# ---------------------------------------------------------------------------
def component_pairs(points, user_points, exclude, comp, shortcut):
    """For one component: unique focal nodes `csub` (in focal-point order), the
    node pairs to solve with their focal-index fan-out, and the index pairs that
    share a node (R = 0, smash_repeats!)."""
    points = np.asarray(points)
    member = np.isin(points, comp) & (points != 0)
    idx_by_node = {}
    for k in np.nonzero(member)[0]:
        idx_by_node.setdefault(int(points[k]), []).append(int(k))
    csub = list(idx_by_node)
    zero, solves = [], []
    for pi, s in enumerate(csub[: (1 if shortcut else len(csub))]):
        si = idx_by_node[s]
        zero += [(si[a], si[b]) for a in range(len(si)) for b in range(a + 1, len(si))]
        for d in csub[pi + 1:]:
            fan = [(ci, cj) for ci in si for cj in idx_by_node[d]
                   if (int(user_points[ci]), int(user_points[cj])) not in exclude]
            if fan:
                solves.append((s, d, fan))
    return csub, solves, zero


def construct_local_node_map(nodemap, comp, polymap):
    """src/utils.jl:10-30: cell -> row of the component's matrix (1-based, 0 = none)."""
    from .graph import construct_node_map
    inside = np.isin(nodemap, comp)
    local = np.where(inside, nodemap, 0)
    if np.array_equal(local, nodemap):
        return local
    if polymap is None or np.size(polymap) == 0:
        flat = local.reshape(-1, order="F")
        nz = flat != 0
        flat = flat.copy()
        flat[nz] = np.arange(1, int(nz.sum()) + 1)
        return flat.reshape(local.shape, order="F")
    return construct_node_map(local, np.where(inside, polymap, 0))


def _scatter(values, local_nodemap):
    out = np.zeros(local_nodemap.shape, dtype=np.float64)
    nz = local_nodemap != 0
    out[nz] = values[local_nodemap[nz] - 1]
    return out


def _process_grid(cmap, cellmap, log_transform, set_null_to_nodata):
    """src/out.jl:305-319."""
    if log_transform:
        pos = cmap > 0
        cmap = np.where(pos, np.log10(np.where(pos, cmap, 1.0)), NODATA)
    if set_null_to_nodata:
        cmap = np.where(cellmap == 0, NODATA, cmap)
    return cmap


def _any_map(o):
    """Whether the job writes any current or voltage map (src/core.jl:356-364: otherwise raster pairwise
    takes the shortcut)."""
    return o.write_volt_maps or o.write_cur_maps or o.write_cum_cur_map_only or o.write_max_cur_maps


def _panels(n, solver):
    """Slices of at most solver.bs columns over n columns (cholmod_batch_size, src/core.jl:448-452)."""
    bs = max(1, int(solver.bs))
    for st in range(0, n, bs):
        yield slice(st, min(st + bs, n))


def _pair_maps(out, sink, key, grid, volt, cur, cellmap, o):
    """One pair's voltage and current maps (src/out.jl:90-112): `grid` scatters a node vector to cells;
    `volt` / `cur` are None when not written.  Handed to `sink`, or kept in out.voltmaps / out.curmaps."""
    if volt is not None:
        vm = _process_grid(grid(volt), cellmap, False, o.set_null_voltages_to_nodata)
        if sink is not None:
            sink.voltmap(key, vm)
        else:
            out.voltmaps[key] = vm
    if cur is not None:
        cm = _process_grid(grid(cur), cellmap, o.log_transform_maps, o.set_null_currents_to_nodata)
        if sink is not None:
            sink.curmap(key, cm)
        else:
            out.curmaps[key] = cm


def _add_current_maps(out, cum, mx, nodemap, npost, cellmap, o):
    """Add the per-node cumulative and max currents of `npost` pairs, scattered by `nodemap`, into
    out.cum_curmap / out.max_curmap.  Each pair's map holds 0 on cells that are no node of `nodemap`, which
    the log transform makes NODATA, and NODATA on NODATA cells under set_null_currents_to_nodata: so those
    cells get NODATA * npost in the sum and NODATA in the max."""
    cmap = _scatter(np.asarray(cum, dtype=np.float64), nodemap)
    off = nodemap == 0
    if o.log_transform_maps:
        cmap = np.where(off, NODATA * npost, cmap)
    if o.set_null_currents_to_nodata:
        cmap = np.where(cellmap == 0, NODATA * npost, cmap)
    out.cum_curmap += cmap
    if out.max_curmap is not None:
        mmap = _scatter(np.asarray(mx, dtype=np.float64), nodemap)
        mmap = np.where(off, NODATA if o.log_transform_maps else 0.0, mmap)
        if o.set_null_currents_to_nodata:
            mmap = np.where(cellmap == 0, NODATA, mmap)
        out.max_curmap = np.maximum(out.max_curmap, mmap)


def _finish_pairwise(out, R, ids):
    """R = 0 on the diagonal, framed by the point ids (src/core.jl:294-299), and the NODATA clamp of the
    cumulative and max maps (src/utils.jl:114-120)."""
    P = len(ids)
    np.fill_diagonal(R, 0.0)
    full = np.zeros((P + 1, P + 1))
    full[0, 1:] = ids
    full[1:, 0] = ids
    full[1:, 1:] = R
    out.resistances = full
    if out.cum_curmap is not None:
        out.cum_curmap = np.where(out.cum_curmap < NODATA, NODATA, out.cum_curmap)
    if out.max_curmap is not None:
        out.max_curmap = np.where(out.max_curmap < NODATA, NODATA, out.max_curmap)
    return out


def _probe_solve(factor, src, dst, focal_rows, focal_col):
    """Shortcut mode: only the voltages at the focal nodes are used (update_voltmatrix!, src/core.jl:685-703),
    so the pairs are solved with probe rows instead of bringing n x k voltages back; R read off the probe."""
    res = factor.solve_sources([([s_, d_], [-1.0, 1.0]) for s_, d_ in zip(src, dst)], ref=src, probe=focal_rows)
    res["R"] = np.array([res["probe_volt"][c, focal_col[int(d_)]] for c, d_ in enumerate(dst)])
    return res


def _raster_factor(cellmap, polymap, nodemap, solver, four_neighbors, avg_res, log_transform=False):
    """The whole-raster handle (S.construct_raster_factor), checked to number its nodes as the host's `nodemap`."""
    factor, dev_nodemap = S.construct_raster_factor(cellmap, polymap, solver, four_neighbors=four_neighbors,
                                                    avg_res=avg_res, log_transform=log_transform)
    if not np.array_equal(np.asarray(dev_nodemap), nodemap):
        factor.close()
        raise RuntimeError("device node map differs from the host's")
    return factor


def _component_labels(adj):
    """(ncomp, label per node) of a construct_graph adjacency, a stored zero being no edge; drops those zeros
    from `adj`."""
    from scipy.sparse import csgraph
    adj.eliminate_zeros()
    return csgraph.connected_components(adj, directed=False)


# ---------------------------------------------------------------------------
# pairwise driver
# ---------------------------------------------------------------------------
def single_ground_all_pairs(prob: GraphProblem, flags: Flags, cfg=None, log=True, sink=None) -> PairwiseOutput:
    """src/core.jl:70-72."""
    return solve(prob, prob.solver, flags, cfg, log, sink=sink)


def solve(prob: GraphProblem, solver: S.CUDASolver, flags: Flags, cfg=None, log=True, sink=None) -> PairwiseOutput:
    """`sink`: optional writer the per-pair results are handed to as each batch finishes -- the
    reference writes every map inside `postprocess` and drops it (src/core.jl:655-683); without a
    sink they are kept in the returned object (tests, small jobs).  A sink has the methods
    `voltmap(key, grid)`, `curmap(key, grid)` (raster) and `network(key, comp, volt, cur, branch)`."""
    o = flags.outputflags
    P = len(prob.points)
    R = -np.ones((P, P))
    shortcut = flags.is_raster and not _any_map(o) and not prob.exclude_pairs    # src/core.jl:356-364
    voltmatrix = np.zeros((P, P))
    shortcut_res = -np.ones((P, P))
    out = PairwiseOutput(resistances=None)
    raster = flags.is_raster
    if raster:
        out.cum_curmap = np.zeros(prob.cellmap.shape)
        out.max_curmap = np.full(prob.cellmap.shape, NODATA) if o.write_max_cur_maps else None
    else:
        out.cum_node = np.zeros(prob.G.shape[0])
        out.cum_branch = np.zeros(len(prob.coords[0]))
        branch_pos = _BranchIndex(prob.coords)
    G = sp.csr_matrix(prob.G)
    points = np.asarray(prob.points)
    ids = np.asarray(prob.user_points)
    # network branch currents from the device (cs_b200_solve_pairs_branch); the superposed driver keeps the
    # host path
    device_branch = not raster and getattr(solver, "branch_on_device", False) and not getattr(solver, "superpose", False)

    for comp in prob.cc:
        comp = np.asarray(comp)
        csub, solves, zero = component_pairs(points, ids, prob.exclude_pairs, comp, shortcut)
        if not csub:
            continue
        for a, b in zero:
            R[a, b] = R[b, a] = 0.0
        if not solves:
            if shortcut:      # duplicates on the anchor only: the reference still runs the update (core.jl:504-506)
                anchor = int(np.nonzero(points == csub[0])[0][0])
                _update_shortcut_resistances(anchor, voltmatrix, shortcut_res, R, points, comp)
            continue
        rows = comp - 1
        matrix = G[rows][:, rows].tocsr()
        local_of = np.zeros(G.shape[0] + 1, dtype=np.int64)
        local_of[comp] = np.arange(len(comp))
        src = np.array([local_of[s] for s, _, _ in solves])
        dst = np.array([local_of[d] for _, d, _ in solves])
        weight = np.array([len(f) for _, _, f in solves], dtype=np.float64)
        need_curr = not shortcut                       # postprocess always builds the current map
        # host network branch currents need v
        per_pair_volt = o.write_volt_maps or (not raster and not shortcut and not device_branch)
        per_pair_curr = need_curr and ((o.write_cur_maps and not o.write_cum_cur_map_only) or not raster)
        local_nodemap = construct_local_node_map(prob.nodemap, comp, prob.polymap) if raster and not shortcut else None
        # only raster maps are log-transformed (src/out.jl:96 process_grid!); the network branch of
        # write_cur_maps accumulates raw node currents (src/out.jl:48-88)
        with S.construct_cholesky_factor(matrix, solver, log_transform=bool(o.log_transform_maps and raster)) as factor:
            if device_branch:
                lo, hi = _branch_index(factor, matrix)
                bpos = branch_pos.positions(comp[lo], comp[hi])
            if shortcut:
                inside = np.nonzero(np.isin(points, comp) & (points != 0))[0]
                focal_rows = np.unique(local_of[points[inside]])
                focal_col = {int(r): i for i, r in enumerate(focal_rows)}

            def batches():
                if getattr(solver, "superpose", False) and not shortcut and len(solves) > 1:
                    # one solve per focal NODE of the component, every pair by superposition
                    # (the Shortcut algebra of src/core.jl:685-739 applied to the voltages)
                    nodes, inv = np.unique(np.concatenate([src, dst]), return_inverse=True)
                    yield slice(0, len(solves)), factor.solve_pairs_superposed(
                        nodes, inv[:len(src)], inv[len(src):], weight, want_volt=per_pair_volt,
                        want_curr=per_pair_curr, accumulate=need_curr)
                    return
                for sl in _panels(len(solves), solver):
                    if shortcut:
                        yield sl, _probe_solve(factor, src[sl], dst[sl], focal_rows, focal_col)
                        continue
                    yield sl, factor.solve_pairs(src[sl], dst[sl], weight[sl], want_volt=per_pair_volt,
                                                 want_curr=per_pair_curr, accumulate=need_curr,
                                                 want_branch=device_branch)

            for sl, res in batches():
                out.stats.append(factor.stats())
                out.num_solves += len(res["R"])
                out.iterations += int(res["iters"].sum())
                for col, (s, d, fan) in enumerate(solves[sl]):
                    r = float(res["R"][col])
                    v = res["volt"][:, col].astype(np.float64) if res.get("volt") is not None else None
                    cur = res["curr"][:, col].astype(np.float64) if res.get("curr") is not None else None
                    if device_branch:
                        br = (comp[lo], comp[hi], np.asarray(res["branch"][:, col], dtype=np.float64))
                    else:
                        br = _branch_currents(matrix, v, comp) if not raster and not shortcut else None
                    for ci, cj in fan:
                        R[ci, cj] = R[cj, ci] = r
                        key = (int(ids[ci]), int(ids[cj]))
                        if shortcut:                                             # src/core.jl:685-703
                            pv = res["probe_volt"][col]
                            for i in inside[inside >= 1]:
                                voltmatrix[i, cj] = 1.0 - float(pv[focal_col[int(local_of[points[i]])]]) / r
                            continue
                        if raster:
                            _pair_maps(out, sink, key, lambda x: _scatter(x, local_nodemap), v, cur, prob.cellmap, o)
                        else:
                            # every id combination is post-processed on its own (src/core.jl:235-249):
                            # its branch currents go into the cumulative vector once each (on the device:
                            # weight[col] = len(fan) times)
                            if not device_branch:
                                branch_pos.add(out.cum_branch, br)
                            if sink is not None:
                                sink.network(key, comp, v if o.write_volt_maps else None, cur, br)
                            else:
                                if o.write_volt_maps:
                                    out.voltmaps[key] = (comp, v)
                                out.curmaps[key] = (comp, cur)
                                out.branch[key] = br
            if need_curr:
                cum, mx = factor.read_currents(want_max=True)
                if raster:
                    _add_current_maps(out, cum, mx, local_nodemap, float(weight.sum()), prob.cellmap, o)
                else:
                    out.cum_node[rows] += cum
                    if device_branch:
                        np.add.at(out.cum_branch, bpos, np.asarray(factor.read_branch_currents(), dtype=np.float64))
        if shortcut:
            anchor = int(np.nonzero(points == csub[0])[0][0])
            _update_shortcut_resistances(anchor, voltmatrix, shortcut_res, R, points, comp)
    return _finish_pairwise(out, shortcut_res if shortcut else R, ids)


def _upper_branches(matrix):
    """(row, col, value) of the stored upper triangle of `matrix` in the order `_convert_to_3col` walks the CSC
    branch matrix (column-major: sorted by column, then row), so written files match the reference's."""
    coo = sp.triu(sp.csr_matrix(matrix), k=1).tocoo()
    order = np.lexsort((coo.row, coo.col))
    return coo.row[order], coo.col[order], coo.data[order]


def _branch_currents(matrix, v, comp):
    """Network mode branch currents |G_ij| |v_i - v_j| over the stored upper triangle
    with the 1e-8 relative zeroing (src/out.jl:154-158, 250-290); host side, network
    graphs only, in the order of _upper_branches."""
    row, col, data = _upper_branches(matrix)
    b = np.abs(data) * (v[row] - v[col])
    if len(b):
        mx = b.max()
        with np.errstate(divide="ignore", invalid="ignore"):
            b = np.where(np.abs(b / mx) < 1e-8, 0.0, b)
    return comp[row], comp[col], np.abs(b)


class _BranchIndex:
    """Position of every graph edge in `coords` (the cumulative branch vector's order,
    src/utils.jl:132-142) by a sorted key table instead of the reference's linear `findfirst`
    per branch (src/out.jl:65-84).  An edge that is not in `coords` raises, like the reference's
    `cbc[nothing]`."""

    def __init__(self, coords):
        a = np.asarray(coords[0], dtype=np.int64)
        b = np.asarray(coords[1], dtype=np.int64)
        self.base = int(max(a.max(initial=0), b.max(initial=0))) + 1
        key = a * self.base + b
        # findfirst semantics: the first occurrence of a repeated edge wins
        self.order = np.argsort(key, kind="stable")
        self.keys = key[self.order]

    def _find(self, a, b):
        key = a * self.base + b
        pos = np.searchsorted(self.keys, key, side="left")
        ok = (pos < len(self.keys))
        ok[ok] = self.keys[pos[ok]] == key[ok]
        return np.where(ok, self.order[np.minimum(pos, len(self.keys) - 1)], -1)

    def positions(self, gr, gc):
        """Position in `coords` of every branch (gr, gc), or of (gc, gr) when only the reversed edge is there."""
        gr = np.asarray(gr, dtype=np.int64)
        gc = np.asarray(gc, dtype=np.int64)
        k = self._find(gr, gc)
        miss = k < 0
        if miss.any():
            k[miss] = self._find(gc[miss], gr[miss])
        if (k < 0).any():
            i = int(np.nonzero(k < 0)[0][0])
            raise KeyError(f"branch ({int(gr[i])}, {int(gc[i])}) is not an edge of the graph")
        return k

    def add(self, cum, branch):
        gr, gc, val = branch
        np.add.at(cum, self.positions(gr, gc), val)


def _branch_index(factor, matrix):
    """The handle's branches (0-based lo, hi), checked against the order _branch_currents writes them in
    (_upper_branches)."""
    lo, hi = factor.branch_index()
    row, col, _ = _upper_branches(matrix)
    if not (np.array_equal(lo, row) and np.array_equal(hi, col)):
        raise RuntimeError("the device's branch order differs from the upper triangle's column-major order")
    return lo, hi


def _update_shortcut_resistances(anchor, voltmatrix, shortcut, resistances, points, comp):
    """src/core.jl:706-739:  R_2x = 2 R_12 V_x2 + R_1x - R_12."""
    check = np.isin(points, comp) & (np.asarray(points) != 0)
    l = resistances.shape[0]
    for px in np.nonzero(check)[0]:
        R1x = resistances[anchor, px]
        if R1x == -1:
            continue
        shortcut[px, anchor] = shortcut[anchor, px] = R1x
        for p2 in range(px, l):
            if not check[p2]:
                continue
            R12 = resistances[anchor, p2]
            if R12 == -1:
                continue
            if R1x != RESISTANCE_INVALID:
                shortcut[anchor, p2] = shortcut[p2, anchor] = R12
                R2x = 2 * R12 * voltmatrix[px, p2] + R1x - R12
                if shortcut[p2, px] != RESISTANCE_INVALID:
                    shortcut[p2, px] = shortcut[px, p2] = R2x
            else:
                shortcut[px, :] = RESISTANCE_INVALID
                shortcut[:, px] = RESISTANCE_INVALID


def compute_3col(r):
    """src/out.jl:12-26."""
    fp = r[1:, 0]
    i, j = np.triu_indices(len(fp), k=1)
    return np.column_stack([fp[i], fp[j], r[j + 1, i + 1]])


# ---------------------------------------------------------------------------
# advanced mode  (src/raster/advanced.jl:151-333)
# ---------------------------------------------------------------------------
@dataclass
class AdvancedProblem:
    """src/raster/advanced.jl:1-15."""
    G: sp.csr_matrix
    cc: list
    sources: np.ndarray
    grounds: np.ndarray
    finitegrounds: np.ndarray       # [-9999.] sentinel when there are none
    nodemap: np.ndarray | None = None
    polymap: np.ndarray | None = None
    cellmap: np.ndarray | None = None
    solver: S.CUDASolver = field(default_factory=S.CUDASolver)


@dataclass
class AdvancedOutput:
    voltages: np.ndarray
    voltmap: np.ndarray | None = None
    curmap: np.ndarray | None = None
    node_currents: np.ndarray | None = None
    branch: tuple | None = None
    result: np.ndarray | None = None      # raster_advanced: what the reference's raster_advanced returns
    num_solves: int = 0                   # raster_advanced: components solved
    iterations: int = 0                   # raster_advanced: PCG iterations over the columns
    stats: dict = field(default_factory=dict)   # raster_advanced: setup_s / solve_s (host clock), columns


def multiple_solver(cfg, solver, a, sources, grounds, finitegrounds, resident=None):
    """src/raster/advanced.jl:274-305: diag += finite grounds; rows/cols of Inf
    grounds deleted (0 V); `multiple_solve`; zeros re-inserted.

    resident = (cache dict, key): keep ONE device factor of the component's Laplacian `a` under `key`
    and move the grounds on the device (cs_b200_set_grounds: identity rows instead of deleted ones)
    -- for the one-to-all / all-to-one loops, where only the grounds change between iterations."""
    if resident is not None:
        cache, key = resident
        f = cache.get(key)
        if f is None:
            f = cache[key] = S.construct_cholesky_factor(sp.csr_matrix(a, dtype=np.float64), solver)
        mask = np.asarray(grounds) == np.inf
        f.set_grounds(None if finitegrounds[0] == NODATA else np.asarray(finitegrounds, dtype=np.float64),
                      mask if mask.any() else None)
        b = np.asarray(sources, dtype=np.float64).copy()
        b[mask] = 0.0
        v = np.asarray(S.solve_linear_system(f, a, b), dtype=np.float64).copy()   # residual gate inside (hook #2)
        v[mask] = 0.0
        return v
    a = sp.csr_matrix(a, dtype=np.float64)
    n = a.shape[0]
    if finitegrounds[0] != NODATA:
        a = (a + sp.diags(finitegrounds)).tocsr()
    keep = np.nonzero(~(grounds == np.inf))[0]
    asolve = a[keep][:, keep].tocsr()
    volt = S.multiple_solve(solver, asolve, np.asarray(sources, dtype=np.float64)[keep])
    v = np.zeros(n)
    v[keep] = volt
    return v


def node_currents_host(G, v, finitegrounds=None):
    """src/out.jl:178-207 on the host (advanced mode solves once per component; the
    pairwise path uses the device kernel instead)."""
    coo = sp.triu(sp.csr_matrix(G), k=1).tocoo()
    n = G.shape[0]
    d = np.abs(coo.data) * (v[coo.row] - v[coo.col])

    def one(b):
        if len(b):
            mx = b.max()
            with np.errstate(divide="ignore", invalid="ignore"):
                b = np.where(np.abs(b / mx) < 1e-8, 0.0, b)
        s = np.zeros(n)
        np.add.at(s, coo.col, np.maximum(b, 0.0))
        np.add.at(s, coo.row, np.maximum(-b, 0.0))
        return s

    p, q = one(d), one(-d)
    if finitegrounds is not None and finitegrounds[0] != NODATA:
        fg = finitegrounds * v
        p = p + np.where(fg < 0, -fg, 0.0)
        q = q + np.where(fg > 0, fg, 0.0)
    return np.where(p > q, p, q)


def advanced_kernel(prob: AdvancedProblem, flags: Flags, cfg=None) -> AdvancedOutput:
    G = sp.csr_matrix(prob.G)
    n = G.shape[0]
    raster = flags.is_raster
    voltages = np.zeros(n)
    outvolt = np.zeros(prob.nodemap.shape) if raster else None
    outcurr = np.zeros(prob.nodemap.shape) if raster else None
    for c in prob.cc:
        rows = np.asarray(c) - 1
        s_local, g_local = prob.sources[rows].copy(), prob.grounds[rows].copy()
        if s_local.sum() == 0 or g_local.sum() == 0:                          # :194-196
            continue
        f_local = prob.finitegrounds[rows] if prob.finitegrounds[0] != NODATA else prob.finitegrounds
        a_local = G[rows][:, rows].tocsr()
        voltages[rows] += multiple_solver(cfg, prob.solver, a_local, s_local, g_local, f_local)
        if raster:
            lm = construct_local_node_map(prob.nodemap, np.asarray(c), prob.polymap)
            outvolt += _scatter(voltages[rows], lm)
            outcurr += _scatter(node_currents_host(a_local, voltages[rows], f_local), lm)
    res = AdvancedOutput(voltages, outvolt, outcurr)
    if not raster:
        res.node_currents = node_currents_host(G, voltages, prob.finitegrounds)
        res.branch = _branch_currents(G, voltages, np.arange(1, n + 1))
    return res


def network_advanced(prob: AdvancedProblem, flags: Flags, cfg=None) -> AdvancedOutput:
    """advanced_kernel for networks (src/raster/advanced.jl:184-242) on ONE whole-graph handle: every connected
    component with sum(sources) != 0, sum(grounds) != 0 and a source off its Inf grounds is one column of
    cs_b200_solve_advanced_network, its Inf grounds a Dirichlet set at 0 V, the finite grounds on the
    operator's diagonal (set_grounds, once).  The node and branch currents are taken of the summed voltages
    under one 1e-8 cut over the whole graph, as the reference takes them, so every column goes into one
    call (the device walks them in panels).  Returns AdvancedOutput with voltages, node_currents and branch
    ((lo, hi) 1-based, values) as advanced_kernel's network output, num_solves, iterations and stats."""
    G = sp.csr_matrix(prob.G)
    n = G.shape[0]
    s, g = np.asarray(prob.sources, dtype=np.float64), np.asarray(prob.grounds, dtype=np.float64)
    f = np.asarray(prob.finitegrounds, dtype=np.float64)
    columns, solved = [], 0
    for c in prob.cc:
        rows = np.asarray(c, dtype=np.int64) - 1
        if s[rows].sum() == 0 or g[rows].sum() == 0:                      # advanced.jl:194-196
            continue
        solved += 1
        inf = g[rows] == np.inf
        src = rows[(s[rows] != 0) & ~inf]                                 # sources on Inf grounds are deleted
        if len(src):                                                      # else b = 0: the component stays at 0 V
            columns.append((rows, rows[inf], src, s[src]))
    out = AdvancedOutput(np.zeros(n), num_solves=solved)
    out.stats = dict(setup_s=0.0, solve_s=0.0, columns=len(columns))
    if not columns:
        out.node_currents = np.zeros(n)
        out.branch = _branch_currents(G, out.voltages, np.arange(1, n + 1))
        return out
    # every diagonal entry stored, so that set_grounds can put a finite ground on a node without edges
    coo = G.tocoo()
    off = coo.row != coo.col
    diag = np.arange(n)
    A = sp.csr_matrix((np.r_[coo.data[off], G.diagonal()], (np.r_[coo.row[off], diag], np.r_[coo.col[off], diag])),
                      shape=(n, n))
    owner = np.full(n, -1, dtype=np.int64)
    sets, gset = [], []
    for j, (rows, gnd, _, _) in enumerate(columns):
        owner[rows] = j
        gset.append(len(sets) if len(gnd) else -1)                       # -1: finite grounds only
        if len(gnd):
            sets.append(gnd)
    t0 = time.perf_counter()
    with S.construct_cholesky_factor(A, prob.solver) as factor:
        if f[0] != NODATA:
            factor.set_grounds(finite=f)
        lo, hi = _branch_index(factor, G)
        t1 = time.perf_counter()
        res = factor.solve_advanced_network(sets, gset, [(c[2], c[3]) for c in columns], owner, want_volt=True,
                                            want_curr=True, want_branch=True)
        t2 = time.perf_counter()
    out.voltages = np.asarray(res["volt"], dtype=np.float64)
    out.node_currents = np.asarray(res["curr"], dtype=np.float64)
    out.branch = (lo + 1, hi + 1, np.asarray(res["branch"], dtype=np.float64))
    out.iterations = int(res["iters"].sum())
    out.stats.update(setup_s=t1 - t0, solve_s=t2 - t1)
    return out


def all_to_one_batched(factor, focal, rtol=None, shard=None, device_resident=False, accumulate=False):
    """All-to-one on a graph WITHOUT finite grounds, batched on one factor.

    Iteration c of the reference's all-to-one loop (src/raster/onetoall.jl:110-118,146-151)
    ties focal node f_c to ground (Dirichlet, row/column deleted in `multiple_solver`,
    src/raster/advanced.jl:286-300) and injects 1 A at every other focal node.  Current
    conservation makes that the singular-Laplacian system  L v = e_others - (P-1) e_fc
    followed by the shift v -= v[f_c] -- the pairwise trick of src/core.jl:224-232 with a
    multi-source right-hand side -- so every iteration shares ONE operator and the P
    solves are columns of one batch instead of P factorizations.  `factor` must hold the
    connected component's Laplacian; `shard=(rank, world)` keeps columns rank::world.

    device_resident=False: through hook #2 (`solve_linear_system`, n x k host batch);
        returns (voltages (n, P'), iters, relres, cols).
    device_resident=True: through cs_b200_solve_sources -- right-hand sides are scattered
        on the device, only the voltages at the focal nodes come back, node currents are
        accumulated into the handle's cumulative / max vectors when `accumulate`;
        returns (focal voltages (P', P), iters, relres, cols)."""
    focal = np.asarray(focal, dtype=np.int64)
    cols = np.arange(len(focal)) if shard is None else np.arange(shard[0], len(focal), shard[1])
    n = factor.n
    if device_resident:
        columns = []
        for c in cols:
            v = np.ones(len(focal))
            v[c] = -(len(focal) - 1.0)
            columns.append((focal, v))
        o = factor.solve_sources(columns, focal[cols], probe=focal, accumulate=accumulate, rtol=rtol)
        return o["probe_volt"], o["iters"], o["relres"], cols
    rhs = np.zeros((n, len(cols)), dtype=factor.io_dtype, order="F")
    for j, c in enumerate(cols):
        rhs[focal, j] = 1.0
        rhs[focal[c], j] = -(len(focal) - 1.0)
    x, iters, relres = factor.solve_rhs(rhs, rtol=rtol)
    x = np.asarray(x).reshape(n, len(cols))
    x -= x[focal[cols], np.arange(len(cols))][None, :]
    return x, iters, relres, cols


# ---------------------------------------------------------------------------
# one-to-all / all-to-one  (src/raster/onetoall.jl) -- callers of the advanced kernel
# ---------------------------------------------------------------------------
def compute_omniscape_current(conductance, source, ground, cs_cfg, solver=None):
    """src/utils.jl:145-257 -- Omniscape's moving-window solve: one advanced-mode solve per
    connected component of a conductance window, returning the node-current raster.

    conductance / source / ground: 2-D arrays of one shape (NODATA or 0 conductance = no
    node; ground values are conductances: the reference hard-wires grnd_file_is_res =
    false, policy :rmvsrc and the average-conductance rule there, utils.jl:190-193);
    cs_cfg: the INI dictionary (only `connect_four_neighbors_only` and the solver keys are
    read).  `solver` overrides `get_solver(cs_cfg)`; tests pass a CPU double here."""
    from . import graph
    cellmap = np.array(conductance, dtype=np.float64)
    cellmap[cellmap == NODATA] = 0.0
    nodemap = graph.construct_node_map(cellmap, None)
    four = _flag(cs_cfg, "connect_four_neighbors_only")
    G = graph.laplacian(graph.construct_graph(cellmap, nodemap, False, four))
    cc = graph.connected_components(G)
    s, g, f = sources_and_grounds_from_maps(np.asarray(source, dtype=np.float64),
                                            np.asarray(ground, dtype=np.float64), nodemap, G.shape[0], "rmvsrc")
    prob = AdvancedProblem(G, cc, s, g, f, nodemap, None, cellmap, solver if solver is not None else get_solver(cs_cfg))
    return advanced_kernel(prob, Flags(is_raster=True, is_advanced=True), cs_cfg).curmap


@dataclass
class OmniscapeBatch:
    """Result of compute_omniscape_currents, one entry per input window in input order."""
    currents: list                 # float64 rasters of each window's own shape
    voltages: list | None          # the same for the voltages (want_voltages=True)
    iterations: np.ndarray         # CG iterations, summed over the window's solved components
    relres: np.ndarray             # largest true relative residual of the window's solved components


def _windows(a, name):
    ws = list(a) if isinstance(a, (list, tuple)) or (isinstance(a, np.ndarray) and a.ndim == 3) else None
    if ws is None:
        raise ValueError(f"{name}: expected a 3-D stack or a list of 2-D windows")
    out = []
    for k, w in enumerate(ws):
        w = np.asarray(w)
        if w.ndim != 2 or w.size == 0 or not (np.issubdtype(w.dtype, np.number) or w.dtype == bool):
            raise ValueError(f"{name}[{k}]: expected a non-empty numeric 2-D window, got shape {w.shape} "
                             f"dtype {w.dtype}")
        out.append(w)
    return out


def compute_omniscape_currents(conductances, sources, grounds, cs_cfg, want_voltages=False, solver=None,
                               max_batch_bytes=1 << 30) -> OmniscapeBatch:
    """`compute_omniscape_current` for many windows at once: window w of the result is what
    compute_omniscape_current(conductances[w], sources[w], grounds[w], cs_cfg) returns, computed by
    cs_b200_solve_advanced_batch (one CTA per window, Jacobi-preconditioned CG per connected
    component; same rtol / itmax / device and 1e-4 residual gate as the per-window path).

    conductances / sources / grounds: 3-D stacks (nwin, nrows, ncols) or lists of 2-D windows; the
    three must agree window by window, but windows may differ in shape -- they are padded to a common
    shape with g = 0 cells (not nodes) and cropped back.  float32 inputs stay float32 on the way in
    when all three are float32; the device arithmetic and the outputs are float64.
    Windows go to the device in batches of at most `max_batch_bytes` of device memory (at least one
    window per batch).  A window whose component fails the gate raises SolverResidualError naming it."""
    gs, ss, ns = (_windows(a, n) for a, n in ((conductances, "conductances"), (sources, "sources"),
                                               (grounds, "grounds")))
    if not len(gs) == len(ss) == len(ns):
        raise ValueError(f"{len(gs)} conductance, {len(ss)} source and {len(ns)} ground windows")
    for k, (g, s, n) in enumerate(zip(gs, ss, ns)):
        if not g.shape == s.shape == n.shape:
            raise ValueError(f"window {k}: conductance {g.shape}, source {s.shape}, ground {n.shape} differ")
    if max_batch_bytes <= 0:
        raise ValueError("max_batch_bytes must be positive")
    solver = solver if solver is not None else get_solver(cs_cfg)
    four = _flag(cs_cfg, "connect_four_neighbors_only")
    nwin = len(gs)
    dtype = np.float32 if all(a.dtype == np.float32 for a in gs + ss + ns) else np.float64
    nr = max((g.shape[0] for g in gs), default=1)
    nc = max((g.shape[1] for g in gs), default=1)
    # one padded shape for every batch, so a window's result does not depend on the split
    per = S.advanced_batch_bytes(nr * nc, np.dtype(dtype).itemsize, want_voltages)
    bw = max(1, int(max_batch_bytes // per))
    out = OmniscapeBatch([], [] if want_voltages else None, np.zeros(nwin, dtype=np.int64), np.zeros(nwin))
    for b0 in range(0, nwin, bw):
        idx = range(b0, min(nwin, b0 + bw))
        stacks = [np.zeros((len(idx), nr, nc), dtype=dtype) for _ in range(3)]
        for j, w in enumerate(idx):
            r, c = gs[w].shape
            for st, src in zip(stacks, (gs[w], ss[w], ns[w])):
                st[j, :r, :c] = src
        res = S.solve_advanced_batch(*stacks, four, solver.device, solver.rtol, solver.itmax, want_voltages)
        if res["rc"] == _lib.ERR_RESIDUAL:
            w = b0 + res["first_failed"]
            err = S.SolverResidualError(res["msg"].replace(f"for window {res['first_failed']} ", f"for window {w} "))
            err.window = w
            raise err
        out.iterations[b0:b0 + len(idx)] = res["iters"]
        out.relres[b0:b0 + len(idx)] = res["relres"]
        for j, w in enumerate(idx):
            r, c = gs[w].shape
            out.currents.append(np.array(res["cur"][j, :r, :c]))
            if want_voltages:
                out.voltages.append(np.array(res["volt"][j, :r, :c]))
    return out


@dataclass
class MovingWindowMap:
    """Result of moving_window_current_map."""
    current: np.ndarray            # (nrows, ncols) float64: the windows' currents summed at their positions
    iterations: np.ndarray         # per window, as OmniscapeBatch.iterations
    relres: np.ndarray             # per window, as OmniscapeBatch.relres


def moving_window_current_map(conductance, source, targets, radius, cs_cfg, *, source_scale=None, ground=np.inf,
                              circular=True, solver=None, max_batch_bytes=1 << 30) -> MovingWindowMap:
    """Omniscape's moving-window loop on the device (cs_b200_solve_moving_windows): for every target, the
    (2 radius + 1)^2 window centred on it is cut from the landscape, solved as compute_omniscape_current
    solves it, and its current raster is added into one landscape map at the window's position, in target
    order, in float64.

    conductance / source: 2-D landscape rasters of one shape, row-major (NODATA, 0 and NaN conductance =
    no node).  targets: (nwin, 2) 0-based (row, col) cells of the landscape.  A window cell is a node when
    it lies inside the landscape on a node and, with `circular`, within distance `radius` of the target.
    The window's sources are source_scale[w] * source there; its only ground is `ground[w]` (a conductance,
    > 0; Inf = direct ground) at the target.  source_scale / ground: None / a scalar / one value per target.
    Settings (`connect_four_neighbors_only`, rtol, itmax, device) are those of compute_omniscape_currents;
    float32 rasters stay float32 on the way in when both are float32.  Windows go to the device in batches
    of at most `max_batch_bytes` (S.advanced_batch_bytes per window, at least one window); the map does not
    depend on the split.  A window whose component fails the 1e-4 gate raises SolverResidualError naming
    it (`.window`)."""
    g, s = np.asarray(conductance), np.asarray(source)
    for a, name in ((g, "conductance"), (s, "source")):
        if a.ndim != 2 or a.size == 0 or not (np.issubdtype(a.dtype, np.number) or a.dtype == bool):
            raise ValueError(f"{name}: expected a non-empty numeric 2-D raster, got shape {a.shape} dtype {a.dtype}")
    if g.shape != s.shape:
        raise ValueError(f"conductance {g.shape} and source {s.shape} differ")
    t = np.asarray(targets)
    if t.size == 0:
        t = t.reshape(0, 2)
    if t.ndim != 2 or t.shape[1] != 2 or not np.issubdtype(t.dtype, np.integer):
        raise ValueError(f"targets: expected an integer (nwin, 2) array of (row, col), got shape {t.shape} "
                         f"dtype {t.dtype}")
    nwin = len(t)

    def per_window(v, name):
        a = np.asarray(v, dtype=np.float64)
        if a.ndim == 0:
            return np.full(nwin, float(a))
        if a.shape != (nwin,):
            raise ValueError(f"{name}: expected a scalar or {nwin} values, got shape {a.shape}")
        return a

    scale = None if source_scale is None else per_window(source_scale, "source_scale")
    gnd = per_window(ground, "ground")
    if max_batch_bytes <= 0:
        raise ValueError("max_batch_bytes must be positive")
    solver = solver if solver is not None else get_solver(cs_cfg)
    dtype = np.float32 if g.dtype == np.float32 and s.dtype == np.float32 else np.float64
    res = S.solve_moving_windows(g.astype(dtype, copy=False), s.astype(dtype, copy=False), t[:, 0], t[:, 1],
                                 radius, circular, scale, gnd, _flag(cs_cfg, "connect_four_neighbors_only"),
                                 solver.device, solver.rtol, solver.itmax, max_batch_bytes)
    if res["rc"] == _lib.ERR_RESIDUAL:
        err = S.SolverResidualError(res["msg"])
        err.window = res["first_failed"]
        raise err
    return MovingWindowMap(res["cum"], res["iters"], res["relres"])


@dataclass
class OmniscapeMaps:
    """Result of omniscape_current_maps (maps (nrows, ncols) float64, -9999 where the conductance is
    NaN or -9999; per-target arrays in target order)."""
    cum_currmap: np.ndarray
    flow_potential: np.ndarray | None              # None unless flow_potential was requested
    normalized_cum_currmap: np.ndarray | None      # cum_currmap / flow_potential where that is > 0, else 0
    targets: np.ndarray                            # (n, 2) int64 (row, col) block centres with amps > 0
    amps: np.ndarray                               # the source strength of each target's block
    scale: np.ndarray                              # each window's source multiplier (0: nothing to inject)
    iterations: np.ndarray                         # per conductance window, as OmniscapeBatch.iterations
    relres: np.ndarray
    fp_iterations: np.ndarray | None               # per flow-potential window
    fp_relres: np.ndarray | None


def omniscape_current_maps(conductance, source_strength, radius, cs_cfg, *, block_size=1, source_threshold=0.0,
                           flow_potential=False, solver=None, max_batch_bytes=1 << 30) -> OmniscapeMaps:
    """A whole Omniscape job on the device (cs_b200_solve_omniscape).

    conductance / source_strength: 2-D landscape rasters of one shape, row-major (NODATA, 0 and NaN
    conductance = no node).  A source counts where it is finite, above `source_threshold` and on a node.
    One target sits at the centre of every `block_size` x `block_size` block (block_size odd) whose sources
    sum to amps > 0.  Its window is the disc of `radius` around it, its sources those in the disc outside
    its block, scaled to sum to amps, its ground a direct ground at the target; the windows' currents are
    summed into cum_currmap in target order.  With `flow_potential` every window is solved once more with
    conductance 1 on every landscape cell in the disc, giving flow_potential and normalized_cum_currmap.
    Settings (`connect_four_neighbors_only`, rtol, itmax, device) are those of compute_omniscape_currents;
    float32 rasters stay float32 on the way in when both are float32.  Targets go to the device in batches
    of at most `max_batch_bytes` (S.advanced_batch_bytes per window); the maps do not depend on the split.
    A window whose component fails the 1e-4 gate raises SolverResidualError naming its target (`.window`)
    and its kind."""
    g, s = np.asarray(conductance), np.asarray(source_strength)
    for a, name in ((g, "conductance"), (s, "source_strength")):
        if a.ndim != 2 or a.size == 0 or not (np.issubdtype(a.dtype, np.number) or a.dtype == bool):
            raise ValueError(f"{name}: expected a non-empty numeric 2-D raster, got shape {a.shape} dtype {a.dtype}")
    if g.shape != s.shape:
        raise ValueError(f"conductance {g.shape} and source_strength {s.shape} differ")
    if isinstance(radius, bool) or not isinstance(radius, (int, np.integer)) or radius < 0:
        raise ValueError(f"radius must be an integer >= 0, got {radius!r}")
    if (isinstance(block_size, bool) or not isinstance(block_size, (int, np.integer)) or block_size < 1
            or block_size % 2 == 0):
        raise ValueError(f"block_size must be an odd integer >= 1, got {block_size!r}")
    if not float(source_threshold) >= 0.0:
        raise ValueError(f"source_threshold must be >= 0, got {source_threshold!r}")
    if max_batch_bytes <= 0:
        raise ValueError("max_batch_bytes must be positive")
    solver = solver if solver is not None else get_solver(cs_cfg)
    dtype = np.float32 if g.dtype == np.float32 and s.dtype == np.float32 else np.float64
    res = S.solve_omniscape(g.astype(dtype, copy=False), s.astype(dtype, copy=False), int(radius), int(block_size),
                            float(source_threshold), bool(flow_potential), _flag(cs_cfg, "connect_four_neighbors_only"),
                            solver.device, solver.rtol, solver.itmax, max_batch_bytes)
    if res["rc"] == _lib.ERR_RESIDUAL:
        err = S.SolverResidualError(res["msg"])
        err.window = res["first_failed"]
        raise err
    return OmniscapeMaps(res["cum"], res["fp"], res["normalized"], res["targets"], res["amps"], res["scale"],
                         res["iters"], res["relres"], res["fp_iters"], res["fp_relres"])


def resolve_conflicts(sources, grounds, policy):
    """src/raster/advanced.jl:119-149 (`rmvall` only zeroes the sources -- pinned upstream by
    test/internal.jl:130-135)."""
    sources = np.array(sources, dtype=np.float64)
    grounds = np.array(grounds, dtype=np.float64)
    finite = np.where(np.isfinite(grounds), grounds, 0.0)
    if not np.any(finite != 0):
        finite = np.array([NODATA])
    both = (sources != 0) & (grounds != 0)
    if policy in ("rmvsrc", "rmvall"):
        sources[both] = 0
    elif policy == "rmvgnd":
        grounds[both] = 0
    grounds[np.isinf(grounds) & (sources > 0)] = 0
    return sources, grounds, finite


def sources_and_grounds_from_maps(source_map, ground_map, nodemap, n, policy):
    """src/raster/advanced.jl:81-117 (raster branch): cell values accumulate on their node."""
    sources = np.zeros(n)
    grounds = np.zeros(n)
    for target, cmap in ((sources, source_map), (grounds, ground_map)):
        sel = (cmap != 0) & (nodemap != 0)
        np.add.at(target, nodemap[sel] - 1, cmap[sel])
    return resolve_conflicts(sources, grounds, policy)


@dataclass
class RasterData:
    """The fields of src/io.jl:34-43 the raster front ends read."""
    cellmap: np.ndarray
    polymap: np.ndarray | None
    points_rc: tuple                 # (rows, cols, ids) 1-based, sorted by id
    strengths: np.ndarray | None = None       # (P, 2) id, strength
    included_pairs: object | None = None      # .mode, .point_ids, .mat
    source_map: np.ndarray | None = None      # advanced mode: source currents per cell (unit currents applied)
    ground_map: np.ndarray | None = None      # advanced mode: ground conductances per cell, Inf = direct ground


@dataclass
class OneToAllOutput:
    resistances: np.ndarray
    curmaps: dict = field(default_factory=dict)
    voltmaps: dict = field(default_factory=dict)
    cum_curmap: np.ndarray | None = None
    max_curmap: np.ndarray | None = None
    num_solves: int = 0


# ---------------------------------------------------------------------------
# raster pairwise front end  (src/raster/pairwise.jl:14-135)
# ---------------------------------------------------------------------------
def raster_pairwise(data: RasterData, flags: Flags, cfg, solver=None, four_neighbors=False, avg_res=False,
                    sink=None) -> PairwiseOutput:
    """src/raster/pairwise.jl:14-30.  Focal points with distinct ids: one graph, single_ground_all_pairs (with
    CUDASolver(pairwise_raster=True): every component's pairs on one whole-raster handle, _raster_pairs_device).
    An id on several cells makes focal regions (_pt_file_polygons_path): every region pair is a Dirichlet
    problem on the raster's own Laplacian (region a at 0 V, region b at 1 V), so the pairs are columns of
    cs_b200_solve_region_pairs on ONE whole-raster handle; pairs that operator cannot express exactly take
    the reference's per-pair path (polygon map, graph and solve per pair).  `sink` as in `solve`."""
    from . import graph
    solver = solver or get_solver(cfg)
    cellmap, polymap = data.cellmap, data.polymap
    points_rc = tuple(np.asarray(a) for a in data.points_rc)
    inc = data.included_pairs
    exclude = set()
    regions = len(points_rc[0]) != len(np.unique(points_rc[2]))
    if inc is not None:
        points_rc, exclude = graph.generate_exclude_pairs(points_rc, inc)
    if not regions and getattr(solver, "pairwise_raster", False):
        return _raster_pairs_device(cellmap, polymap, points_rc, exclude, flags, solver, four_neighbors, avg_res,
                                    sink)
    if not regions:
        nodemap = graph.construct_node_map(cellmap, polymap)
        G = graph.laplacian(graph.construct_graph(cellmap, nodemap, avg_res, four_neighbors))
        points = nodemap[points_rc[0] - 1, points_rc[1] - 1]
        prob = GraphProblem(G, graph.connected_components(G), points, points_rc[2], exclude, nodemap, polymap,
                            cellmap, solver)
        return single_ground_all_pairs(prob, flags, cfg, sink=sink)
    return _focal_region_pairs(cellmap, polymap, points_rc, exclude, flags, solver, four_neighbors, avg_res, sink)


def _raster_pairs_device(cellmap, polymap, points_rc, exclude, flags, solver, four_neighbors, avg_res, sink):
    """`solve` for raster focal points with distinct ids (CUDASolver(pairwise_raster=True)) on ONE whole-raster
    handle: node map and operator assembled on the device, connected components labelled there
    (cs_b200_components), no host graph.  Each component's pairs come from component_pairs on its focal nodes;
    the pairs of every component are columns of the same solve_pairs / solve_sources panels (the operator is
    block-diagonal: a column's other components stay constant, so they carry no current).  Components whose
    construct_local_node_map numbers cells unlike the node map (a NODATA cell of a merged polygon) bring their
    currents back and are scattered by their own map on the host.  Returns what `solve` returns."""
    o = flags.outputflags
    shortcut = not _any_map(o) and not exclude                                   # src/core.jl:356-364
    need_curr = not shortcut
    per_pair_curr = need_curr and o.write_cur_maps and not o.write_cum_cur_map_only
    superpose = getattr(solver, "superpose", False) and not shortcut
    ids = np.asarray(points_rc[2])
    P = len(ids)
    R = -np.ones((P, P))
    voltmatrix = np.zeros((P, P))
    shortcut_res = -np.ones((P, P))
    out = PairwiseOutput(resistances=None)
    out.cum_curmap = np.zeros(cellmap.shape)
    out.max_curmap = np.full(cellmap.shape, NODATA) if o.write_max_cur_maps else None
    factor, nodemap = S.construct_raster_factor(cellmap, polymap, solver, four_neighbors=four_neighbors,
                                                avg_res=avg_res, log_transform=o.log_transform_maps)
    with factor:
        nodemap = np.asarray(nodemap, dtype=np.int64)
        _, comp_of = factor.components()
        points = nodemap[points_rc[0] - 1, points_rc[1] - 1]
        focal = np.nonzero(points != 0)[0]
        # one entry per component holding focal points, in component order: (index, focal nodes 1-based)
        fcomp = comp_of[points[focal] - 1]
        comps = [(int(ci), np.unique(points[focal[fcomp == ci]])) for ci in np.unique(fcomp)]
        columns, own, super_comps = [], {}, []      # columns: (component, src row, dst row, fan)
        for ci, cnodes in comps:
            _, solves, zero = component_pairs(points, ids, exclude, cnodes, shortcut)
            for a, b in zero:
                R[a, b] = R[b, a] = 0.0
            if not solves:
                continue
            if need_curr and polymap is not None and not _local_map_is_global(nodemap, comp_of, ci, polymap):
                rows = np.nonzero(comp_of == ci)[0]
                own[ci] = (rows, construct_local_node_map(nodemap, rows + 1, polymap))
            cols = [(ci, s - 1, d - 1, fan) for s, d, fan in solves]
            if superpose and len(solves) > 1:
                super_comps.append(cols)
            else:
                columns += cols
        if need_curr:
            factor.reset_currents()
        focal_rows = np.unique(points[focal] - 1)
        focal_col = {int(r): i for i, r in enumerate(focal_rows)}
        host_cum = {ci: (np.zeros(len(rows)), np.full(len(rows), NODATA), 0.0) for ci, (rows, _) in own.items()}
        masks = {}

        def batches():
            """(columns, result) per device call: the own-map columns apart, with accumulate=False"""
            for acc in (True, False):
                sel = [c for c in columns if (c[0] in own) != acc]
                for sl in _panels(len(sel), solver):
                    chunk = sel[sl]
                    src = np.array([c[1] for c in chunk], dtype=np.int64)
                    dst = np.array([c[2] for c in chunk], dtype=np.int64)
                    if shortcut:
                        res = _probe_solve(factor, src, dst, focal_rows, focal_col)
                    else:
                        res = factor.solve_pairs(src, dst, np.array([len(c[3]) for c in chunk], dtype=np.float64),
                                                 want_volt=o.write_volt_maps, want_curr=per_pair_curr or not acc,
                                                 accumulate=acc)
                    yield chunk, res
            for chunk in super_comps:
                acc = chunk[0][0] not in own
                src = np.array([c[1] for c in chunk], dtype=np.int64)
                dst = np.array([c[2] for c in chunk], dtype=np.int64)
                nodes, inv = np.unique(np.concatenate([src, dst]), return_inverse=True)
                yield chunk, factor.solve_pairs_superposed(
                    nodes, inv[:len(src)], inv[len(src):], np.array([len(c[3]) for c in chunk], dtype=np.float64),
                    want_volt=o.write_volt_maps, want_curr=per_pair_curr or not acc, accumulate=acc)

        def local(ci, x):
            """column x (n,) restricted to component ci, as a cell map of that component's local node map"""
            if ci in own:
                rows, lm = own[ci]
                return _scatter(np.asarray(x, dtype=np.float64)[rows], lm)
            if ci not in masks:
                masks[ci] = comp_of == ci
            return _scatter(np.where(masks[ci], np.asarray(x, dtype=np.float64), 0.0), nodemap)

        for chunk, res in batches():
            out.stats.append(factor.stats())
            out.num_solves += len(res["R"])
            out.iterations += int(res["iters"].sum())
            for col, (ci, s, d, fan) in enumerate(chunk):
                r = float(res["R"][col])
                cur = None if res.get("curr") is None else res["curr"][:, col]
                if ci in own:                          # the accumulation of `solve`'s handle, on the host
                    rows = own[ci][0]
                    c = np.asarray(cur, dtype=np.float64)[rows]
                    if o.log_transform_maps:
                        c = np.where(c > 0, np.log10(np.where(c > 0, c, 1.0)), NODATA)
                    cum, mx, w = host_cum[ci]
                    host_cum[ci] = (cum + len(fan) * c, np.maximum(mx, c), w + len(fan))
                for ci_, cj in fan:
                    R[ci_, cj] = R[cj, ci_] = r
                    key = (int(ids[ci_]), int(ids[cj]))
                    if shortcut:                                                 # src/core.jl:685-703
                        pv = res["probe_volt"][col]
                        inside = focal[fcomp == ci]
                        for i in inside[inside >= 1]:
                            voltmatrix[i, cj] = 1.0 - float(pv[focal_col[int(points[i]) - 1]]) / r
                        continue
                    _pair_maps(out, sink, key, lambda x: local(ci, x),
                               res["volt"][:, col] if o.write_volt_maps else None,
                               cur if per_pair_curr else None, cellmap, o)
        accumulated = [c for c in columns + [x for sc in super_comps for x in sc] if c[0] not in own]
        if need_curr and accumulated:
            # the device's cumulative / max vectors: a column adds f(0) (0, or -9999 under log) on every row of the
            # other components, which is what `solve` adds there per component; cells that are no node get the same
            cum, mx = factor.read_currents(want_max=True)
            _add_current_maps(out, cum, mx, nodemap, float(sum(len(c[3]) for c in accumulated)), cellmap, o)
    for ci, (cum, mx, npost) in host_cum.items():                      # as `solve` scatters one component
        _add_current_maps(out, cum, mx, own[ci][1], npost, cellmap, o)
    if shortcut:
        for ci, cnodes in comps:
            csub = [int(points[k]) for k in focal[fcomp == ci]]
            _update_shortcut_resistances(int(np.nonzero(points == csub[0])[0][0]), voltmatrix, shortcut_res, R,
                                         points, cnodes)
        R = shortcut_res
    return _finish_pairwise(out, R, ids)


@dataclass
class RegionPlan:
    """How the focal-region driver serves each id pair (i, j) (indices into `ids`, i < j): `batched`
    pairs are columns of cs_b200_solve_region_pairs with `sets[p]` (0-based rows of L0) as id p's region,
    `per_pair` pairs take the reference's per-pair path (`reasons` says why), `unconnected` pairs have
    no L0 component touching both regions (R = -1, nothing solved)."""
    ids: list
    sets: dict
    batched: list
    per_pair: list
    unconnected: list
    reasons: dict


def _region_cells(cellmap, polymap, points_rc, p):
    """Id p on the per-pair polygon map (graph.create_pair_polymap), flat column-major cell indices:
    (cells merged with p's first point, cells relabelled elsewhere).  Raises graph.RegionPolymapError."""
    from . import graph
    rr, cc_, ids = points_rc
    nr = cellmap.shape[0]
    k = int(np.nonzero(ids == p)[0][0])
    x = int((cc_[k] - 1) * nr + (rr[k] - 1))
    none = np.zeros(0, dtype=np.int64)
    if polymap is None or np.size(polymap) == 0:
        sel = ids == p
        return np.unique((cc_[sel] - 1) * nr + (rr[sel] - 1)), none
    pm = np.asarray(polymap).reshape(-1, order="F")
    mask = graph.region_relabel(np.asarray(polymap), points_rc, p)
    own = np.nonzero(pm == pm[x])[0] if pm[x] != 0 else np.array([x])
    if mask is None:
        return own, none
    q = np.nonzero(mask.reshape(-1, order="F"))[0]
    return (q, none) if mask.reshape(-1, order="F")[x] else (own, q)


def plan_region_pairs(cellmap, polymap, points_rc, exclude, nodemap, comp_of):
    """Decide each region pair's path from L0's node map (`nodemap`, 1-based, 0 = none) and component
    label per L0 node (`comp_of`, 0-based node index).  A pair is batched when, for both ids, every cell
    the per-pair polygon map merges is already an L0 node, those nodes hold no other cell, the map changes
    nothing else, and the two regions share no cell and no node."""
    from . import graph
    ids = np.asarray(points_rc[2])
    pts = list(dict.fromkeys(int(p) for p in ids))
    node_of = np.asarray(nodemap).reshape(-1, order="F")
    region, bad = {}, {}
    for p in pts:
        try:
            cells, extra = _region_cells(cellmap, polymap, points_rc, p)
        except graph.RegionPolymapError:
            bad[p] = "the reference's error branch (raised by the per-pair path)"
            continue
        nodes = node_of[cells]
        if np.any(nodes == 0):
            bad[p] = "a region cell is not a node of the raster's graph"
            continue
        s = np.unique(nodes)
        if np.count_nonzero(np.isin(node_of, s)) != len(cells):
            bad[p] = "the region's nodes hold cells outside the region"
            continue
        if len(extra) and (np.any(node_of[extra] == 0) or len(np.unique(node_of[extra])) > 1):
            bad[p] = "the polygon map merges polygons outside the region"
            continue
        region[p] = (s - 1, np.union1d(cells, extra))
    plan = RegionPlan(pts, {p: r[0] for p, r in region.items()}, [], [], [], {})
    for i in range(len(pts)):
        for j in range(i + 1, len(pts)):
            a, b = pts[i], pts[j]
            if (a, b) in exclude or (b, a) in exclude:
                continue
            why = bad.get(a) or bad.get(b)
            if why is None and (np.intersect1d(region[a][0], region[b][0]).size or
                                np.intersect1d(region[a][1], region[b][1]).size):
                why = "the two regions overlap"
            if why is not None:
                plan.per_pair.append((i, j))
                plan.reasons[(i, j)] = why
            elif np.intersect1d(comp_of[region[a][0]], comp_of[region[b][0]]).size:
                plan.batched.append((i, j))
            else:
                plan.unconnected.append((i, j))
    return plan


def _focal_region_pairs(cellmap, polymap, points_rc, exclude, flags, solver, four_neighbors, avg_res, sink):
    """src/raster/pairwise.jl:72-135 on one whole-raster operator (see raster_pairwise).  With
    CUDASolver(front_end_on_device=True) the node map and component labels come from that handle (created first)
    instead of a host graph; the per-pair path still builds its own."""
    from . import graph
    o = flags.outputflags
    want_maps = _any_map(o)
    per_pair_curr = o.write_cur_maps and not o.write_cum_cur_map_only
    factor = None
    if getattr(solver, "front_end_on_device", False):       # node map and labels from the whole-raster handle
        factor, nodemap = S.construct_raster_factor(cellmap, polymap, solver, four_neighbors=four_neighbors,
                                                    avg_res=avg_res, log_transform=o.log_transform_maps)
        try:
            nodemap = np.asarray(nodemap, dtype=np.int64)
            comp_of = factor.components()[1]
            plan = plan_region_pairs(cellmap, polymap, points_rc, exclude, nodemap, comp_of)
        except BaseException:
            factor.close()
            raise
        if not plan.batched:
            factor.close()
    else:
        nodemap = graph.construct_node_map(cellmap, polymap)
        _, comp_of = _component_labels(graph.construct_graph(cellmap, nodemap, avg_res, four_neighbors))
        plan = plan_region_pairs(cellmap, polymap, points_rc, exclude, nodemap, comp_of)
    pts = plan.ids
    P = len(pts)
    R = -np.ones((P, P))
    out = PairwiseOutput(resistances=None)
    out.cum_curmap = np.zeros(cellmap.shape)
    out.max_curmap = np.full(cellmap.shape, NODATA) if o.write_max_cur_maps else None
    if plan.batched:
        if factor is None:
            factor = _raster_factor(cellmap, polymap, nodemap, solver, four_neighbors, avg_res, o.log_transform_maps)
        with factor:
            used = sorted({pts[i] for i, _ in plan.batched} | {pts[j] for _, j in plan.batched})
            slot = {p: s for s, p in enumerate(used)}
            sets = [plan.sets[p] for p in used]
            if want_maps:
                factor.reset_currents()
            for sl in _panels(len(plan.batched), solver):
                chunk = plan.batched[sl]
                res = factor.solve_region_pairs(sets, [slot[pts[i]] for i, _ in chunk],
                                                [slot[pts[j]] for _, j in chunk], want_volt=o.write_volt_maps,
                                                want_curr=per_pair_curr, accumulate=want_maps)
                out.stats.append(factor.stats())
                out.num_solves += len(chunk)
                out.iterations += int(res["iters"].sum())
                for col, (i, j) in enumerate(chunk):
                    R[i, j] = R[j, i] = float(res["R"][col])
                    _pair_maps(out, sink, (pts[i], pts[j]), lambda x: _scatter(x.astype(np.float64), nodemap),
                               res["volt"][:, col] if o.write_volt_maps else None,
                               res["curr"][:, col] if per_pair_curr else None, cellmap, o)
            if want_maps:
                # the per-node accumulation of every batched pair, as core.solve scatters it
                cum, mx = factor.read_currents(want_max=True)
                _add_current_maps(out, cum, mx, nodemap, float(len(plan.batched)), cellmap, o)
    rr, cc_, ids = points_rc
    for i, j in plan.per_pair:                                   # the reference's own algorithm
        p1, p2 = pts[i], pts[j]
        newpoly = graph.create_pair_polymap(cellmap, polymap, points_rc, p1, p2)
        nm = graph.construct_node_map(cellmap, newpoly)
        G = graph.laplacian(graph.construct_graph(cellmap, nm, avg_res, four_neighbors))
        x = int(np.nonzero(ids == p1)[0][0])
        y = int(np.nonzero(ids == p2)[0][0])
        pn = np.array([nm[rr[x] - 1, cc_[x] - 1], nm[rr[y] - 1, cc_[y] - 1]])
        r = single_ground_all_pairs(GraphProblem(G, graph.connected_components(G), pn, np.array([p1, p2]), set(),
                                                 nm, newpoly, cellmap, solver), flags, sink=sink)
        R[i, j] = R[j, i] = r.resistances[1, 2]
        out.num_solves += r.num_solves
        out.iterations += r.iterations
        out.voltmaps.update(r.voltmaps)
        out.curmaps.update(r.curmaps)
        out.cum_curmap += r.cum_curmap
        if out.max_curmap is not None:
            out.max_curmap = np.maximum(out.max_curmap, r.max_curmap)
    # every pair's map goes into one shared cumulative map, clamped once when it is written
    # (write_cum_maps -> postprocess_cum_curmap!, src/out.jl:467-479): a cell that is NODATA in every pair's
    # map stays NODATA instead of adding up to -9999 * pairs
    return _finish_pairwise(out, R, pts)


def _one_to_all_batched_raster(G, comps, nodemap, newpoly, point_map, unique_point_map, uniq, rr, cc_,
                               strengths, solver):
    """One-to-all without include/exclude lists: iteration p puts a current source on focal node p and
    ties every OTHER focal node to ground (src/raster/onetoall.jl:100-109).  With F the focal nodes of
    a component and N the rest, all iterations share B = L[N, N] (the Laplacian with every focal
    row/column deleted, SPD); block elimination of the one live focal node gives
        B w_p = -L[N, p] ,   v_p = s_p / (L[p, p] + L[p, N] w_p) ,   v_N = v_p w_p ,   v = 0 on the other focal nodes,
    so the iterations of a component are columns of ONE n_N x |F| batch on one factor (hook #2) instead
    of one factor + solve per iteration.  Returns {iteration: (voltage raster, current raster,
    source-cell voltage / strength)}; iterations it cannot serve take the per-iteration path."""
    n_nodes = G.shape[0]
    if strengths is not None and len(strengths) != len(uniq):
        return {}
    comp_of = np.zeros(n_nodes + 1, dtype=np.int64) - 1
    for ci, comp in enumerate(comps):
        comp_of[np.asarray(comp)] = ci
    plans = {}
    for i, n in enumerate(uniq):
        if point_map.sum() == n:
            continue
        strv = float(strengths[i, 1]) if strengths is not None else 1.0
        source_map = np.where(unique_point_map == n, strv, 0.0)
        ground_map = np.where((point_map != n) & (point_map > 0), np.inf, 0.0)
        s_, g_, f_ = sources_and_grounds_from_maps(source_map, ground_map, nodemap, n_nodes, "rmvgnd")
        check_node = nodemap[rr[i] - 1, cc_[i] - 1]
        snodes = np.nonzero(s_ != 0)[0]
        if len(snodes) != 1 or f_[0] != NODATA or check_node == 0 or not np.all(np.isinf(g_[g_ != 0])):
            continue
        ci = comp_of[check_node]
        if ci < 0 or comp_of[snodes[0] + 1] != ci:
            continue
        rows = np.asarray(comps[ci]) - 1
        if not np.any(np.isinf(g_[rows])):
            continue                                   # no ground in this component: nothing is solved
        plans.setdefault(ci, []).append((i, int(snodes[0]), float(s_[snodes[0]]),
                                         frozenset(np.nonzero(np.isinf(g_[rows]))[0].tolist())))
    served = {}
    for ci, items in plans.items():
        rows = np.asarray(comps[ci]) - 1
        local = np.zeros(n_nodes, dtype=np.int64) - 1
        local[rows] = np.arange(len(rows))
        a_local = G[rows][:, rows].tocsr()
        F = sorted({int(local[p]) for _, p, _, _ in items} | set().union(*[g for *_x, g in items]))
        # every served iteration must ground exactly F minus its own source node
        items = [it for it in items if it[3] == frozenset(F) - {int(local[it[1]])}]
        if not items or len(F) >= len(rows):
            continue
        Nidx = np.setdiff1d(np.arange(len(rows)), F)
        B = a_local[Nidx][:, Nidx].tocsr()
        cols = [int(local[p]) for _, p, _, _ in items]
        rhs = -a_local[Nidx][:, cols].toarray()
        if not np.any(rhs):
            continue
        live = np.nonzero(np.abs(rhs).sum(axis=0) > 0)[0]
        W = np.zeros_like(rhs)
        with S.construct_cholesky_factor(B, solver) as factor:
            W[:, live] = np.asarray(S.solve_linear_system(factor, B, np.asfortranarray(rhs[:, live]))).reshape(len(Nidx), -1)
        lm = construct_local_node_map(nodemap, np.asarray(comps[ci]), newpoly)
        for c, (i, p, sval, _) in enumerate(items):
            pl = cols[c]
            lpn = a_local[pl, Nidx].toarray().ravel()
            denom = a_local[pl, pl] + lpn @ W[:, c]
            v = np.zeros(len(rows))
            v[pl] = sval / denom
            v[Nidx] = v[pl] * W[:, c]
            cur = node_currents_host(a_local, v, None)
            # the reported value is read off the voltage RASTER at the source cell, through the local
            # node map, exactly as the per-iteration path does (advanced.jl:252-263) -- with a NODATA
            # cell inside a focal region the local numbering can differ from the matrix's
            volt = np.zeros(lm.shape)
            volt[lm != 0] = v[lm[lm != 0] - 1]
            smap = np.where(unique_point_map == uniq[i], sval, 0.0)
            val = (volt[smap != 0] / smap[smap != 0])[0]
            served[i] = (_scatter(v, lm), _scatter(cur, lm), val)
    return served


def _all_to_one_batched_raster(G, comps, nodemap, newpoly, point_map, unique_point_map, uniq, rr, cc_,
                                strengths, solver, o):
    """All-to-one without include/exclude lists: every iteration keeps the same node map and operator
    and differs only in which focal node is tied to ground, so the iterations of one connected
    component are columns of ONE sparse-RHS batch on the component's singular Laplacian
    (cs_b200_solve_sources; ground = reference row carrying minus the summed sources) instead of
    one factor + solve per iteration (src/raster/onetoall.jl:110-151 through
    src/raster/advanced.jl:274-305).  Returns {iteration index: (voltage raster, current raster)}
    for the iterations it could serve; the caller runs the rest through the per-iteration path."""
    n_nodes = G.shape[0]
    strength_map = None
    if strengths is not None:
        strength_map = np.zeros(point_map.shape)
        strength_map[rr - 1, cc_ - 1] = strengths[:, 1] if len(strengths) == len(rr) else 0.0
        if len(strengths) != len(rr):
            return {}
    plans = {}      # component index -> list of (iteration, ground node, source nodes, source values)
    comp_of = np.zeros(n_nodes + 1, dtype=np.int64) - 1
    for ci, comp in enumerate(comps):
        comp_of[np.asarray(comp)] = ci
    for i, n in enumerate(uniq):
        if point_map.sum() == n:
            continue
        if strength_map is not None:
            source_map = np.where(unique_point_map == n, 0.0, strength_map)
        else:
            source_map = np.where((unique_point_map != 0) & (point_map != n), 1.0, 0.0)
        ground_map = np.where(point_map == n, np.inf, 0.0)
        s_, g_, f_ = sources_and_grounds_from_maps(source_map, ground_map, nodemap, n_nodes, "rmvsrc")
        gnodes = np.nonzero(np.isinf(g_))[0]
        check_node = nodemap[rr[i] - 1, cc_[i] - 1]
        if len(gnodes) != 1 or f_[0] != NODATA or check_node == 0:
            continue                                   # several ground nodes: per-iteration path
        ci = comp_of[check_node]
        if ci < 0 or comp_of[gnodes[0] + 1] != ci:
            continue
        rows = np.asarray(comps[ci]) - 1
        local = np.zeros(n_nodes, dtype=np.int64) - 1
        local[rows] = np.arange(len(rows))
        src_nodes = np.nonzero(s_[rows] != 0)[0]
        if len(src_nodes) == 0:
            continue
        plans.setdefault(ci, []).append((i, int(local[gnodes[0]]), src_nodes, s_[rows][src_nodes]))
    served = {}
    for ci, items in plans.items():
        rows = np.asarray(comps[ci]) - 1
        a_local = G[rows][:, rows].tocsr()
        lm = construct_local_node_map(nodemap, np.asarray(comps[ci]), newpoly)
        columns, refs = [], []
        for _, gl, sn, sv in items:
            columns.append((np.concatenate([sn, [gl]]), np.concatenate([sv, [-sv.sum()]])))
            refs.append(gl)
        with S.construct_cholesky_factor(a_local, solver) as factor:
            r = factor.solve_sources(columns, refs, want_volt=True, want_curr=True)
        for c, (i, *_rest) in enumerate(items):
            served[i] = (_scatter(r["volt"][:, c].astype(np.float64), lm),
                         _scatter(r["curr"][:, c].astype(np.float64), lm))
    return served


@dataclass
class OneToAllColumn:
    """One iteration as a column on the whole-raster operator L0: `ground` (0-based rows, sorted) at 0 V,
    `vals` injected at `rows` (0-based, sorted), both inside L0 component `comp`; `strength` divides the
    one-to-all source voltage into the reported value."""
    i: int
    comp: int
    ground: np.ndarray
    rows: np.ndarray
    vals: np.ndarray
    strength: float


@dataclass
class OneToAllPlan:
    """How CUDASolver(onetoall_raster=True) serves each iteration i (index into `ids`): `columns` are solved
    on one whole-raster handle; `skipped[i] = (value, emits)` need no solve (`emits`: the iteration still
    writes all-zero maps, as the loop does when no component is solved); `per_iteration` take the existing
    loop (`reasons[i]` says why)."""
    ids: list
    columns: list
    skipped: dict
    per_iteration: list
    reasons: dict


def _local_map_is_global(nodemap, comp_of, ci, newpoly):
    """Whether construct_local_node_map of component `ci` numbers its cells like L0 restricted to the
    component (utils.jl:10-30 renumbers column-major; a NODATA cell of a merged polygon can move a node)."""
    comp = np.nonzero(comp_of == ci)[0] + 1
    if len(comp) == len(comp_of):
        return True
    lm = construct_local_node_map(nodemap, comp, newpoly)
    rank = np.zeros(len(comp_of) + 1, dtype=np.int64)
    rank[comp] = np.arange(1, len(comp) + 1)
    return np.array_equal(lm, rank[nodemap])


def plan_onetoall(gmap, newpoly, points_rc, nodemap, comp_of, one_to_all, strengths=None, included_pairs=None):
    """Sort the iterations of onetoall_kernel from L0's node map (`nodemap`, 1-based, 0 = none, built from
    `newpoly`) and component label per L0 node (`comp_of`, 0-based node index).  Works on the focal cells
    only; reproduces the loop's source / ground maps (onetoall.jl:93-118), sources_and_grounds_from_maps
    with rmvgnd / rmvsrc, the component picked through row i of points_rc (sic, onetoall.jl:120) and the
    sum tests of advanced.jl:186-196."""
    rr, cc_, ids = (np.asarray(a) for a in points_rc)
    uniq = list(dict.fromkeys(int(p) for p in ids))
    plan = OneToAllPlan(uniq, [], {}, [], {})
    if included_pairs is not None:
        for i in range(len(uniq)):
            plan.per_iteration.append(i)
            plan.reasons[i] = "an include/exclude list: the loop builds each iteration's node map (onetoall.jl:88-90)"
        return plan
    nr, nc = gmap.shape
    flat = ((cc_ - 1) * nr + (rr - 1)).astype(np.int64)          # column-major cell of each point row
    node_of = np.asarray(nodemap).reshape(-1, order="F")
    pm = {}                                                      # point_map: the last row on a cell wins
    for x, p in zip(flat.tolist(), ids.tolist()):
        pm[x] = int(p)
    upm = {}                                                     # unique_point_map: each id's first cell
    for p in uniq:
        upm[int(flat[int(np.nonzero(ids == p)[0][0])])] = p
    smap = None
    if strengths is not None:                                    # onetoall.jl:93-101 (raises like the loop)
        st = np.array(strengths, dtype=np.float64)
        st[np.array([pm[x] for x in flat.tolist()]) == 0, 1] = 1
        sm = np.zeros(gmap.shape)
        sm[rr - 1, cc_ - 1] = st[:, 1]
        smf = sm.reshape(-1, order="F")
        smap = {x: float(smf[x]) for x in pm}
    pm_sum = sum(pm.values())
    rowmajor = lambda x: (x % nr) * nc + x // nr                 # np.add.at visits cells in C order
    lm_ok = {}
    for i, n in enumerate(uniq):
        if pm_sum == n:                                          # no other focal node left
            plan.skipped[i] = (-1.0, False)
            continue
        strv = 1.0
        if one_to_all:
            strv = float(strengths[i, 1]) if strengths is not None else 1.0
            src = [(x, strv) for x, p in upm.items() if p == n]
            gnd = [x for x, p in pm.items() if p != n and p > 0]
        else:
            if smap is not None:
                src = [(x, v) for x, v in smap.items() if upm.get(x) != n]
            else:
                src = [(x, 1.0) for x, p in upm.items() if p != 0 and pm[x] != n]
            gnd = [x for x, p in pm.items() if p == n]
        s = {}
        for x, v in sorted(src, key=lambda t: rowmajor(t[0])):
            if v != 0 and node_of[x] != 0:
                s[int(node_of[x]) - 1] = s.get(int(node_of[x]) - 1, 0.0) + v
        s = {k: v for k, v in s.items() if v != 0}
        g = {int(node_of[x]) - 1 for x in gnd if node_of[x] != 0}
        if one_to_all:
            g -= set(s)                                          # rmvgnd
        else:
            s = {k: v for k, v in s.items() if k not in g}       # rmvsrc
        check_node = int(node_of[flat[i]])                       # (sic) row i of points_rc
        if check_node == 0:
            plan.skipped[i] = (-1.0, True)
            continue
        ci = int(comp_of[check_node - 1])
        rows = np.array(sorted(k for k in s if comp_of[k] == ci), dtype=np.int64)
        vals = np.array([s[k] for k in rows.tolist()], dtype=np.float64)
        ground = np.array(sorted(k for k in g if comp_of[k] == ci), dtype=np.int64)
        if vals.sum() == 0 or len(ground) == 0:                  # advanced.jl:194-196: nothing solved
            plan.skipped[i] = (-1.0, True)
            continue
        if ci not in lm_ok:
            lm_ok[ci] = _local_map_is_global(nodemap, comp_of, ci, newpoly)
        if not lm_ok[ci]:
            plan.per_iteration.append(i)
            plan.reasons[i] = "the component's local node map numbers cells unlike L0 (utils.jl:10-30)"
            continue
        plan.columns.append(OneToAllColumn(i, ci, ground, rows, vals, strv))
    return plan


def _onetoall_columns(plan, factor, nodemap, comp_of, one_to_all, o, solver):
    """Solve the plan's columns on the open whole-raster handle `factor`.  one-to-all and all-to-one iterations with
    several ground rows: cs_b200_solve_grounded (Dirichlet rows at the grounds); all-to-one with one ground
    row: the singular form of cs_b200_solve_sources (ref = the ground), whose voltages outside the
    component are zeroed here.  Node currents go into the handle's cumulative / max vectors.
    -> ({i: (value, voltmap | None, curmap | None)}, cumulative map, max map | None, iterations)."""
    want_v = o.write_volt_maps
    want_c = o.write_cur_maps or o.write_cum_cur_map_only
    served = {}
    iters = 0
    factor.reset_currents()
    singular = lambda c: (not one_to_all) and len(c.ground) == 1
    for kind in (False, True):
        cols = [c for c in plan.columns if singular(c) == kind]
        for sl in _panels(len(cols), solver):
            chunk = cols[sl]
            if kind:
                res = factor.solve_sources(
                    [(np.r_[c.rows, c.ground], np.r_[c.vals, -c.vals.sum()]) for c in chunk],
                    [int(c.ground[0]) for c in chunk], want_volt=want_v, want_curr=want_c, accumulate=True)
            else:
                res = factor.solve_grounded([c.ground for c in chunk], np.arange(len(chunk)),
                                            [(c.rows, c.vals) for c in chunk], want_volt=want_v,
                                            want_curr=want_c, accumulate=True)
            iters += int(res["iters"].sum())
            for col, c in enumerate(chunk):
                val = 0.0
                if one_to_all:
                    val = float(res["src_volt"][col]) / c.strength
                    val = -1.0 if np.isclose(val, 0) else val               # advanced.jl:252-263
                out = comp_of != c.comp
                vm = cm = None
                if want_v:
                    v = np.asarray(res["volt"][:, col], dtype=np.float64).copy()
                    v[out] = 0.0
                    vm = _scatter(v, nodemap)
                if want_c:
                    cur = np.asarray(res["curr"][:, col], dtype=np.float64).copy()
                    cur[out] = 0.0
                    cm = _scatter(cur, nodemap)
                served[c.i] = (val, vm, cm)
    cum, mx = factor.read_currents(want_max=o.write_max_cur_maps)
    cmap = _scatter(np.asarray(cum, dtype=np.float64), nodemap)
    mmap = None if mx is None or not plan.columns else _scatter(np.asarray(mx, dtype=np.float64), nodemap)
    return served, cmap, mmap, iters


def _onetoall_output(plan, device, gmap, o, out=None, res=None):
    """The results of the iterations the plan keeps out of the loop, into `out` / `res`; with out=None a
    new, finished OneToAllOutput (the loop's NODATA clamp of the cumulative map included)."""
    finish = out is None
    if finish:
        out = OneToAllOutput(resistances=None)
        out.cum_curmap = np.zeros(gmap.shape)
        out.max_curmap = np.full(gmap.shape, NODATA) if o.write_max_cur_maps else None
        res = np.zeros(len(plan.ids))
    served = device.get("served", {})
    for i, n in enumerate(plan.ids):
        if i in plan.skipped:
            res[i], emits = plan.skipped[i]
            if not emits:
                continue
            if o.write_volt_maps:
                out.voltmaps[n] = np.zeros(gmap.shape)
            if o.write_cur_maps or o.write_cum_cur_map_only:
                out.curmaps[n] = np.zeros(gmap.shape)
            if out.max_curmap is not None:
                out.max_curmap = np.maximum(out.max_curmap, 0.0)
        elif i in served:
            res[i], vm, cm = served[i]
            out.num_solves += 1
            if vm is not None:
                out.voltmaps[n] = vm
            if cm is not None:
                out.curmaps[n] = cm
    if device:
        out.cum_curmap += device["cum"]
        if out.max_curmap is not None and device["max"] is not None:
            out.max_curmap = np.maximum(out.max_curmap, device["max"])
    if finish:
        out.resistances = np.column_stack([plan.ids, res])
        out.cum_curmap = np.where(out.cum_curmap < NODATA, NODATA, out.cum_curmap)
    return out


def onetoall_kernel(data: RasterData, flags: Flags, cfg, solver=None, one_to_all=None,
                    four_neighbors=False, avg_res=False) -> OneToAllOutput:
    """src/raster/onetoall.jl:13-167.  One advanced-mode solve per focal id: one-to-all = unit
    (or variable-strength) source at the focal node, every other focal node a direct ground;
    all-to-one = the reverse.  Every solve goes through `multiple_solver` -> hook #3.  With
    CUDASolver(onetoall_raster=True, front_end_on_device=True) and no include / exclude list the whole-raster handle
    is created first and gives the node map and component labels; the host graph is built only when some iteration
    takes the loop."""
    from . import graph
    solver = solver or get_solver(cfg)
    if one_to_all is None:
        one_to_all = cfg.get("scenario") in ("one-to-all", "one_to_all")
    o = flags.outputflags
    gmap, polymap = data.cellmap, data.polymap
    rr, cc_, ids = (np.asarray(a) for a in data.points_rc)
    strengths = None if data.strengths is None else np.array(data.strengths, dtype=np.float64)
    inc = data.included_pairs
    mode = 0 if (inc is not None and inc.mode == "include") else 1
    if inc is not None:
        keep = np.isin(ids, inc.point_ids)
        rr, cc_, ids = rr[keep], cc_[keep], ids[keep]
        if strengths is not None:
            strengths = strengths[np.isin(strengths[:, 0], inc.point_ids)]
    points_rc = (rr, cc_, ids)
    point_map = np.zeros(gmap.shape, dtype=np.int64)
    point_map[rr - 1, cc_ - 1] = ids
    uniq = list(dict.fromkeys(int(p) for p in ids))
    newpoly = graph.create_new_polymap(gmap, polymap, points_rc, point_map)
    device, plan = {}, None
    onetoall_raster = getattr(solver, "onetoall_raster", False)   # precedence over batch_one_to_all / batch_all_to_one
    columns = lambda factor: dict(zip(("served", "cum", "max", "iters"),
                                      _onetoall_columns(plan, factor, nodemap, comp_of, one_to_all, o, solver)))
    if onetoall_raster and inc is None and getattr(solver, "front_end_on_device", False):
        # node map and component labels from the whole-raster handle; the host graph only for the loop's iterations
        factor, nodemap = S.construct_raster_factor(gmap, newpoly, solver, four_neighbors=four_neighbors,
                                                    avg_res=avg_res)
        with factor:
            nodemap = np.asarray(nodemap, dtype=np.int64)
            comp_of = factor.components()[1]
            plan = plan_onetoall(gmap, newpoly, points_rc, nodemap, comp_of, one_to_all, strengths, inc)
            if plan.columns:
                device = columns(factor)
        if not plan.per_iteration:
            return _onetoall_output(plan, device, gmap, o)
        adj = graph.construct_graph(gmap, nodemap, avg_res, four_neighbors)
    else:
        nodemap = graph.construct_node_map(gmap, newpoly)
        adj = graph.construct_graph(gmap, nodemap, avg_res, four_neighbors)
        if onetoall_raster:
            comp_of = _component_labels(adj.copy())[1]
            plan = plan_onetoall(gmap, newpoly, points_rc, nodemap, comp_of, one_to_all, strengths, inc)
            if plan.columns:
                with _raster_factor(gmap, newpoly, nodemap, solver, four_neighbors, avg_res) as factor:
                    device = columns(factor)
            if not plan.per_iteration:
                return _onetoall_output(plan, device, gmap, o)
    comps = graph.connected_components(adj)
    G = graph.laplacian(adj)
    first = {p: int(np.nonzero(ids == p)[0][0]) for p in uniq}
    unique_point_map = np.zeros(gmap.shape, dtype=np.int64)
    for p, k in first.items():
        unique_point_map[rr[k] - 1, cc_[k] - 1] = p
    out = OneToAllOutput(resistances=None)
    out.cum_curmap = np.zeros(gmap.shape)
    out.max_curmap = np.full(gmap.shape, NODATA) if o.write_max_cur_maps else None
    res = np.zeros(len(uniq))
    strength_map = np.zeros(gmap.shape) if strengths is not None else None
    batched = {}
    if (not one_to_all) and inc is None and plan is None and getattr(solver, "batch_all_to_one", False):
        batched = _all_to_one_batched_raster(G, comps, nodemap, newpoly, point_map, unique_point_map, uniq,
                                             rr, cc_, strengths, solver, o)
    batched1 = {}
    if one_to_all and inc is None and plan is None and getattr(solver, "batch_one_to_all", False):
        batched1 = _one_to_all_batched_raster(G, comps, nodemap, newpoly, point_map, unique_point_map, uniq,
                                              rr, cc_, strengths, solver)
    resident_factors = {}          # CUDASolver(resident_grounds=True): one device factor per component

    def record(n, outvolt, outcurr):
        """iteration n's voltage and current rasters into the output maps"""
        if o.write_volt_maps:
            out.voltmaps[n] = outvolt
        if o.write_cur_maps or o.write_cum_cur_map_only:
            out.curmaps[n] = outcurr
        out.cum_curmap += outcurr
        if out.max_curmap is not None:
            out.max_curmap = np.maximum(out.max_curmap, outcurr)

    for i, n in enumerate(uniq):
        if plan is not None and i not in plan.reasons:              # served by the plan (_onetoall_output)
            continue
        pm, nm, npoly = point_map.copy(), nodemap, newpoly
        if inc is not None:
            for j, other in enumerate(inc.point_ids):
                if i != j and inc.mat[i, j] == mode:
                    pm[pm == int(other)] = 0
            npoly = graph.create_new_polymap(gmap, polymap, points_rc, pm)
            nm = graph.construct_node_map(gmap, polymap)            # (sic) onetoall.jl:88
        if strengths is not None:
            st = strengths.copy()
            st[pm[rr - 1, cc_ - 1] == 0, 1] = 1
            strength_map[rr - 1, cc_ - 1] = st[:, 1]
        if pm.sum() == n:                                           # no other focal node left
            res[i] = -1
            continue
        if i in batched1:                                           # one-to-all column of the grounded batch
            outvolt, outcurr, val = batched1[i]
            out.num_solves += 1
            res[i] = -1 if np.isclose(val, 0) else val               # advanced.jl:252-263
            record(n, outvolt, outcurr)
            continue
        if i in batched:                                            # solved as a column of the batch
            outvolt, outcurr = batched[i]
            out.num_solves += 1
            res[i] = 0
            record(n, outvolt, outcurr)
            continue
        if one_to_all:
            strv = strengths[i, 1] if strengths is not None else 1.0
            source_map = np.where(unique_point_map == n, float(strv), 0.0)
            ground_map = np.where((pm != n) & (pm > 0), np.inf, 0.0)
            policy = "rmvgnd"
        else:
            if strengths is not None:
                source_map = np.where(unique_point_map == n, 0.0, strength_map)
            else:
                source_map = np.where((unique_point_map != 0) & (pm != n), 1.0, 0.0)
            ground_map = np.where(pm == n, np.inf, 0.0)
            policy = "rmvsrc"
        check_node = nm[rr[i] - 1, cc_[i] - 1]                      # (sic) row i of points_rc
        s_, g_, f_ = sources_and_grounds_from_maps(source_map, ground_map, nm, G.shape[0], policy)
        volt = np.zeros(gmap.shape)
        outvolt, outcurr, called = np.zeros(gmap.shape), np.zeros(gmap.shape), False
        for comp in comps:
            if check_node not in comp:                               # advanced.jl:186-188
                continue
            rows = np.asarray(comp) - 1
            sl, gl = s_[rows].copy(), g_[rows].copy()
            if sl.sum() == 0 or gl.sum() == 0:
                continue
            fl = f_[rows] if f_[0] != NODATA else f_
            a_local = G[rows][:, rows].tocsr()
            v = multiple_solver(cfg, solver, a_local, sl, gl, fl,
                                resident=(resident_factors, tuple(rows[:2]) + (len(rows),))
                                if getattr(solver, "resident_grounds", False) else None)
            out.num_solves += 1
            lm = construct_local_node_map(nm, np.asarray(comp), npoly)
            called = True
            outvolt += _scatter(v, lm)
            outcurr += _scatter(node_currents_host(a_local, v, fl), lm)
            volt[lm != 0] = v[lm[lm != 0] - 1]
        if not called:
            res[i] = -1                                              # advanced.jl:246-250
        elif one_to_all:
            val = volt[source_map != 0] / source_map[source_map != 0]
            res[i] = -1 if np.isclose(val[0], 0) else val[0]         # advanced.jl:252-263
        else:
            res[i] = 0
        record(n, outvolt, outcurr)
    for f in resident_factors.values():
        f.close()
    if plan is not None:
        _onetoall_output(plan, device, gmap, o, out, res)
    out.resistances = np.column_stack([uniq, res])
    out.cum_curmap = np.where(out.cum_curmap < NODATA, NODATA, out.cum_curmap)
    return out


# ---------------------------------------------------------------------------
# raster advanced mode on one whole-raster operator  (src/raster/advanced.jl:17-80, 151-305)
# ---------------------------------------------------------------------------
def _advanced_front_end_device(data, solver, four_neighbors, avg_res, policy):
    """raster_advanced's front end on the whole-raster handle (CUDASolver(front_end_on_device=True)): the node map
    from the create, the columns from B200Factor.plan_advanced, which also applies the finite grounds.  No host
    graph.  Returns (open factor, nodemap, n, columns as raster_advanced builds them, solved components)."""
    factor, nodemap = S.construct_raster_factor(data.cellmap, data.polymap, solver, four_neighbors=four_neighbors,
                                                avg_res=avg_res)
    try:
        nodemap = np.asarray(nodemap, dtype=np.int64)
        plan = factor.plan_advanced(nodemap, data.source_map, data.ground_map, policy)
        col_of_row = np.asarray(plan["col_of_row"], dtype=np.int64)
        k = len(plan["col_comp"])
        # each column's rows, ascending: the rows of its component (the rows of col -1 belong to no column)
        groups = np.split(np.argsort(col_of_row, kind="stable"),
                          np.cumsum(np.bincount(col_of_row + 1, minlength=k + 1))[:-1])[1:]
        sp_, sq = plan["set_ptr"], plan["src_ptr"]
        columns = []
        for j, rows in enumerate(groups):
            lm = None
            if data.polymap is not None and not _local_map_is_global(nodemap, col_of_row, j, data.polymap):
                lm = construct_local_node_map(nodemap, rows + 1, data.polymap)
            columns.append((rows, plan["set_rows"][sp_[j]:sp_[j + 1]], plan["src_rows"][sq[j]:sq[j + 1]],
                            plan["src_vals"][sq[j]:sq[j + 1]], lm))
    except BaseException:
        factor.close()
        raise
    return factor, nodemap, factor.n, columns, int(plan["nsolved"])


def raster_advanced(data: RasterData, flags: Flags, cfg, solver=None, four_neighbors=False,
                    avg_res=False) -> AdvancedOutput:
    """src/raster/advanced.jl raster_advanced / compute_advanced_data / advanced_kernel: every connected
    component with sum(sources) != 0 and sum(grounds) != 0 is one column of cs_b200_solve_advanced on ONE
    whole-raster handle, its Inf grounds a Dirichlet set at 0 V, the finite grounds on the operator's
    diagonal (set_grounds, once).  Each column meets its own stop rule, residual gate and 1e-8 current cut,
    as the reference's per-component solve does.  `data.source_map` / `data.ground_map` are the maps as
    io.jl delivers them (ground conductances, Inf for direct grounds, unit currents applied); the policy is
    cfg's remove_src_or_gnd.  Returns AdvancedOutput: voltmap (the column voltages scattered by the node
    map), curmap (the node currents summed over the columns, no log transform or nodata), voltages per node,
    and result: the voltage raster, or the 1 x 1 [-1] when no component was solved (advanced.jl:246-249).
    With CUDASolver(front_end_on_device=True) the handle is created first and its plan_advanced gives the columns
    and applies the finite grounds (_advanced_front_end_device): no host graph, labels or node values."""
    from . import graph
    solver = solver or get_solver(cfg)
    cellmap, polymap = data.cellmap, data.polymap
    policy = cfg.get("remove_src_or_gnd", "keepall")
    factor, f = None, None
    t0 = time.perf_counter()
    if getattr(solver, "front_end_on_device", False):
        factor, nodemap, n, columns, solved = _advanced_front_end_device(data, solver, four_neighbors, avg_res, policy)
    else:
        nodemap = graph.construct_node_map(cellmap, polymap)
        adj = graph.construct_graph(cellmap, nodemap, avg_res, four_neighbors)
        n = adj.shape[0]
        ncomp, comp_of = _component_labels(adj)
        s, g, f = sources_and_grounds_from_maps(np.asarray(data.source_map, dtype=np.float64),
                                                np.asarray(data.ground_map, dtype=np.float64), nodemap, n, policy)
        order = np.argsort(comp_of, kind="stable")
        comps = np.split(order, np.cumsum(np.bincount(comp_of, minlength=ncomp))[:-1]) if n else []
        # one column per solved component: (its rows, Inf-ground rows, source rows, values, local node map or
        # None when construct_local_node_map numbers the component like the node map, utils.jl:10-30)
        columns, solved = [], 0
        for ci, rows in enumerate(comps):
            if s[rows].sum() == 0 or g[rows].sum() == 0:              # advanced.jl:194-196
                continue
            solved += 1
            inf = g[rows] == np.inf
            src = rows[(s[rows] != 0) & ~inf]                         # sources on Inf grounds are deleted
            if not len(src):
                continue                                              # b = 0: the component stays at 0 V
            lm = None
            if polymap is not None and not _local_map_is_global(nodemap, comp_of, ci, polymap):
                lm = construct_local_node_map(nodemap, rows + 1, polymap)
            columns.append((rows, rows[inf], src, s[src], lm))
    out = AdvancedOutput(np.zeros(n), np.zeros(nodemap.shape), np.zeros(nodemap.shape), num_solves=solved)
    out.stats = dict(setup_s=0.0, solve_s=0.0, columns=len(columns))
    if not columns and factor is not None:
        factor.close()
    if columns:
        if factor is None:
            t0 = time.perf_counter()
            factor = _raster_factor(cellmap, polymap, nodemap, solver, four_neighbors, avg_res)
        with factor:
            if f is not None and f[0] != NODATA:
                factor.set_grounds(finite=f)
            t1 = time.perf_counter()
            factor.reset_currents()
            # columns whose local node map is the node map accumulate on the device; the others bring their
            # currents back to be scattered by their own map
            for own_map in (False, True):
                cols = [c for c in columns if (c[4] is not None) == own_map]
                for sl in _panels(len(cols), solver):
                    chunk = cols[sl]
                    sets, gset = [], []
                    for c in chunk:                                   # -1: finite grounds only
                        gset.append(len(sets) if len(c[1]) else -1)
                        if len(c[1]):
                            sets.append(c[1])
                    res = factor.solve_advanced(sets, gset, [(c[2], c[3]) for c in chunk], want_volt=True,
                                                want_curr=own_map, accumulate=not own_map)
                    out.iterations += int(res["iters"].sum())
                    for j, (rows, _, _, _, lm) in enumerate(chunk):
                        v = np.asarray(res["volt"][rows, j], dtype=np.float64)
                        out.voltages[rows] = v
                        if lm is not None:
                            out.voltmap += _scatter(v, lm)
                            out.curmap += _scatter(np.asarray(res["curr"][rows, j], dtype=np.float64), lm)
            cum, _ = factor.read_currents(want_max=False)
            t2 = time.perf_counter()
        out.stats.update(setup_s=t1 - t0, solve_s=t2 - t1)
        glob = np.zeros(n, dtype=bool)
        for rows, _, _, _, lm in columns:
            glob[rows] = lm is None
        vg = np.where(glob, out.voltages, 0.0)
        out.voltmap += _scatter(vg, nodemap)
        out.curmap += _scatter(np.where(glob, np.asarray(cum, dtype=np.float64), 0.0), nodemap)
    out.result = out.voltmap.copy() if solved else np.array([[-1.0]])
    return out

"""The V-cycle, residual-gate and node-current kernels against float64 references (tests/reference_ops.py).

A wrong preconditioner does not give a wrong answer -- CG corrects it and only spends iterations -- so
the cycle is checked on its own through one application (B200Factor.apply_precond) against the cycle
rebuilt in float64 from the handle's own downloaded levels.  The residual gate is checked against the
true residual of the X it returns, away from convergence, and the node-current kernels against the
currents of the voltages they return.  Every case first asserts that it runs the kernel path it is
named after.  Needs an H100: `pytest -m gpu`."""
import numpy as np
import pytest
import scipy.sparse as sp

import circuitscape_b200 as cb
from circuitscape_b200 import _lib, graph

from .reference_ops import node_currents, stencil_wraps, true_relres, vcycle

pytestmark = pytest.mark.gpu

U32 = np.finfo(np.float32).eps / 2          # unit roundoff
NNZ_CAP = 2304                             # kernels.cuh: entries staged per row block


# ---- operators ---------------------------------------------------------------------------------
def laplacian_of(g, four=False):
    nm = graph.construct_node_map(g)
    G = graph.laplacian(graph.construct_graph(g, nm, False, four))
    big = max(graph.connected_components(G), key=len) - 1
    return G[big][:, big].tocsr()


def conductance(nr, nc, seed, sigma=0.0):
    rng = np.random.default_rng(seed)
    if sigma:
        return np.exp(rng.normal(0.0, sigma, (nr, nc)))
    return 1.0 / rng.uniform(1.0, 10.0, (nr, nc))


def nodata_prefix():
    """Four-neighbour raster whose first cells in memory order are NODATA: every vertical edge that
    crosses a column boundary lands on the +-1 diagonal (a wrapped neighbour)."""
    g = conductance(301, 97, 2)
    g[0:5, 0] = 0.0
    return laplacian_of(g, four=True)


def ragged(four=False):
    g = conductance(301, 97, 3)
    g[120:, 96] = 0.0                      # last raster column ends early: a legitimate stencil form
    return laplacian_of(g, four)


def holey(seed=4, sigma=1.0):
    rng = np.random.default_rng(seed)
    g = conductance(160, 140, seed, sigma)      # > 20 000 nodes: P and R get window records too
    g[rng.random(g.shape) < 0.05] = 0.0
    return laplacian_of(g)


def hub_network():
    """Preferential-attachment graph (>= 20 entries per row: 4 lanes per row in k_spmm) plus one hub
    row longer than a row block can stage."""
    L = graph.power_law_laplacian(12000, m=10, seed=5)
    rng = np.random.default_rng(5)
    W = sp.diags(L.diagonal()) - L
    nb = rng.choice(np.arange(1, L.shape[0]), 3000, replace=False)
    H = sp.coo_matrix((rng.uniform(0.1, 1.0, nb.size), (np.zeros(nb.size, dtype=np.int64), nb)), shape=L.shape)
    return graph.laplacian((W + H + H.T).tocsr())


def full(nr, nc, four=False, seed=1, sigma=0.0):
    return laplacian_of(conductance(nr, nc, seed, sigma), four)


# name -> (operator, solver options, claimed path); built once per module
OPERATORS = {
    "full8_301x97": (lambda: full(301, 97), dict(stencil="on"), "stencil01"),
    "full8_20x37": (lambda: full(20, 37), dict(stencil="on"), "stencil"),
    "full8_65x43": (lambda: full(65, 43), dict(stencil="on"), "stencil"),
    "full8_257x29": (lambda: full(257, 29), dict(stencil="on"), "stencil"),
    "full4_65x43": (lambda: full(65, 43, four=True), dict(stencil="on"), "stencil"),
    "ragged8": (lambda: ragged(), dict(stencil="on"), "stencil"),
    "nodata_prefix4": (nodata_prefix, dict(stencil="on"), "no_stencil"),
    "holey_windowed": (holey, dict(window="on"), "windowed"),
    "holey_plain": (holey, dict(window="off"), "plain"),
    "hub_lpr4": (hub_network, dict(window="off"), "wide"),
}
_CACHE = {}


def operator(name):
    if name not in _CACHE:
        _CACHE[name] = OPERATORS[name][0]()
    return _CACHE[name]


def assert_path(f, A, claim):
    """The case runs the kernels it is named after (a threshold change must not turn it into a
    silent duplicate of another case)."""
    lv = f.levels()
    assert len(lv) >= 2, "no multigrid hierarchy"
    l0 = lv[0]
    if claim == "stencil01":
        assert l0["A_stencil"] and lv[1]["A_stencil"], "level 0 and level 1 must have the stencil form"
    elif claim == "stencil":
        assert l0["A_stencil"]
        nr, off, wrapped = stencil_wraps(A)
        assert off == 0 and wrapped == 0
    elif claim == "no_stencil":
        nr, off, wrapped = stencil_wraps(A)
        assert off == 0 and wrapped > 0, "the case must have wrapped neighbours"
        assert not any(l["A_stencil"] for l in lv), "an operator with wrapped neighbours has no stencil form"
    elif claim == "windowed":
        assert l0["A_windowed"] and not l0["A_stencil"] and l0["P_windowed"] and l0["R_windowed"]
    elif claim in ("plain", "wide"):
        assert not l0["A_windowed"] and not l0["P_windowed"]
    if claim == "wide":
        rl = np.diff(A.indptr)
        assert A.nnz / A.shape[0] >= 20 and rl.max() > NNZ_CAP
    return lv


CONFIGS = {                     # name -> solver options
    "f64": dict(mixed=False),
    "mixed": dict(mixed=True),
    "f32": dict(precision="single", f32_compute=True),
}


def make_solver(config, **kw):
    return cb.CUDASolver(**CONFIGS[config], **kw)


def coarse_pinv_f64(A, config, opts):
    """The dense coarse solve of the device is built from the fp64 coarsest operator even when the
    cycle runs in fp32; take that operator from a fp64 handle of the same values."""
    from .reference_ops import coarse_pinv
    A = A.astype(np.float32).astype(np.float64) if config == "f32" else A
    with cb.B200Factor(A, cb.CUDASolver(mixed=False, **opts)) as f64:
        C = f64.levels()[-1]["A"]
    return C, (coarse_pinv(C) if C.shape[0] <= 320 else None)


# ---- (a) the V-cycle ---------------------------------------------------------------------------
@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("name", list(OPERATORS))
def test_vcycle_matches_float64_reference(name, config, record_property):
    """z = M^-1 r from one application of the device cycle (every level kernel: SP_RES0 / SP_RES,
    restriction, dense coarse solve, fused or separate prolongation + post-smoothing, SP_JACOBI_DOT)
    against the same cycle in float64 on the downloaded levels; r.z; symmetry; determinism."""
    A = operator(name)
    _, opts, claim = OPERATORS[name]
    n = A.shape[0]
    rng = np.random.default_rng(11)
    with cb.B200Factor(A, make_solver(config, **opts)) as f:
        lv = assert_path(f, A, claim)
        C, pinv = coarse_pinv_f64(A, config, opts)
        assert C.shape == lv[-1]["A"].shape and C.nnz == lv[-1]["A"].nnz
        if config == "f64":
            tol = 1e-10
        else:
            # fp32 unit roundoff x (levels) x (9-term stencil sums): 2e-5 leaves room for the growth
            # of the coarse correction; rows of m > 9 entries scale it by sqrt(m / 9)
            tol = 2e-5 * max(1.0, np.sqrt(np.diff(A.indptr).max() / 9.0))
        worst = 0.0
        for k in (1, 2, 4, 8):
            R = rng.standard_normal((n, k))
            if config != "f64":
                R = R.astype(np.float32).astype(np.float64)    # the cycle sees r in fp32
            Z, rz = f.apply_precond(R)
            Zref = vcycle(lv, R, pinv)
            err = np.abs(Z - Zref).max() / np.abs(Zref).max()
            worst = max(worst, err)
            assert err <= tol, (k, err)
            rzref = np.einsum("ij,ij->j", R, Zref)
            assert np.all(np.abs(rz - np.abs(rzref)) <= tol * np.abs(rzref)), (k, rz, rzref)
            Z2, rz2 = f.apply_precond(R)
            assert np.array_equal(Z, Z2) and np.array_equal(rz, rz2), "two applications differ"
        record_property("max_rel_err", worst)
        if config == "f64":
            u = rng.standard_normal((n, 4))
            v = u + rng.standard_normal((n, 4))
            Mu, _ = f.apply_precond(u)
            Mv, _ = f.apply_precond(v)
            a, b = np.einsum("ij,ij->j", u, Mv), np.einsum("ij,ij->j", v, Mu)
            asym = np.abs(a - b) / np.abs(a)
            record_property("max_asymmetry", float(asym.max()))
            assert asym.max() <= 1e-12, asym


def test_apply_precond_needs_a_hierarchy():
    A = full(20, 37)
    with cb.B200Factor(A, cb.CUDASolver(precond="jacobi")) as f:
        with pytest.raises(cb.B200Error) as e:
            f.apply_precond(np.ones(A.shape[0]))
        assert e.value.code == _lib.ERR_UNSUPPORTED


# ---- (b) the residual gate ---------------------------------------------------------------------
GATE_OPERATORS = ["full8_301x97", "holey_windowed", "holey_plain"]


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("grounded", [False, True])
@pytest.mark.parametrize("name", GATE_OPERATORS)
def test_residual_gate_reports_the_true_residual(name, grounded, config, record_property):
    """relres of solve_rhs stopped early (itmax = 2: relres far above roundoff) is ||B - A X|| / ||B||
    of the X it returns, for every column of panels of width 8, 4, 2, 1 (21 columns: 8 + 8 + 4 + 1);
    a column at or above 1e-4 is reported as failing."""
    A = operator(name)
    _, opts, claim = OPERATORS[name]
    n = A.shape[0]
    rng = np.random.default_rng(3)
    if grounded:
        d = np.zeros(n)
        d[rng.choice(n, 5, replace=False)] = rng.uniform(0.5, 2.0, 5)
        A = (A + sp.diags(d)).tocsr()
    with cb.B200Factor(A, make_solver(config, **opts)) as f:
        assert_path(f, A, claim if claim != "stencil01" else "stencil")
        Ad = A.astype(f.dtype).astype(np.float64)
        m = np.diff(A.indptr).max()
        for k in (1, 2, 4, 8, 21):
            B = rng.standard_normal((n, k))
            if not grounded:
                B -= B.mean(axis=0)                     # b orthogonal to the null space
            B = B.astype(f.dtype)
            X, iters, relres = f.solve_rhs(B, itmax=2, raise_on_residual=False)
            ref = true_relres(Ad, X, B)
            assert ref.min() > 1e-6, ref                # not at roundoff: the comparison is sharp
            if f.dtype == np.float64:
                bound = 1e-10 * ref
            else:
                # fp32 residual of an m-entry row: |dr_i| <= (m + 1) u (|b_i| + sum_j |a_ij x_j|)
                Bd, Xd = B.astype(np.float64), X.astype(np.float64)
                bound = (m + 1) * U32 * np.linalg.norm(np.abs(Bd) + abs(Ad) @ np.abs(Xd), axis=0) / np.linalg.norm(Bd, axis=0)
            dev = np.abs(relres - ref)
            record_property(f"k{k}_max_dev_over_bound", float((dev / bound).max()))
            assert np.all(dev <= bound), (k, relres, ref, bound)
            assert np.array_equal(relres >= 1e-4, ref >= 1e-4)
            if np.any(ref >= 1e-4):
                with pytest.raises(cb.SolverResidualError):
                    f.solve_rhs(B, itmax=2)
        if f.dtype == np.float64:                       # converged: the gate passes every column
            X, _, relres = f.solve_rhs(B)
            assert relres.max() < 1e-4 and true_relres(Ad, X, B).max() < 1e-4


# ---- (c) node currents -------------------------------------------------------------------------
def corridor():
    """Lognormal raster (sigma = 3) with a one-cell-wide dead-end corridor inside a NODATA block:
    branch currents over many decades, many near the 1e-8 cut, and corridor nodes that carry exactly
    zero current."""
    g = conductance(120, 110, 6, sigma=3.0)
    g[50:71, 0:41] = 0.0
    g[60, 0:41] = 1.0
    return laplacian_of(g)


def pockets():
    """Full lognormal raster (sigma = 3: a stencil form) with two corner pockets behind two-cell walls
    of conductance 1e-7 and 1e-5: the pockets' branch currents sit decades below the rest, around the
    1e-8 cut, where cutting inflow and outflow against the wrong maximum changes the result."""
    g = conductance(130, 111, 8, sigma=3.0)
    g[30:32, 0:32] = 1e-7
    g[0:32, 30:32] = 1e-7
    g[98:100, 79:] = 1e-5
    g[98:, 79:81] = 1e-5
    return laplacian_of(g)


CURRENT_OPERATORS = {
    "corridor_csr": (corridor, dict(window="off"), "plain"),
    "pockets_stencil": (pockets, dict(stencil="on"), "stencil"),
}
_CUR_CACHE = {}


@pytest.mark.parametrize("log_transform", [False, True])
@pytest.mark.parametrize("pw", [1, 2, 4, 8])
@pytest.mark.parametrize("config", ["mixed", "f32"])
@pytest.mark.parametrize("name", list(CURRENT_OPERATORS))
def test_node_currents_match_float64_reference(name, config, pw, log_transform, record_property):
    """Per-pair currents, the weighted cumulative map and the max map (k_cur_max[_dia] +
    k_cur_acc[_dia]) against the currents of the voltages solve_pairs returns, so that solver error
    drops out; with and without the log10 accumulation (src/out.jl:305-309, -9999 for zero)."""
    make, opts, claim = CURRENT_OPERATORS[name]
    if name not in _CUR_CACHE:
        _CUR_CACHE[name] = make()
    A = _CUR_CACHE[name]
    n = A.shape[0]
    rng = np.random.default_rng(pw)
    k = 11
    nodes = rng.choice(n, 2 * k, replace=False)
    src, dst = nodes[:k], nodes[k:]                     # both orientations of the node order occur
    weight = rng.integers(1, 4, k).astype(np.float64)
    # fp64: solved far below the default rtol so that the dead-end corridor's branch currents (zero in
    # exact arithmetic) fall under the 1e-8 cut and its nodes carry exactly zero current
    rtol = 1e-12 if config == "mixed" else None
    with cb.B200Factor(A, make_solver(config, panel_width=pw, **opts), log_transform=log_transform) as f:
        assert f.operator_form() == {"plain": "csr", "windowed": "windowed", "stencil": "stencil"}[claim]
        assert_path(f, A, claim)
        out = f.solve_pairs(src, dst, weight, want_volt=True, want_curr=True, accumulate=True, rtol=rtol,
                            raise_on_residual=False)
        cum, mx = f.read_currents()
        eps = np.finfo(f.dtype).eps
        Ad = A.astype(f.dtype).astype(np.float64)
        arow = np.asarray(abs(Ad).sum(axis=1)).ravel() - np.abs(Ad.diagonal())     # sum_j |a_ij|, j != i
        rel = 1e-12 if f.dtype == np.float64 else 10 * U32       # 8-term sums in the kernel's type
        refs, bounds, masked = [], [], np.zeros(n, dtype=bool)
        zeros = 0
        for c in range(k):
            v = out["volt"][:, c].astype(np.float64)
            # the kernel differences the unshifted solution, the returned voltages are shifted by
            # v[src]: v_i - v_j agree to 4 eps max|v|, which widens the margin and the bound
            dv = 4 * eps * np.abs(v).max()
            ref, mask = node_currents(Ad, v, dv=dv)
            b = rel * ref + arow * dv
            cur = out["curr"][:, c].astype(np.float64)
            dev = np.abs(cur - ref)[~mask]
            record_property(f"col{c}_masked", int(mask.sum()))
            assert np.all(dev <= b[~mask]), (c, dev.max(), np.nonzero(dev > b[~mask])[0][:5])
            zeros += int(((ref == 0) & ~mask).sum())
            refs.append(ref); bounds.append(b); masked |= mask
        refs, bounds = np.array(refs), np.array(bounds)
        record_property("zero_current_nodes", zeros)
        if name.startswith("corridor") and config == "mixed":
            assert zeros > 0, "the dead-end corridor must carry exactly zero current"
        keep = ~masked
        if log_transform:
            with np.errstate(divide="ignore"):
                vals = np.where(refs > 0, np.log10(np.where(refs > 0, refs, 1.0)), -9999.0)
                vb = np.where(refs > 0, bounds / (np.where(refs > 0, refs, 1.0) * np.log(10.0)), 0.0)
            vb = vb + eps * np.maximum(1.0, np.abs(vals))           # log10 rounded to the kernel's type
        else:
            vals, vb = refs, bounds
        cref = (weight[:, None] * vals).sum(axis=0)
        # + one rounding of the stored map per panel
        cb_ = (weight[:, None] * vb).sum(axis=0) + (k + 1) * eps * (weight[:, None] * np.abs(vals)).sum(axis=0)
        mref = np.maximum(vals.max(axis=0), -9999.0)
        assert np.all(np.abs(cum.astype(np.float64) - cref)[keep] <= cb_[keep])
        assert np.all(np.abs(mx.astype(np.float64) - mref)[keep] <= vb.max(axis=0)[keep] + eps * np.abs(mref[keep]))
        record_property("masked_nodes", int(masked.sum()))


# ---- (d) the stencil form is taken exactly when it is sound --------------------------------------
def test_nodata_prefix_raster_has_no_stencil_form():
    """A NODATA prefix wraps neighbours into the next raster column: the operator keeps the CSR path
    under stencil = on, and its SpMM is still exact."""
    A = nodata_prefix()
    nr, off, wrapped = stencil_wraps(A)
    assert nr == 301 and off == 0 and wrapped > 0
    rng = np.random.default_rng(1)
    with cb.B200Factor(A, cb.CUDASolver(stencil="on", precond="jacobi")) as f:
        assert f.operator_form() != "stencil"
        X = rng.standard_normal((A.shape[0], 4))
        assert np.abs(f.spmm(X) - A @ X).max() <= 1e-13 * np.abs(A).sum(axis=1).max() * np.abs(X).max()

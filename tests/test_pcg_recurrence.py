"""The PCG recurrence that joins the kernels -- alpha in the SP_CG epilogues, k_cg_update_r0 /
k_cg_update_xp2 (AMG) and k_cg_init / k_cg_update_r / k_cg_update_xp (Jacobi), cg_after_precond's
beta, stop test, stall guard and per-column freezing, k_loop_cond and the three loop drivers --
against the float64 recurrence of tests/reference_ops.py `pcg`.

CG hides mistakes here: a wrong beta, an alpha left on for a frozen column or a V-cycle started from
the wrong x0 costs iterations, not accuracy, so the final answers and the 1e-4 gate do not see it.
These tests compare the iterates after m steps, the stop iteration of every column, frozen columns
and the drivers with the reference recurrence run on the handle's own downloaded hierarchy.

CPU: the reference itself (three eigenvalues, batched = column by column, itmax, the host hierarchy
harness).  GPU (`pytest -m gpu`): everything else."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp

from .reference_ops import ATOL, _vcycle, pcg, vcycle

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
U32 = np.finfo(np.float32).eps / 2          # unit roundoff of fp32
F32 = np.float32


# ---- CPU: the reference --------------------------------------------------------------------------
def _small_laplacian(nr=30, nc=25, seed=0, ground=True):
    from circuitscape_b200 import graph
    A, _ = graph.synthetic_raster_laplacian(nr, nc, seed=seed)
    A = sp.csr_matrix(A, dtype=np.float64)
    if ground:
        d = np.zeros(A.shape[0])
        d[[3, A.shape[0] // 2]] = [0.7, 1.3]
        A = (A + sp.diags(d)).tocsr()
    return A


def _textbook_pcg(A, b, M, m):
    """m steps of textbook PCG (x updated before r), no stop test."""
    x = np.zeros_like(b); r = b.copy(); z = M(r); p = z.copy(); g = r @ z
    for _ in range(m):
        Ap = A @ p; a = g / (p @ Ap); x += a * p; r -= a * Ap
        z = M(r); gn = r @ z; p = z + (gn / g) * p; g = gn
    return x


def test_three_eigenvalues_take_three_iterations():
    """In exact arithmetic CG ends after as many iterations as A has distinct eigenvalues."""
    rng = np.random.default_rng(0)
    d = np.repeat([1.0, 3.0, 10.0], 20)
    A = sp.diags(d).tocsr()
    B = rng.standard_normal((d.size, 4))
    X, iters, rho, tol = pcg(A, B, lambda R: R, rtol=1e-10, itmax=50)
    assert np.array_equal(iters, [3, 3, 3, 3])
    assert rho.shape == (4, 4) and np.all(np.sqrt(rho[2]) > tol) and np.all(np.sqrt(rho[3]) <= tol)
    assert np.abs(X - B / d[:, None]).max() <= 1e-12 * np.abs(B / d[:, None]).max()


def test_batched_equals_column_by_column():
    """A column's recurrence does not see the other columns of its panel: the batched solve equals the
    one-column solves bit for bit (zero, tiny and ordinary columns, different stop iterations)."""
    A = _small_laplacian()
    n = A.shape[0]
    dinv = 1.0 / A.diagonal()
    M = lambda R: R * dinv[:, None]
    rng = np.random.default_rng(1)
    B = rng.standard_normal((n, 6))
    B[:, 1] = 0.0
    B[:, 3] *= 1e-12                                   # inactive from the start: atol decides
    B[:, 4] = A @ np.linspace(0.0, 1.0, n)             # stops early
    X, iters, rho, tol = pcg(A, B, M, rtol=1e-8, itmax=400, stall_limit=2000)
    assert iters[1] == 0 and iters[3] == 0 and len(set(iters[[0, 2, 4, 5]])) > 1
    for c in range(B.shape[1]):
        x, it, r, t = pcg(A, B[:, c], M, rtol=1e-8, itmax=400, stall_limit=2000)
        assert np.array_equal(x[:, 0], X[:, c]) and it[0] == iters[c] and t[0] == tol[c]
        assert np.array_equal(r[:, 0], rho[:r.shape[0], c], equal_nan=True)
        assert np.all(np.isnan(rho[r.shape[0]:, c]))


def test_itmax_returns_the_mth_iterate():
    """itmax = m stops every active column at iteration m with the m-th iterate (the deferred
    x += alpha p still runs on the stopping iteration); a zero column and itmax = 0 return X = 0."""
    A = _small_laplacian(seed=2)
    n = A.shape[0]
    dinv = 1.0 / A.diagonal()
    rng = np.random.default_rng(2)
    B = rng.standard_normal((n, 3))
    B[:, 2] = 0.0
    for m in (1, 2, 3, 5, 8):
        X, iters, rho, _ = pcg(A, B, lambda R: R * dinv[:, None], rtol=1e-14, itmax=m)
        assert np.array_equal(iters, [m, m, 0]) and rho.shape[0] == m + 1
        for c in (0, 1):
            x = _textbook_pcg(A, B[:, c], lambda r: r * dinv, m)
            assert np.abs(X[:, c] - x).max() <= 1e-12 * np.abs(x).max(), (m, c)
        assert not X[:, 2].any()
    X, iters, _, _ = pcg(A, B, lambda R: R * dinv[:, None], rtol=1e-6, itmax=0)
    assert not X.any() and not iters.any()


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("amgh") / "libamgh.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so,
                           os.path.join(HERE, "amg_host_harness.cpp")])
    lib = C.CDLL(so)
    lib.amgh_build.restype = C.c_void_p
    lib.amgh_build.argtypes = [C.c_long, C.c_long, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.amgh_nlevels.argtypes = [C.c_void_p]
    lib.amgh_dims.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 4
    lib.amgh_copy.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.amgh_pinv.argtypes = [C.c_void_p, C.c_void_p]
    lib.amgh_free.argtypes = [C.c_void_p]
    return lib


@pytest.mark.parametrize("grounded", [False, True])
def test_matches_host_hierarchy_pcg(harness, grounded):
    """With the V-cycle of the host hierarchy, `pcg` takes the iterations of the plain PCG of
    tests/test_amg_host.py and returns the same X."""
    from .test_amg_host import build, pcg as host_pcg
    A = _small_laplacian(120, 90, seed=3, ground=grounded)
    n = A.shape[0]
    levels, pinv = build(harness, A)
    assert len(levels) >= 3
    M = lambda r: vcycle(levels, r, pinv)
    b = np.zeros(n); b[3] = -1.0; b[n - 5] = 1.0
    for rtol in (1e-6, 1e-10):
        x, it = host_pcg(A, b, M, rtol=rtol, itmax=500)
        X, iters, _, _ = pcg(A, b, M, rtol=rtol, itmax=500)
        assert iters[0] == it > 3
        assert np.abs(X[:, 0] - x).max() <= 1e-12 * np.abs(x).max()


# ---- GPU: shared set-up --------------------------------------------------------------------------
def _kp():
    from . import test_kernel_parity as kp
    return kp


CASES = {   # name -> (kernel-parity operator, grounded, claimed path)
    "full8_301x97": ("full8_301x97", False, "stencil01"),
    "ragged8": ("ragged8", False, "stencil"),
    "holey_windowed": ("holey_windowed", False, "windowed"),
    "holey_plain": ("holey_plain", False, "plain"),
    "hub_lpr4": ("hub_lpr4", False, "wide"),
    "grounded_windowed": ("holey_windowed", True, "windowed"),
    "full8_20x37": ("full8_20x37", False, "stencil"),
}
FORM = {"stencil01": "stencil", "stencil": "stencil", "windowed": "windowed", "plain": "csr", "wide": "csr"}
_OPS = {}


def case_operator(name):
    if name not in _OPS:
        base, grounded, _ = CASES[name]
        A = _kp().operator(base)
        if grounded:                                   # advanced-mode shape: SPD, grounds on 5 nodes
            rng = np.random.default_rng(3)
            d = np.zeros(A.shape[0])
            d[rng.choice(A.shape[0], 5, replace=False)] = rng.uniform(0.5, 2.0, 5)
            A = (A + sp.diags(d)).tocsr()
        _OPS[name] = A
    return _OPS[name]


def rhs(name, k, seed):
    """k columns of standard normals; orthogonal to the constants unless the operator is grounded."""
    n = case_operator(name).shape[0]
    B = np.random.default_rng(seed).standard_normal((n, k))
    if not CASES[name][1]:
        B -= B.mean(axis=0)
    return B


def make_factor(name, config, precond="amg", **kw):
    import circuitscape_b200 as cb
    kp = _kp()
    A = case_operator(name)
    base, _, claim = CASES[name]
    opts = kp.OPERATORS[base][1]
    f = cb.B200Factor(A, kp.make_solver(config, precond=precond, **opts, **kw))
    assert f.operator_form() == FORM[claim], (name, f.operator_form())
    if precond == "amg":
        kp.assert_path(f, A, claim)
    return f


class Reference:
    """The float64 recurrence on the handle's own operator and hierarchy, and for the fp32
    configurations a second one with fp32 storage and an fp32 cycle, whose distance from the first
    sizes the bound (never the device's output).

      f64    A, cycle and vectors in fp64
      mixed  fp64 A and vectors; r rounded to fp32 before the fp64 cycle on the fp32 levels
      f32    fp32 A and levels widened to fp64, r rounded to fp32 before the cycle
    The perturbed recurrence (mixed, f32) runs the cycle in fp32 arithmetic and, for f32, stores
    x, r, p, z and A p in fp32, as the device does."""

    def __init__(self, f, name, config, precond):
        kp = _kp()
        A = case_operator(name)
        self.config, self.precond = config, precond
        self.stall = 40 if precond == "amg" else 2000
        self.A = A.astype(f.dtype).astype(np.float64) if f.dtype == np.float32 else A
        self.A32 = A.astype(F32)
        if precond == "jacobi":
            dinv = 1.0 / self.A.diagonal()
            dinv32 = (1.0 / self.A32.diagonal()).astype(F32)
            self.M = lambda R: R * dinv[:, None]
            self.M32 = lambda R: np.asarray(R, dtype=F32) * dinv32[:, None]
        else:
            lv = f.levels()
            _, pinv = kp.coarse_pinv_f64(case_operator(name), config, kp.OPERATORS[CASES[name][0]][1])
            if config == "f64":
                self.M = lambda R: vcycle(lv, R, pinv)
            else:
                self.M = lambda R: vcycle(lv, np.asarray(R, dtype=F32), pinv)
            lv32 = [dict(A=L["A"].astype(F32), P=None if L["P"] is None else L["P"].astype(F32),
                         R=None if L["R"] is None else L["R"].astype(F32), omega=L["omega"]) for L in lv]
            p32 = None if pinv is None else pinv.astype(F32)
            self.M32 = lambda R: _vcycle(lv32, p32, np.asarray(R, dtype=F32), 0)

    def run(self, B, rtol, itmax):
        B = np.asarray(B, dtype=np.float64)
        return pcg(self.A, B, self.M, rtol, itmax, stall_limit=self.stall)

    def bound(self, B, rtol, itmax, X):
        """Per-column bound on |X_device - X| for the reference iterate X."""
        scale = np.abs(X).max(axis=0)
        if self.config == "f64":
            return 1e-10 * scale                       # the cycle alone is checked at 1e-10
        if self.config == "f32":
            Xp = pcg(self.A32, np.asarray(B, dtype=F32), self.M32, rtol, itmax, stall_limit=self.stall,
                     dtype=F32)[0]
        else:
            Xp = pcg(self.A, B, self.M32, rtol, itmax, stall_limit=self.stall)[0]
        spread = np.abs(Xp.astype(np.float64) - X).max(axis=0)
        # two fp32 evaluations of the recurrence differ by the same order as each from fp64: 8x the
        # spread, plus a floor of 64 fp32 roundings of the column's largest entry
        return 8.0 * spread + 64 * U32 * scale


def device_solve(f, B, **kw):
    X, iters, relres = f.solve_rhs(np.asarray(B, dtype=f.dtype), raise_on_residual=False, **kw)
    return np.asarray(X, dtype=np.float64).reshape(B.shape[0], -1), iters, relres


def near_tie(rho, tol, iters, delta):
    """Columns whose sqrt(rho)/tol lies within delta of 1 at the reference's stop iteration or the one
    before it: there two correct implementations may stop one iteration apart."""
    out = np.zeros(len(iters), dtype=bool)
    for c, s in enumerate(iters):
        for j in (s - 1, s):
            if 0 <= j < rho.shape[0] and np.isfinite(rho[j, c]):
                out[c] |= abs(np.sqrt(rho[j, c]) / tol[c] - 1.0) <= delta
    return out


DELTA = {"f64": 1e-8, "mixed": 1e-3, "f32": 1e-2}
K_ALL = 23                         # panels of 8 + 8 + 4 + 2 + 1: every width, a ragged split


# ---- (a) iterates after m steps ------------------------------------------------------------------
def check_iterates(name, config, precond="amg"):
    """solve_rhs stopped at itmax = m against the reference's m-th iterate, m in 1, 2, 3, 5, 8, for
    23 columns (every panel width); returns the largest measured / bound."""
    B = rhs(name, K_ALL, seed=7)
    worst = 0.0
    with make_factor(name, config, precond) as f:
        ref = Reference(f, name, config, precond)
        Bd = B.astype(f.dtype).astype(np.float64)
        for m in (1, 2, 3, 5, 8):
            X, iters, _ = device_solve(f, Bd, rtol=1e-10, itmax=m)
            Xr, it_r, _, _ = ref.run(Bd, 1e-10, m)
            assert np.array_equal(it_r, np.full(K_ALL, m)), (m, it_r)
            assert np.array_equal(iters, it_r), (m, iters)
            bound = ref.bound(Bd, 1e-10, m, Xr)
            err = np.abs(X - Xr).max(axis=0)
            worst = max(worst, float((err / bound).max()))
            bad = np.nonzero(err > bound)[0]
            assert not bad.size, (m, bad, err[bad], bound[bad])
    return worst


ITERATE_CASES = ([(name, config, "amg") for name in ("full8_301x97", "ragged8", "holey_windowed", "holey_plain",
                                                     "hub_lpr4", "grounded_windowed")
                  for config in ("f64", "mixed", "f32")] +
                 [(name, config, "jacobi") for name in ("full8_301x97", "holey_windowed") for config in ("f64", "f32")])


@pytest.mark.gpu
@pytest.mark.parametrize("name,config,precond", ITERATE_CASES, ids=lambda v: str(v))
def test_iterates_after_m_steps(name, config, precond, record_property):
    record_property("max_err_over_bound", check_iterates(name, config, precond))


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["f64", "mixed"])
def test_iterates_with_stored_x0_on_a_stencil_level(config):
    """The same check on the stencil-form operator with the pre-smoothed x0 stored
    (CS_B200_NO_IMPLICIT_X0): k_cg_update_r0 writes x0 and the stencil kernels read it.  The switch
    is read once per process, hence the child."""
    env = dict(os.environ, CS_B200_NO_IMPLICIT_X0="1")
    code = ("from tests.test_pcg_recurrence import check_iterates; "
            f"print('max_err_over_bound', check_iterates('full8_301x97', {config!r}))")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]


# ---- (b) stop iterations -------------------------------------------------------------------------
# f32 runs at rtol 1e-6 on the grounded operator and the Jacobi case only.  At 1e-10 the fp32
# recurrence stagnates and the stall guard picks the stop.  On a Laplacian without grounds, rounding A
# to fp32 leaves a near-null mode that B is not orthogonal to, and resolving it takes a number of
# iterations set by rounding (measured on an H100: 9-76 against 10-18 in fp64 arithmetic).
STOP_CASES = ([(name, config, "amg", rtol) for name in ("full8_301x97", "holey_windowed", "hub_lpr4")
               for config in ("f64", "mixed") for rtol in (1e-6, 1e-10)] +
              [("grounded_windowed", config, "amg", rtol) for config in ("f64", "mixed") for rtol in (1e-6, 1e-10)] +
              [("grounded_windowed", "f32", "amg", 1e-6)] +
              [("full8_20x37", "f64", "jacobi", rtol) for rtol in (1e-6, 1e-10)] +
              [("full8_20x37", "f32", "jacobi", 1e-6)])


@pytest.mark.gpu
@pytest.mark.parametrize("name,config,precond,rtol", STOP_CASES, ids=lambda v: str(v))
def test_stop_iterations_match(name, config, precond, rtol, record_property):
    """Solved to convergence, every column stops at the reference's iteration (within one in the fp32
    configurations), except near-ties, which may not exceed a fifth of the columns."""
    B = rhs(name, K_ALL, seed=11)
    with make_factor(name, config, precond) as f:
        ref = Reference(f, name, config, precond)
        Bd = B.astype(f.dtype).astype(np.float64)
        X, iters, relres = device_solve(f, Bd, rtol=rtol, itmax=500)
        Xr, it_r, rho, tol = ref.run(Bd, rtol, 500)
        assert it_r.max() < 500 and it_r.min() > 1
        tie = near_tie(rho, tol, it_r, DELTA[config])
        record_property("near_ties", int(tie.sum()))
        record_property("iterations", [int(v) for v in it_r])
        assert (~tie).sum() >= 0.8 * K_ALL, (tie.sum(), it_r)
        diff = np.abs(iters - it_r)[~tie]
        assert diff.max() <= (0 if config == "f64" else 1), (iters, it_r, tie)


# ---- (c) freezing and column independence --------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("config", ["f64", "mixed", "f32"])
def test_frozen_columns_do_not_move(config, record_property):
    """A target column in panels of widths 8, 4 and 2 at every position, next to a zero column, a
    column that stops after 1-2 iterations, a column the atol term leaves inactive and columns that
    iterate longer: within a width its X, iters and relres are bit-identical across placements and
    companions and match the reference at its own stop iteration; the companions that stop early
    match the reference too (a frozen column does not move).

    The stop iterations are set through the atol term: a column whose sqrt(rho0) is c * atol stops
    once rho has fallen by about c^2 (c = 1e3: the target, about 5 iterations; c = 3: 1-2
    iterations; c = 1e-3: inactive), while the unscaled point-source columns run to rtol."""
    name = "full8_301x97"
    A = case_operator(name)
    n = A.shape[0]
    rng = np.random.default_rng(5)
    noise = rng.standard_normal((n, 3))
    noise -= noise.mean(axis=0)
    slow = []
    for s in range(4):
        b = np.zeros(n); b[rng.choice(n, 2, replace=False)] = [-1.0, 1.0]
        slow.append(b)
    with make_factor(name, config) as f:
        ref = Reference(f, name, config, "amg")
        rtol = 1e-6
        rho0 = np.abs(np.einsum("ij,ij->j", noise, ref.M(noise)))
        noise = noise * (np.array([1e3, 3.0, 1e-3]) * ATOL / np.sqrt(rho0))
        cols = {"target": noise[:, 0], "zero": np.zeros(n), "quick": noise[:, 1], "tiny": noise[:, 2],
                **{f"slow{s}": b for s, b in enumerate(slow)}}
        cols = {k: v.astype(f.dtype).astype(np.float64) for k, v in cols.items()}
        refs = {}
        for k in ("target", "quick", "tiny", "slow0"):
            Xr, it_r, _, _ = ref.run(cols[k], rtol, 500)
            refs[k] = (Xr, it_r[0], ref.bound(cols[k], rtol, 500, Xr))
        assert refs["tiny"][1] == 0 and 1 <= refs["quick"][1] <= 2, refs["quick"][1]
        assert refs["slow0"][1] > refs["target"][1] + 1, (refs["slow0"][1], refs["target"][1])
        layouts = {8: [["zero", "quick", "tiny", "slow0", "slow1", "slow2", "slow3"]],
                   4: [["zero", "quick", "slow0"], ["tiny", "slow1", "slow2"]],
                   2: [["zero"], ["quick"], ["tiny"], ["slow0"]]}
        worst = 0.0
        for w, comps in layouts.items():
            seen = None
            for comp in comps:
                for pos in range(w):
                    names = comp[:pos] + ["target"] + comp[pos:]
                    X, iters, relres = device_solve(f, np.stack([cols[k] for k in names], axis=1),
                                                    rtol=rtol, itmax=500)
                    got = (X[:, pos].tobytes(), iters[pos], relres[pos])
                    if seen is None:
                        seen = got
                        Xr, it_r, bound = refs["target"]
                        assert iters[pos] == it_r, (w, iters[pos], it_r)
                        err = np.abs(X[:, pos] - Xr[:, 0]).max()
                        worst = max(worst, err / bound[0])
                        assert err <= bound[0], (w, err, bound[0])
                    assert got == seen, (w, names)
                    for c, k in enumerate(names):
                        if k == "zero":
                            assert not X[:, c].any() and iters[c] == 0 and relres[c] == 0.0
                        elif k in ("quick", "tiny"):
                            Xr, it_r, bound = refs[k]
                            assert iters[c] == it_r, (w, names, k, iters[c], it_r)
                            assert np.abs(X[:, c] - Xr[:, 0]).max() <= bound[0], (w, names, k)
        record_property("max_err_over_bound", float(worst))


# ---- (d) loop drivers ----------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("precond", ["amg", "jacobi"])
def test_loop_drivers_agree(precond):
    """The device WHILE graph, host-polled graph chunks and plain launches, each with check_every 1,
    3 and 16 (AMG chunks of 1, 3 and 4 iterations), stopped by itmax before, at and after chunk
    boundaries and by convergence: bit-identical X, iters and relres, the reference's iterates and
    stop iterations, and the same result from a second call on the cached graph.  itmax = 0 returns
    X = 0, iters = 0, relres = 1 and fails the residual gate."""
    import circuitscape_b200 as cb
    name, config, k, rtol = "full8_20x37", "f64", 11, 1e-6
    B = rhs(name, k, seed=13)
    results = {}
    refs = {}
    for use_graph in (True, "chunk", False):
        for check_every in (1, 3, 16):
            with make_factor(name, config, precond, use_graph=use_graph, check_every=check_every) as f:
                if not refs:
                    ref = Reference(f, name, config, precond)
                    for itmax in (1, 4, 5, 7, 500):
                        Xr, it_r, rho, tol = ref.run(B, rtol, itmax)
                        refs[itmax] = (Xr, it_r, near_tie(rho, tol, it_r, DELTA[config]),
                                       ref.bound(B, rtol, itmax, Xr) if itmax <= 8 else None)
                    assert 5 < refs[500][1].max() < 500
                for itmax in (0, 1, 4, 5, 7, 500):
                    got = device_solve(f, B, rtol=rtol, itmax=itmax)
                    again = device_solve(f, B, rtol=rtol, itmax=itmax)
                    assert all(np.array_equal(a, b) for a, b in zip(got, again)), (use_graph, check_every, itmax)
                    X, iters, relres = got
                    if itmax == 0:
                        assert not X.any() and not iters.any() and np.all(relres == 1.0)
                        with pytest.raises(cb.SolverResidualError):
                            f.solve_rhs(B, rtol=rtol, itmax=0)
                    else:
                        Xr, it_r, tie, bound = refs[itmax]
                        assert np.array_equal(iters[~tie], it_r[~tie]), (use_graph, check_every, itmax, iters, it_r)
                        if itmax <= 8:      # the bound of the iterates after m steps; a converged
                            # Jacobi solve (~90 iterations) has amplified its rounding far beyond it
                            assert np.all(np.abs(X - Xr).max(axis=0) <= bound), (use_graph, check_every, itmax)
                    if itmax in results:
                        first = results[itmax]
                        assert all(np.array_equal(a, b) for a, b in zip(got, first)), (use_graph, check_every, itmax)
                    else:
                        results[itmax] = got
    assert (~refs[500][2]).sum() >= 0.8 * k


# ---- (e) power-of-two scaling --------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("config,precond", [("f64", "amg"), ("mixed", "amg"), ("f32", "amg"),
                                            ("f64", "jacobi"), ("f32", "jacobi")])
@pytest.mark.parametrize("name", ["full8_301x97", "holey_windowed"])
def test_power_of_two_scaling_is_exact(name, config, precond):
    """B -> 2^s B (s = -20, 20) scales X exactly and keeps iters and relres: no absolute threshold or
    underflow inside the kernels or the fp32 cycle.  The base B is scaled by 2^30 so that atol stays
    below 1e-3 of the rtol term of every scaled column."""
    rtol, itmax = 1e-6, 60
    B = rhs(name, 11, seed=17) * 2.0 ** 30
    with make_factor(name, config, precond) as f:
        ref = Reference(f, name, config, precond)
        Bd = B.astype(f.dtype).astype(np.float64)
        rho0 = np.abs(np.einsum("ij,ij->j", Bd, ref.M(Bd)))
        assert np.all(ATOL <= 1e-3 * rtol * np.sqrt(rho0) * 2.0 ** -20)
        X, iters, relres = device_solve(f, Bd, rtol=rtol, itmax=itmax)
        assert iters.min() > 1
        for s in (-20, 20):
            Xs, its, rels = device_solve(f, Bd * 2.0 ** s, rtol=rtol, itmax=itmax)
            assert np.array_equal(Xs, X * 2.0 ** s), s
            assert np.array_equal(its, iters) and np.array_equal(rels, relres), s


# ---- (f) the pair driver -------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("config,precond", [("f64", "amg"), ("mixed", "amg"), ("f32", "amg"), ("f64", "jacobi")])
@pytest.mark.parametrize("name", ["full8_301x97", "holey_windowed"])
def test_pair_driver_runs_the_same_recurrence(name, config, precond):
    """solve_pairs(src, dst) is solve_rhs on e_dst - e_src: its voltages are X - X[src] bit for bit,
    the same iterations, and R = X[dst] - X[src]."""
    n = case_operator(name).shape[0]
    rng = np.random.default_rng(19)
    k = 11
    nodes = rng.choice(n, 2 * k, replace=False)
    src, dst = nodes[:k], nodes[k:]
    B = np.zeros((n, k))
    B[src, np.arange(k)] = -1.0
    B[dst, np.arange(k)] = 1.0
    itmax = 500 if precond == "amg" else 60
    with make_factor(name, config, precond) as f:
        X, iters, _ = f.solve_rhs(B.astype(f.dtype), itmax=itmax, raise_on_residual=False)
        out = f.solve_pairs(src, dst, want_volt=True, itmax=itmax, raise_on_residual=False)
        cols = np.arange(k)
        assert np.array_equal(out["iters"], iters)
        assert np.array_equal(out["volt"], X - X[src, cols][None, :])
        assert np.array_equal(out["R"], X[dst, cols] - X[src, cols])

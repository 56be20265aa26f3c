"""The fused CG step of the stencil-form AMG-PCG loop (kernels.cuh k_stencil_cg: p = z + beta p, A p, p.Ap and
the deferred x updates, two at a time, in one kernel) against the unfused CG SpMM + k_cg_update_xp2 pair it
replaces (CS_B200_NO_FUSED_CG).  The fused step forms every value with the pair's expressions and keeps the
SpMM's grid, tile order and reductions, so X, iters, relres, R, voltages and current maps must be
bit-identical: solve_rhs, solve_pairs and region pairs, panels of width 8, 4, 2 and 1, fp64 / mixed / fp32
cycles, itmax 1-6 (the paired update's pending terms of both parities) and converged, under the device WHILE
graph, host-polled graph chunks and plain launches.  A column frozen early keeps its X bit-for-bit while the
others iterate on.  The switch is read once per process, so each setting runs in a child.  Needs an H100."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "full8_301x97"                  # stencil form on levels 0 and 1
DRIVERS = {"graph": dict(use_graph=True), "chunk": dict(use_graph="chunk", check_every=3),
           "plain": dict(use_graph=False, check_every=3)}
ITMAX = (1, 2, 3, 4, 5, 6, 500)
K = 15                                 # panels of 8 + 4 + 2 + 1


def _sets(nr, nc, count, seed):
    """count disjoint 2 x 2 blocks of raster cells (column-major node numbering)."""
    rng = np.random.default_rng(seed)
    out, used = [], set()
    while len(out) < count:
        r, c = int(rng.integers(1, nr - 2)), int(rng.integers(1, nc - 2))
        cells = {(r + i, c + j) for i in range(2) for j in range(2)}
        if cells & used:
            continue
        used |= {(a + i, b + j) for a, b in cells for i in (-1, 0, 1) for j in (-1, 0, 1)}
        out.append(np.array(sorted(b * nr + a for a, b in cells), dtype=np.int64))
    return out


def _collect(config, out_path):
    """Every result of the cases above for one setting of the switch, into an npz."""
    import circuitscape_b200 as cb
    from circuitscape_b200 import graph
    from tests import test_kernel_parity as kp
    from tests.reference_ops import ATOL

    A = kp.operator(NAME)
    opts = kp.OPERATORS[NAME][1]
    n = A.shape[0]
    rng = np.random.default_rng(21)
    B = rng.standard_normal((n, K))
    B -= B.mean(axis=0)
    src, dst = graph.all_pairs(graph.focal_nodes(n, 6, seed=5))
    sets = _sets(301, 97, 6, seed=9)
    sa, sb = np.triu_indices(len(sets), 1)
    res = {}
    fused_ran = None
    for dname, dopts in DRIVERS.items():
        with cb.B200Factor(A, kp.make_solver(config, **opts, **dopts)) as f:
            lv = f.levels()
            assert len(lv) >= 3 and lv[0]["A_stencil"], (len(lv), lv[0]["A_stencil"])
            dt = f.dtype
            if fused_ran is None:
                f.profile_spmm(True)
                f.solve_rhs(B[:, :8].astype(dt), itmax=3, raise_on_residual=False)
                fused_ran = any(k.startswith("cg_step_fused") for k in f.profile_classes())
                f.profile_spmm(False)
            for m in ITMAX:
                X, it, rr = f.solve_rhs(B.astype(dt), rtol=1e-6, itmax=m, raise_on_residual=False)
                res[f"{dname}/rhs/{m}/X"], res[f"{dname}/rhs/{m}/iters"], res[f"{dname}/rhs/{m}/relres"] = X, it, rr
                for kind in ("pairs", "regions"):
                    f.reset_currents()
                    if kind == "pairs":
                        o = f.solve_pairs(src, dst, want_volt=True, want_curr=True, accumulate=True, rtol=1e-6,
                                          itmax=m, raise_on_residual=False)
                    else:
                        o = f.solve_region_pairs(sets, sa, sb, want_volt=True, want_curr=True, accumulate=True,
                                                 rtol=1e-6, itmax=m, raise_on_residual=False)
                    cum, mx = f.read_currents()
                    for key in ("R", "volt", "curr", "iters", "relres"):
                        res[f"{dname}/{kind}/{m}/{key}"] = o[key]
                    res[f"{dname}/{kind}/{m}/cum"], res[f"{dname}/{kind}/{m}/max"] = cum, mx
            # frozen column: sqrt(rho0) = 3 atol stops it after 1-2 iterations; 7 point-source columns go on
            # (rtol 1e-10: they need far more than 6)
            quick = B[:, 0] * (3.0 * ATOL / np.sqrt(f.apply_precond(B[:, :1].astype(dt))[1][0]))
            slow = np.zeros((n, 7))
            for c in range(7):
                slow[[src[c], dst[c]], c] = [-1.0, 1.0]
            P = np.column_stack([quick, slow]).astype(dt)
            seen = {}
            for m in (1, 2, 3, 4, 5, 6):
                X, it, _ = f.solve_rhs(P, rtol=1e-10, itmax=m, raise_on_residual=False)
                assert np.all(it[1:] == m), (dname, m, it)
                seen[m] = (X[:, 0].copy(), int(it[0]))
                res[f"{dname}/frozen/{m}/X"] = X
            stop = seen[6][1]
            assert 1 <= stop < 6, stop
            for m in range(stop, 7):
                assert seen[m][1] == stop and np.array_equal(seen[m][0], seen[stop][0]), (dname, m)
    res["fused_ran"] = np.array(fused_ran)
    np.savez(out_path, **{k: np.asarray(v) for k, v in res.items()})


def _run(config, fused, tmp_path):
    out = str(tmp_path / f"{config}_{'fused' if fused else 'unfused'}.npz")
    env = dict(os.environ)
    env.pop("CS_B200_NO_FUSED_CG", None)
    if not fused:
        env["CS_B200_NO_FUSED_CG"] = "1"
    code = f"from tests.test_fused_cg_step import _collect; _collect({config!r}, {out!r})"
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return np.load(out)


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["f64", "mixed", "f32"])
def test_fused_step_is_bit_identical(config, tmp_path):
    new, old = _run(config, True, tmp_path), _run(config, False, tmp_path)
    assert bool(new["fused_ran"]) and not bool(old["fused_ran"])
    keys = sorted(k for k in new.files if k != "fused_ran")
    assert keys == sorted(k for k in old.files if k != "fused_ran")
    bad = [k for k in keys if not np.array_equal(new[k], old[k])]
    assert not bad, bad[:10]

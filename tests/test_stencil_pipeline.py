"""The pipelined stencil kernels (kernels.cuh k_stencil_pipe, k_stencil_cg_pipe: operands staged in shared memory by
cp.async several column steps ahead) against the register-gather kernels they replace (CS_B200_NO_STENCIL_PIPE).
Tiles, tile walk, grid, per-thread step order and every expression are kept, so X, iters, relres, R, voltages and
current maps must be bit-identical: solve_rhs, solve_pairs and region pairs, panels of width 8, 4, 2 and 1, fp64 /
mixed / fp32 cycles, itmax 1-6 and converged, under the device WHILE graph, host-polled graph chunks and plain
launches, with the fused CG step on and off.  Shapes: nr not a multiple of the tile rows, a ragged last raster
column, a 4-neighbour raster, nr below the tile rows, two raster columns (a tile narrower than its 16 columns),
all with fewer tiles than CTAs except the large ragged raster.  Every shape asserts that level 0 took the stencil
form.  CPU: the KT = 8 instantiations keep no per-thread stack.  The GPU cases need an H100."""
import os
import subprocess
import sys

import numpy as np
import pytest

from .test_transfer_kernels import _mangled, _resource_usage

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DRIVERS = {"graph": dict(use_graph=True), "chunk": dict(use_graph="chunk", check_every=3),
           "plain": dict(use_graph=False, check_every=3)}
K = 15                                 # panels of 8 + 4 + 2 + 1


def _operator(shape):
    from tests import test_kernel_parity as kp
    from tests.test_transfer_kernels import _raster
    if shape == "ragged8":
        return _raster("ragged8")
    if shape == "cols2":
        return kp.full(200, 2)
    return kp.operator(shape)


def _collect(shape, config, itmax, drivers, out_path):
    """Every result of the cases above for one setting of the switches, into an npz."""
    import circuitscape_b200 as cb
    from circuitscape_b200 import graph
    from tests import test_kernel_parity as kp
    from tests.test_fused_cg_step import _sets

    A = _operator(shape)
    n = A.shape[0]
    rng = np.random.default_rng(21)
    B = rng.standard_normal((n, K))
    B -= B.mean(axis=0)
    src, dst = graph.all_pairs(graph.focal_nodes(n, 5, seed=5))
    res = {}
    for dname in drivers:
        with cb.B200Factor(A, kp.make_solver(config, stencil="on", **DRIVERS[dname])) as f:
            assert f.levels()[0]["A_stencil"], shape
            dt = f.dtype
            for m in itmax:
                X, it, rr = f.solve_rhs(B.astype(dt), rtol=1e-6, itmax=m, raise_on_residual=False)
                res[f"{dname}/rhs/{m}/X"], res[f"{dname}/rhs/{m}/iters"], res[f"{dname}/rhs/{m}/relres"] = X, it, rr
                kinds = ("pairs", "regions") if shape == "full8_301x97" else ("pairs",)
                for kind in kinds:
                    f.reset_currents()
                    if kind == "pairs":
                        o = f.solve_pairs(src, dst, want_volt=True, want_curr=True, accumulate=True, rtol=1e-6,
                                          itmax=m, raise_on_residual=False)
                    else:
                        sets = _sets(301, 97, 5, seed=9)
                        sa, sb = np.triu_indices(len(sets), 1)
                        o = f.solve_region_pairs(sets, sa, sb, want_volt=True, want_curr=True, accumulate=True,
                                                 rtol=1e-6, itmax=m, raise_on_residual=False)
                    cum, mx = f.read_currents()
                    for key in ("R", "volt", "curr", "iters", "relres"):
                        res[f"{dname}/{kind}/{m}/{key}"] = o[key]
                    res[f"{dname}/{kind}/{m}/cum"], res[f"{dname}/{kind}/{m}/max"] = cum, mx
    np.savez(out_path, **{k: np.asarray(v) for k, v in res.items()})


def _run(tmp_path, shape, config, fused, pipe, itmax, drivers):
    out = str(tmp_path / f"{shape}_{config}_{int(fused)}_{int(pipe)}.npz")
    env = dict(os.environ)
    env.pop("CS_B200_NO_FUSED_CG", None)
    env.pop("CS_B200_NO_STENCIL_PIPE", None)
    if not fused:
        env["CS_B200_NO_FUSED_CG"] = "1"
    if not pipe:
        env["CS_B200_NO_STENCIL_PIPE"] = "1"
    code = (f"from tests.test_stencil_pipeline import _collect; "
            f"_collect({shape!r}, {config!r}, {tuple(itmax)!r}, {tuple(drivers)!r}, {out!r})")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return np.load(out)


def _same(new, old):
    keys = sorted(new.files)
    assert keys and keys == sorted(old.files)
    bad = [k for k in keys if not np.array_equal(new[k], old[k])]
    assert not bad, bad[:10]


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "unfused"])
@pytest.mark.parametrize("config", ["f64", "mixed", "f32"])
def test_pipeline_is_bit_identical(config, fused, tmp_path):
    args = ("full8_301x97", config, fused)
    itmax, drivers = (1, 2, 3, 4, 5, 6, 500), tuple(DRIVERS)
    _same(_run(tmp_path, *args, True, itmax, drivers), _run(tmp_path, *args, False, itmax, drivers))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["ragged8", "full4_65x43", "full8_20x37", "full8_257x29", "cols2"])
def test_pipeline_is_bit_identical_on_edge_shapes(shape, tmp_path):
    itmax, drivers = (1, 2, 500), ("graph",)
    for config in ("f64", "mixed"):
        _same(_run(tmp_path, shape, config, True, True, itmax, drivers),
              _run(tmp_path, shape, config, True, False, itmax, drivers))


# SP_CG = 1, SP_RESNORM = 2, SP_RES = 3, SP_JACOBI = 4, SP_JACOBI_DOT = 5, SP_RES0 = 7
NO_STACK = ([("k_stencil_cg_pipe", "double", 8), ("k_stencil_cg_pipe", "float", 8)] +
            [("k_stencil_pipe", t, 8, mode) for t in ("float", "double") for mode in (1, 2, 3, 4, 5, 7)])


@pytest.mark.parametrize("kernel", NO_STACK, ids=lambda k: "-".join(map(str, k)))
def test_stencil_pipe_kernels_do_not_spill(kernel):
    funcs = _resource_usage()
    key = _mangled(kernel[0], kernel[1:])
    hits = {f: s for f, s in funcs.items() if key in f}
    assert hits, f"{kernel} is not in the library"
    assert all(s == 0 for s in hits.values()), hits

"""The fused residual sweep (kernels.cuh k_stencil_res_update: r -= alpha A p, r32 = (float) r and the fp32 level-0
residual in one pass, with A p formed again from the stored p instead of stored by the CG step) against the
k_cg_update_r0 + SP_RES0 pair it replaces (CS_B200_NO_FUSED_RES).  A p is the CG step's row sum, r' the same fma,
the residual the SP_RES0 expressions, so X, iters, relres, R, voltages and current maps must be bit-identical:
solve_rhs, solve_pairs and region pairs (masked panels, which keep the pair), panels of width 8, 4, 2 and 1, fp64 /
mixed / fp32 cycles, itmax 1-6 and converged, under the device WHILE graph, host-polled graph chunks and plain
launches, on the shapes of test_stencil_pipeline.  The mixed cases assert that the fused sweep ran.  CPU: the new
kernel and the CG step without the A p store keep no per-thread stack and fit three CTAs per SM.  The GPU cases
need an H100."""
import os
import subprocess
import sys

import numpy as np
import pytest

from .test_stencil_pipeline import DRIVERS, _operator, _same
from .test_symmetric_stencil import _registers_and_stack
from .test_transfer_kernels import _mangled

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ran(shape, config, out_path):
    """How often a mixed solve on the shape launched the fused sweep, the CG step and the SP_RES0 sweep."""
    import circuitscape_b200 as cb
    from tests import test_kernel_parity as kp

    A = _operator(shape)
    B = np.random.default_rng(3).standard_normal((A.shape[0], 8))
    B -= B.mean(axis=0)
    with cb.B200Factor(A, kp.make_solver(config, stencil="on", **DRIVERS["plain"])) as f:
        f.profile_spmm(True)
        _, it, _ = f.solve_rhs(B.astype(f.dtype), itmax=4, raise_on_residual=False)
        cls = f.profile_classes()
        f.profile_spmm(False)
    count = {k: cls.get(k, (0.0, 0.0, 0))[2] for k in ("residual_sweep_fused_f64", "cg_step_fused_f64", "residual_f32")}
    np.savez(out_path, fused=count["residual_sweep_fused_f64"], cg=count["cg_step_fused_f64"],
             res0=count["residual_f32"], iters=int(np.max(it)))


def _run(tmp_path, shape, config, on, itmax, drivers):
    out = str(tmp_path / f"{shape}_{config}_{int(on)}.npz")
    env = dict(os.environ)
    env.pop("CS_B200_NO_FUSED_RES", None)
    if not on:
        env["CS_B200_NO_FUSED_RES"] = "1"
    code = (f"from tests.test_stencil_pipeline import _collect; "
            f"_collect({shape!r}, {config!r}, {tuple(itmax)!r}, {tuple(drivers)!r}, {out!r})")
    if on and config == "mixed":
        code += f"; from tests.test_fused_residual_sweep import _ran; _ran({shape!r}, {config!r}, {out + '.ran.npz'!r})"
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    if on and config == "mixed":
        ran = np.load(out + ".ran.npz")
        # one fused sweep per CG step; only the first V-cycle of the panel keeps its SP_RES0 sweep
        assert int(ran["fused"]) == int(ran["cg"]) >= int(ran["iters"]) > 0, dict(ran)
        assert int(ran["res0"]) == 1, dict(ran)
    return np.load(out)


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["f64", "mixed", "f32"])
def test_fused_residual_sweep_is_bit_identical(config, tmp_path):
    itmax, drivers = (1, 2, 3, 4, 5, 6, 500), tuple(DRIVERS)
    _same(_run(tmp_path, "full8_301x97", config, True, itmax, drivers),
          _run(tmp_path, "full8_301x97", config, False, itmax, drivers))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["ragged8", "full4_65x43", "full8_20x37", "full8_257x29", "cols2"])
def test_fused_residual_sweep_is_bit_identical_on_edge_shapes(shape, tmp_path):
    itmax, drivers = (1, 2, 500), ("graph", "chunk")
    _same(_run(tmp_path, shape, "mixed", True, itmax, drivers), _run(tmp_path, shape, "mixed", False, itmax, drivers))


# the new kernel at every panel width, and the CG step without the A p store (half form, fp32 z), at their
# __launch_bounds__ (RU_MINB, CGP_MINB = 3 CTAs per SM)
FUSED_RES_KERNELS = ([("k_stencil_res_update", "double", "float", kt) for kt in (1, 2, 4, 8)] +
                     [("k_stencil_cg_pipe", "double", kt, "float", True, False) for kt in (1, 2, 4, 8)])


@pytest.mark.parametrize("kernel", FUSED_RES_KERNELS, ids=lambda k: "-".join(map(str, k)))
def test_fused_residual_kernels_fit_three_ctas_without_stack(kernel):
    funcs = _registers_and_stack()
    key = _mangled(kernel[0], kernel[1:])
    hits = {f: v for f, v in funcs.items() if key in f}
    assert hits, f"{kernel} is not in the library"
    for f, (reg, stack) in hits.items():
        assert stack == 0, (f, stack)
        assert reg * 256 * 3 <= 65536, (f, reg)

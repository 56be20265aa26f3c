"""The finest-level grid-transfer kernels of the V-cycle: the fused prolongation + post-smoothing
(k_stencil_prolong_jacobi) and the windowed SpMM that restricts the residual (k_spmm_win).

CPU: the built library's resource usage -- the KT = 8 instantiations keep no per-thread stack (no
register spills to local memory).  GPU: one V-cycle application on rasters large enough that the
prolongation kernel's CTAs sweep many strips, with strip and run boundaries inside the raster, against
the float64 reference cycle."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                   "circuitscape_b200", "lib", "libcsb200.so")


# ---- resource usage (no GPU) -------------------------------------------------------------------
def _resource_usage():
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.isfile(LIB):
        pytest.skip("libcsb200.so is not built")
    if not os.path.isfile(cuobjdump):
        pytest.skip("cuobjdump is not available")
    out = subprocess.run([cuobjdump, "--dump-resource-usage", LIB], capture_output=True, text=True,
                         check=True).stdout
    funcs = {}
    name = None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"STACK:(\d+)", line)
        if name and m:
            funcs[name] = int(m.group(1))
            name = None
    return funcs


def _mangled(kernel, args):
    """Itanium-mangled leading template arguments of a csb kernel: (k_x, float, 8, 5) -> 3k_xIfLi8ELi5E,
    which every k_x<float, 8, 5, ...> instantiation starts with"""
    enc = {"float": "f", "double": "d", True: "Lb1E", False: "Lb0E"}
    parts = "".join(enc[a] if isinstance(a, (str, bool)) else f"Li{a}E" for a in args)
    return f"{len(kernel)}{kernel}I{parts}"


# SP_PLAIN = 0 (the restriction), SP_JACOBI = 4, SP_JACOBI_DOT = 5, SP_ADD = 6
NO_STACK = ([("k_stencil_prolong_jacobi", t, 8, mode) for t in ("float", "double") for mode in (4, 5)] +
            [("k_spmm_win", "float", 8, mode, wide) for mode in (0, 6, 4, 5) for wide in (False, True)])


@pytest.mark.parametrize("kernel", NO_STACK, ids=lambda k: "-".join(map(str, k)))
def test_transfer_kernels_do_not_spill(kernel):
    funcs = _resource_usage()
    key = _mangled(kernel[0], kernel[1:])
    hits = {f: s for f, s in funcs.items() if key in f}
    assert hits, f"{kernel} is not in {LIB}"
    assert all(s == 0 for s in hits.values()), hits


# ---- one V-cycle on large rasters (GPU) --------------------------------------------------------
def _raster(kind):
    from .test_kernel_parity import conductance, laplacian_of
    g = conductance(1100, 900, 21)
    if kind == "ragged8":
        g[500:, 899] = 0.0                 # the last raster column ends early
    return laplacian_of(g, four=kind == "full4")


def _check_vcycle(kind, config):
    """One V-cycle application (widths 1, 2, 4, 8) against the float64 reference; returns the worst error."""
    import circuitscape_b200 as cb
    from .reference_ops import vcycle
    from .test_kernel_parity import assert_path, coarse_pinv_f64, make_solver

    A = _raster(kind)
    n = A.shape[0]
    opts = dict(stencil="on")
    rng = np.random.default_rng(23)
    with cb.B200Factor(A, make_solver(config, **opts)) as f:
        lv = assert_path(f, A, "stencil")
        _, pinv = coarse_pinv_f64(A, config, opts)
        tol = 1e-10 if config == "f64" else 2e-5
        worst = 0.0
        for k in (1, 2, 4, 8):
            R = rng.standard_normal((n, k))
            if config != "f64":
                R = R.astype(np.float32).astype(np.float64)
            Z, rz = f.apply_precond(R)
            Zref = vcycle(lv, R, pinv)
            err = np.abs(Z - Zref).max() / np.abs(Zref).max()
            worst = max(worst, err)
            assert err <= tol, (k, err)
            rzref = np.einsum("ij,ij->j", R, Zref)
            assert np.all(np.abs(rz - np.abs(rzref)) <= tol * np.abs(rzref)), (k, rz, rzref)
            Z2, rz2 = f.apply_precond(R)
            assert np.array_equal(Z, Z2) and np.array_equal(rz, rz2), "two applications differ"
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["f64", "mixed", "f32"])
@pytest.mark.parametrize("kind", ["full8", "full4", "ragged8"])
def test_large_vcycle_matches_float64_reference(kind, config, record_property):
    record_property("max_rel_err", _check_vcycle(kind, config))


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["f64", "mixed"])
def test_large_vcycle_with_stored_x0(config):
    """The same check with the pre-smoothed x0 stored (CS_B200_NO_IMPLICIT_X0): the fused kernel reads x0
    from its panel instead of forming omega D^-1 b.  The switch is read once per process, hence the child."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, CS_B200_NO_IMPLICIT_X0="1")
    code = ("from tests.test_transfer_kernels import _check_vcycle; "
            f"print('max_rel_err', _check_vcycle('ragged8', {config!r}))")
    r = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]

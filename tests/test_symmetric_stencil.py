"""The half stencil form (setup_device.hpp halve_dia, kernels.cuh DiaDev::half): a bitwise symmetric stencil-form
operator is stored as its 5 upper diagonals, and the kernels take each lower diagonal from the neighbour row's
upper one.  The kernels multiply the same numbers in the same slot order, so every result must be bit-identical
to the 9-diagonal form that CS_B200_FULL_STENCIL keeps: solve_rhs, pairs and region pairs with voltage, current
and cumulative maps, fp64 / mixed / fp32 cycles, the fused CG step on and off, the three loop drivers, itmax 1-6
and converged, the edge shapes of tests/test_stencil_pipeline.py, and solve_sources after set_grounds(finite=...).
The form query (levels()[l]["A_stencil_slots"]) reports 5 on those level-0 operators, 9 for an operator one ulp
off symmetric (whose SpMM then equals the forced 9-slot form's) and under CS_B200_NO_STENCIL_PIPE, whose
register-gather kernels read 9 slots.  CPU: the half-form instantiations of the benchmark path keep no per-thread
stack and fit the registers of their CTAs per SM.  The GPU cases need an H100."""
import os
import subprocess
import sys

import numpy as np
import pytest

from .test_stencil_pipeline import DRIVERS, _same
from .test_transfer_kernels import LIB, _mangled

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = ["full8_301x97", "ragged8", "full4_65x43", "full8_20x37", "full8_257x29", "cols2"]
SWITCHES = ("CS_B200_FULL_STENCIL", "CS_B200_NO_STENCIL_PIPE", "CS_B200_NO_FUSED_CG")


def _sub(code, out, **switches):
    """run `code` in a fresh interpreter (the switches are read once per process) and load the npz it wrote"""
    env = {k: v for k, v in os.environ.items() if k not in SWITCHES}
    env.update({k: "1" for k, on in switches.items() if on})
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return np.load(out)


def _collect_run(tmp_path, shape, config, fused, full, itmax, drivers):
    out = str(tmp_path / f"{shape}_{config}_{int(fused)}_{int(full)}.npz")
    code = (f"from tests.test_stencil_pipeline import _collect; "
            f"_collect({shape!r}, {config!r}, {tuple(itmax)!r}, {tuple(drivers)!r}, {out!r})")
    return _sub(code, out, CS_B200_FULL_STENCIL=full, CS_B200_NO_FUSED_CG=not fused)


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "unfused"])
@pytest.mark.parametrize("config", ["f64", "mixed", "f32"])
def test_half_form_is_bit_identical(config, fused, tmp_path):
    args = (tmp_path, "full8_301x97", config, fused)
    itmax, drivers = (1, 2, 3, 4, 5, 6, 500), tuple(DRIVERS)
    _same(_collect_run(*args, False, itmax, drivers), _collect_run(*args, True, itmax, drivers))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES[1:])
def test_half_form_is_bit_identical_on_edge_shapes(shape, tmp_path):
    itmax, drivers = (1, 2, 500), ("graph",)
    for config in ("f64", "mixed"):
        _same(_collect_run(tmp_path, shape, config, True, False, itmax, drivers),
              _collect_run(tmp_path, shape, config, True, True, itmax, drivers))


def _grounded_sources(config, out_path):
    """solve_sources with volt / curr / cumulative maps after set_grounds(finite=...), into an npz"""
    import circuitscape_b200 as cb
    from tests import test_kernel_parity as kp
    A = kp.operator("full8_301x97")
    n = A.shape[0]
    rng = np.random.default_rng(4)
    g = np.zeros(n)
    g[rng.choice(n, 40, replace=False)] = rng.uniform(0.5, 2.0, 40)
    nodes = rng.choice(n, 6, replace=False)
    cols = [(np.array([s]), np.array([1.0])) for s in nodes]
    with cb.B200Factor(A, kp.make_solver(config, stencil="on")) as f:
        f.set_grounds(finite=g.astype(f.dtype))
        slots = f.levels()[0]["A_stencil_slots"]
        o = f.solve_sources(cols, nodes, want_volt=True, want_curr=True, accumulate=True, rtol=1e-6)
        cum, mx = f.read_currents()
    np.savez(out_path, slots=slots, volt=o["volt"], curr=o["curr"], iters=o["iters"], relres=o["relres"],
             cum=cum, max=mx)


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["f64", "mixed"])
def test_half_form_after_finite_grounds(config, tmp_path):
    res = {}
    for full in (False, True):
        out = str(tmp_path / f"grounds_{config}_{int(full)}.npz")
        code = f"from tests.test_symmetric_stencil import _grounded_sources; _grounded_sources({config!r}, {out!r})"
        res[full] = _sub(code, out, CS_B200_FULL_STENCIL=full)
    assert int(res[False]["slots"]) == 5 and int(res[True]["slots"]) == 9
    for key in ("volt", "curr", "iters", "relres", "cum", "max"):
        assert np.array_equal(res[False][key], res[True][key]), key


def _operator(shape):
    from .test_stencil_pipeline import _operator as op
    return op(shape)


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["f64", "f32"])
@pytest.mark.parametrize("shape", SHAPES)
def test_level0_reports_the_half_form(shape, config):
    import circuitscape_b200 as cb
    from tests import test_kernel_parity as kp
    with cb.B200Factor(_operator(shape), kp.make_solver(config, stencil="on")) as f:
        lv = f.levels()
        assert lv[0]["A_stencil"] and lv[0]["A_stencil_slots"] == 5
        assert all(l["A_stencil_slots"] == 0 for l in lv if not l["A_stencil"])


def _ulp_off():
    """full8_301x97 with one off-diagonal entry moved by one float32 ulp: no longer bitwise symmetric, in fp64 nor
    in its fp32 copy"""
    from tests import test_kernel_parity as kp
    A = kp.operator("full8_301x97").tocsr(copy=True)
    r = 5000
    k = next(q for q in range(A.indptr[r], A.indptr[r + 1]) if A.indices[q] == r + 1)
    A.data[k] = np.float64(np.nextafter(np.float32(A.data[k]), np.float32(np.inf)))
    return A


def _ulp_spmm(config, out_path):
    import circuitscape_b200 as cb
    from tests import test_kernel_parity as kp
    A = _ulp_off()
    X = np.random.default_rng(8).standard_normal((A.shape[0], 8))
    with cb.B200Factor(A, kp.make_solver(config, stencil="on")) as f:
        np.savez(out_path, slots=f.levels()[0]["A_stencil_slots"], Y=f.spmm(X.astype(f.dtype)))


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["f64", "f32"])
def test_one_ulp_off_symmetric_keeps_nine_slots(config, tmp_path):
    res = {}
    for full in (False, True):
        out = str(tmp_path / f"ulp_{config}_{int(full)}.npz")
        code = f"from tests.test_symmetric_stencil import _ulp_spmm; _ulp_spmm({config!r}, {out!r})"
        res[full] = _sub(code, out, CS_B200_FULL_STENCIL=full)
    assert int(res[False]["slots"]) == 9 and int(res[True]["slots"]) == 9
    assert np.array_equal(res[False]["Y"], res[True]["Y"])


@pytest.mark.gpu
def test_dirichlet_grounds_keep_the_operator_symmetric():
    """set_grounds(dirichlet=...) zeroes the node's column with its row: the operator stays bitwise symmetric and
    keeps the half form, and restoring the pristine operator keeps it too"""
    import circuitscape_b200 as cb
    from tests import test_kernel_parity as kp
    A = kp.operator("full8_301x97")
    m = np.zeros(A.shape[0], dtype=bool)
    m[[17, 4000, 12345]] = True
    with cb.B200Factor(A, kp.make_solver("f64", stencil="on")) as f:
        f.set_grounds(dirichlet=m)
        A0 = f.levels()[0]
        assert A0["A_stencil_slots"] == 5
        D = A0["A"]
        assert (D != D.T).nnz == 0
        f.set_grounds()
        assert f.levels()[0]["A_stencil_slots"] == 5


def _slots(config, out_path):
    import circuitscape_b200 as cb
    from tests import test_kernel_parity as kp
    with cb.B200Factor(kp.operator("full8_301x97"), kp.make_solver(config, stencil="on")) as f:
        np.savez(out_path, slots=[l["A_stencil_slots"] for l in f.levels()])


@pytest.mark.gpu
@pytest.mark.parametrize("switch", ["CS_B200_NO_STENCIL_PIPE", "CS_B200_FULL_STENCIL"])
def test_switches_keep_nine_slots(switch, tmp_path):
    out = str(tmp_path / "slots.npz")
    code = f"from tests.test_symmetric_stencil import _slots; _slots('mixed', {out!r})"
    slots = _sub(code, out, **{switch: True})["slots"]
    assert slots[0] == 9 and all(s in (0, 9) for s in slots)


# ---- resource usage (no GPU) -------------------------------------------------------------------
def _registers_and_stack():
    import re
    import shutil
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.isfile(LIB):
        pytest.skip("libcsb200.so is not built")
    if not os.path.isfile(cuobjdump):
        pytest.skip("cuobjdump is not available")
    out = subprocess.run([cuobjdump, "--dump-resource-usage", LIB], capture_output=True, text=True,
                         check=True).stdout
    funcs, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if name and m:
            funcs[name] = (int(m.group(1)), int(m.group(2)))
            name = None
    return funcs


# (kernel, template arguments) -> CTAs per SM of its __launch_bounds__; SP_RESNORM = 2, SP_JACOBI_DOT = 5,
# SP_RES0 = 7
HALF_ON_BENCH_PATH = {("k_stencil_cg_pipe", "double", 8, "float", True): 3,
                      ("k_stencil_pipe", "float", 8, 7, True): 3,
                      ("k_stencil_pipe", "double", 8, 2, True): 3,
                      ("k_stencil_prolong_jacobi", "float", 8, 5, 3): 3}


@pytest.mark.parametrize("kernel", list(HALF_ON_BENCH_PATH), ids=lambda k: "-".join(map(str, k)))
def test_half_form_kernels_fit_their_occupancy(kernel):
    funcs = _registers_and_stack()
    key = _mangled(kernel[0], kernel[1:])
    hits = {f: v for f, v in funcs.items() if key in f}
    assert hits, f"{kernel} is not in the library"
    minb = HALF_ON_BENCH_PATH[kernel]
    for f, (reg, stack) in hits.items():
        assert stack == 0, (f, stack)
        assert reg * 256 * minb <= 65536, (f, reg)

"""The passes around a fused AMG-PCG panel's loop (cs_b200.cu panel_ends: no X / P fills, r and r32 from one
k_panel_start pass, a pairs panel's b taken from ctl by its start pass and residual gate, no B written) against the
fills, B, copy and conversion they replace (CS_B200_NO_FUSED_PANEL_ENDS).  Only known zeros and the pairs rule are
substituted for loads, no expression or reduction order changes, so every output must be bit-identical: solve_rhs,
solve_pairs (accumulate on and off, voltages, currents), region pairs, solve_sources, solve_grounded, superposed
pairs, advanced columns with finite grounds, panels whose columns all meet their tolerance at the start (rtol 1:
a loop of 0 iterations; the C ABI refuses src == dst, whose rule test_panel_start_rhs.py checks), itmax 1 and 2 (one
and two x updates pending after the loop) and a residual-gate failure (same message).  k = 15: panels of 8, 4, 2
and 1.  Half-form mixed, full-form fp64 (CS_B200_FULL_STENCIL), windowed and plain-CSR operators, under the device WHILE graph and
plain launches.  CPU: every CG-step instantiation keeps the register count it had before the change, the other
kernels the change touches keep no per-thread stack.  The GPU cases need an H100."""
import os
import subprocess
import sys

import numpy as np
import pytest

from .test_stencil_pipeline import DRIVERS, _same
from .test_symmetric_stencil import _registers_and_stack
from .test_transfer_kernels import _mangled

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = 15
SWITCH = "CS_B200_NO_FUSED_PANEL_ENDS"


def _collect(name, config, out_path):
    """Every result of the cases above for one setting of the switch, into an npz."""
    import circuitscape_b200 as cb
    from circuitscape_b200 import graph
    from tests import test_kernel_parity as kp
    from tests.test_fused_cg_step import _sets

    A = kp.operator(name)
    opts = kp.OPERATORS[name][1]
    n = A.shape[0]
    rng = np.random.default_rng(21)
    B = rng.standard_normal((n, K))
    B -= B.mean(axis=0)
    nodes = graph.focal_nodes(n, 6, seed=5)
    src, dst = graph.all_pairs(nodes, limit=K)
    cols = [(np.array([int(nodes[c % 6]), int(nodes[(c + 1) % 6])]), np.array([1.0, -0.5 - c / K]))
            for c in range(K)]
    res = {}

    def keep(prefix, o):
        for k, v in o.items():
            if v is not None:
                res[f"{prefix}/{k}"] = np.asarray(v)

    for dname in ("graph", "plain"):
        with cb.B200Factor(A, kp.make_solver(config, **opts, **DRIVERS[dname])) as f:
            dt = f.dtype
            for m in (1, 2, 500):
                p = f"{dname}/{m}"
                X, it, rr = f.solve_rhs(B.astype(dt), rtol=1e-6, itmax=m, raise_on_residual=False)
                keep(f"{p}/rhs", dict(X=X, iters=it, relres=rr))
                for acc in (True, False):
                    f.reset_currents()
                    o = f.solve_pairs(src, dst, want_volt=True, want_curr=True, accumulate=acc, rtol=1e-6, itmax=m,
                                      raise_on_residual=False)
                    keep(f"{p}/pairs{int(acc)}", o)
                    keep(f"{p}/pairs{int(acc)}/maps", dict(zip(("cum", "max"), f.read_currents())))
                f.reset_currents()
                keep(f"{p}/pairs_novolt", f.solve_pairs(src, dst, accumulate=True, rtol=1e-6, itmax=m,
                                                        raise_on_residual=False))
                keep(f"{p}/pairs_novolt/maps", dict(zip(("cum", "max"), f.read_currents())))
                f.reset_currents()
                # rtol 1: every column meets its tolerance at the start, the loop runs 0 iterations
                keep(f"{p}/inactive", f.solve_pairs(src, dst, want_volt=True, want_curr=True, accumulate=True,
                                                    rtol=1.0, itmax=m, raise_on_residual=False))
                keep(f"{p}/inactive/maps", dict(zip(("cum", "max"), f.read_currents())))
                f.reset_currents()
                keep(f"{p}/superposed", f.solve_pairs_superposed(nodes, np.zeros(K, np.int64), np.arange(K) % 5 + 1,
                                                                 want_volt=True, want_curr=True, accumulate=True,
                                                                 rtol=1e-6, itmax=m, raise_on_residual=False))
                keep(f"{p}/sources", f.solve_sources(cols, np.full(K, nodes[0]), probe=nodes, want_volt=True,
                                                     want_curr=True, rtol=1e-6, itmax=m, raise_on_residual=False))
                if name == "full8_301x97":
                    sets = _sets(301, 97, 5, seed=9)
                    sa, sb = np.triu_indices(len(sets), 1)
                    keep(f"{p}/regions", f.solve_region_pairs(sets, sa, sb, want_volt=True, want_curr=True,
                                                              rtol=1e-6, itmax=m, raise_on_residual=False))
                    gset = np.arange(K) % len(sets)
                    srcs = [(np.array([int(nodes[c % 6])]), np.array([1.0])) for c in range(K)]
                    keep(f"{p}/grounded", f.solve_grounded(sets, gset, srcs, want_volt=True, want_curr=True,
                                                           rtol=1e-6, itmax=m, raise_on_residual=False))
            try:                                                  # the residual gate after one iteration
                f.solve_pairs(src, dst, itmax=1)
                res[f"{dname}/gate"] = np.array("passed")
            except Exception as e:  # noqa: BLE001
                res[f"{dname}/gate"] = np.array(f"{type(e).__name__}: {e}")
            # advanced columns: finite grounds on every node (the fg path of the node currents), last because
            # set_grounds re-derives the operator
            f.set_grounds(finite=np.full(n, 0.01 if config != "f32" else 0.05).astype(dt))
            srcs = [(np.array([int(nodes[c % 6])]), np.array([1.0 + c])) for c in range(K)]
            for m in (1, 2, 500):
                f.reset_currents()
                keep(f"{dname}/{m}/advanced", f.solve_advanced([], np.full(K, -1), srcs, want_volt=True,
                                                               want_curr=True, accumulate=True, rtol=1e-6, itmax=m,
                                                               raise_on_residual=False))
                keep(f"{dname}/{m}/advanced/maps", dict(zip(("cum", "max"), f.read_currents())))
    np.savez(out_path, **res)


def _run(tmp_path, name, config, on, extra_env=()):
    out = str(tmp_path / f"{name}_{config}_{int(on)}.npz")
    env = dict(os.environ)
    env.pop(SWITCH, None)
    if not on:
        env[SWITCH] = "1"
    env.update(dict(extra_env))
    code = f"from tests.test_panel_ends import _collect; _collect({name!r}, {config!r}, {out!r})"
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return np.load(out)


CASES = [("full8_301x97", "mixed", ()), ("full8_301x97", "f64", ()), ("full8_301x97", "f32", ()),
         ("full8_301x97", "f64", (("CS_B200_FULL_STENCIL", "1"),)),
         ("holey_windowed", "mixed", ()), ("holey_plain", "mixed", ())]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}-{c[1]}" + ("-full" if c[2] else ""))
def test_panel_ends_are_bit_identical(case, tmp_path):
    name, config, env = case
    new, old = _run(tmp_path, name, config, True, env), _run(tmp_path, name, config, False, env)
    _same(new, old)
    assert "Residual" in str(new["graph/gate"]) or "residual" in str(new["graph/gate"]), str(new["graph/gate"])


# Registers (cuobjdump --dump-resource-usage, sm_90a) of every instantiation of the CG step, whose zero staging at
# iterations 0 and 1 must not cost the loop a register: the counts of the library before the change
CG_STEP_REGS = {("double", 1, "double", False, True): 70, ("double", 1, "double", True, True): 72,
                ("double", 1, "float", False, True): 70, ("double", 1, "float", True, False): 72,
                ("double", 1, "float", True, True): 72,
                **{("double", kt, tv, half, ap): 80 for kt in (2, 4, 8) for tv, half, ap in
                   (("double", False, True), ("double", True, True), ("float", False, True),
                    ("float", True, False), ("float", True, True))},
                ("double", 8, "double", False, True): 78,
                ("float", 1, "float", False, True): 58, ("float", 1, "float", True, True): 58,
                ("float", 2, "float", False, True): 77, ("float", 2, "float", True, True): 79,
                **{("float", kt, "float", half, True): 80 for kt in (4, 8) for half in (False, True)}}


@pytest.mark.parametrize("args", sorted(CG_STEP_REGS, key=str), ids=lambda k: "-".join(map(str, k)))
def test_cg_step_keeps_its_registers(args):
    funcs = _registers_and_stack()
    key = _mangled("k_stencil_cg_pipe", args)
    hits = {f: v for f, v in funcs.items() if key in f}
    assert len(hits) == 1, (args, list(hits))
    (reg, stack), = hits.values()
    assert stack == 0 and reg == CG_STEP_REGS[args], (args, reg, stack)


# the other kernels the change touches, at every panel width: the residual gate (b from ctl), the x tail and the
# start pass.  The tail is launched once per panel: at <= 32 registers its 256-thread CTAs still fill an SM.
TOUCHED = ([("k_stencil_pipe", t, kt, 2, half) for t in ("double", "float") for kt in (1, 2, 4, 8)
            for half in (False, True)] +
           [("k_cg_x_tail", t, kt) for t in ("double", "float") for kt in (1, 2, 4, 8)] +
           [("k_panel_start", t, kt) for t in ("double", "float") for kt in (1, 2, 4, 8)])


@pytest.mark.parametrize("kernel", TOUCHED, ids=lambda k: "-".join(map(str, k)))
def test_panel_end_kernels_keep_no_stack(kernel):
    funcs = _registers_and_stack()
    key = _mangled(kernel[0], kernel[1:])
    hits = {f: v for f, v in funcs.items() if key in f}
    assert hits, f"{kernel} is not in the library"
    for f, (reg, stack) in hits.items():
        assert stack == 0, (f, stack)
        if kernel[0] == "k_cg_x_tail":
            assert reg <= 32, (f, reg)

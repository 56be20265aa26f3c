"""The per-launch profile (cs_b200_profile_spmm / _classes_n / _bytes) accounts for every finest-level launch once:
over one profiled solve_pairs call of k = 15 columns (panels of 8, 4, 2 and 1) the launches summed over
profile_classes() equal the call's stats()["spmm_launches"], the bytes summed over the classes equal
profile_bytes(), and the kernel classes of the handle's iteration are the ones that appear.  Five handles: a
half-form stencil raster under mixed AMG (fused CG step and fused residual sweep), the same with
CS_B200_NO_FUSED_RES (the CG step stores A p and the fp32 cycle keeps its level-0 SP_RES0 sweep), the same in fp64
with the fp32 cycle off, a windowed raster with NODATA holes and a plain-CSR operator.  Each runs in a child
process, so the switch is read fresh.  Needs an H100."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K = 15

# name -> (operator, solver options, CS_B200_NO_FUSED_RES, operator form, classes that must appear, must not appear)
CASES = {
    "stencil_mixed": ("stencil", dict(mixed=True, stencil="on"), False, "stencil",
                      {"cg_step_fused_f64", "residual_sweep_fused_f64", "residual_f32", "prolong_jacobi_fused_f32",
                       "residual_gate_f64"}, {"cg_f64"}),
    "stencil_mixed_no_fused_res": ("stencil", dict(mixed=True, stencil="on"), True, "stencil",
                                   {"cg_step_fused_f64", "residual_f32", "prolong_jacobi_fused_f32",
                                    "residual_gate_f64"}, {"residual_sweep_fused_f64"}),
    "stencil_f64": ("stencil", dict(mixed=False, stencil="on"), False, "stencil",
                    {"cg_step_fused_f64", "residual_f64", "prolong_jacobi_fused_f64", "residual_gate_f64"},
                    {"residual_sweep_fused_f64", "residual_f32", "prolong_jacobi_fused_f32"}),
    "windowed_mixed": ("holes", dict(mixed=True), False, "windowed",
                       {"cg_f64", "residual_f32", "jacobi_dot_f32", "residual_gate_f64"},
                       {"cg_step_fused_f64", "residual_sweep_fused_f64"}),
    "csr_mixed": ("csr", dict(mixed=True, window="off", stencil="off"), False, "csr",
                  {"cg_f64", "residual_f32", "jacobi_dot_f32", "residual_gate_f64"},
                  {"cg_step_fused_f64", "residual_sweep_fused_f64"}),
}


def _operator(kind):
    from circuitscape_b200 import graph
    from tests import test_kernel_parity as kp
    if kind == "stencil":
        return kp.full(301, 97)
    holes = 1.0 / np.random.default_rng(3).uniform(1.0, 10.0, size=(190, 130))
    holes[np.random.default_rng(4).random(holes.shape) < 0.04] = 0.0
    nm = graph.construct_node_map(holes, None)
    G = graph.laplacian(graph.construct_graph(holes, nm, False, False))
    big = max(graph.connected_components(G), key=len) - 1
    L = G[big][:, big].tocsr()
    return L if kind == "holes" else L[:9000][:, :9000].tocsr()


def _account(case, out_path):
    """One profiled solve_pairs call on the case's handle: its form, {class: (bytes, launches)}, profile_bytes()
    and stats()["spmm_launches"], as JSON."""
    import circuitscape_b200 as cb
    kind, opts = CASES[case][:2]
    L = _operator(kind)
    pick = np.random.default_rng(7).choice(L.shape[0], size=2 * K, replace=False)
    with cb.B200Factor(L, cb.CUDASolver(**opts)) as f:
        f.profile_spmm(True)
        f.solve_pairs(pick[:K], pick[K:])
        out = dict(form=f.operator_form(), classes={c: [b, n] for c, (_, b, n) in f.profile_classes().items()},
                   bytes=f.profile_bytes(), spmm_launches=f.stats()["spmm_launches"])
        f.profile_spmm(False)
    with open(out_path, "w") as fh:
        json.dump(out, fh)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_profile_accounts_for_every_finest_level_launch(case, tmp_path):
    _, _, no_fused_res, form, present, absent = CASES[case]
    out = str(tmp_path / f"{case}.json")
    env = dict(os.environ)
    env.pop("CS_B200_NO_FUSED_RES", None)
    if no_fused_res:
        env["CS_B200_NO_FUSED_RES"] = "1"
    code = f"from tests.test_profile_accounting import _account; _account({case!r}, {out!r})"
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    with open(out) as fh:
        got = json.load(fh)
    classes = got["classes"]
    assert got["form"] == form, got
    assert sum(n for _, n in classes.values()) == got["spmm_launches"] > 0, got
    assert sum(b for b, _ in classes.values()) == pytest.approx(got["bytes"], rel=1e-12), got
    assert present <= set(classes), (sorted(present - set(classes)), got)
    assert not absent & set(classes), (sorted(absent & set(classes)), got)

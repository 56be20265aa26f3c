"""The one create sequence behind every cs_b200_create* entry: each entry built by the host builder and by the
device builder (opts.setup) gives the same operator and the same hierarchy, the borrowed-CSR and broadcast entries
solve, and a create that fails after its handle exists reports why and leaves the thread ready for the next
create.  Needs an H100: `pytest -m gpu`."""
import numpy as np
import pytest
import torch  # before the library loads NCCL (cs_b200_create_bcast), so that torch binds its own

import circuitscape_b200 as cb
from circuitscape_b200 import _lib, dist, graph
from oracle import circuitscape_oracle as co

pytestmark = pytest.mark.gpu

SETUPS = ("host", "device")


def _raster():
    g = 1.0 / np.random.default_rng(9).uniform(1.0, 10.0, size=(200, 170))
    return g, graph.stencil_laplacian_from_conductance(g).tocsr()


def _solver(setup):
    # fp64 cycle and windows everywhere: nothing is rounded, every operator has a form to compare
    return cb.CUDASolver(setup=setup, mixed=False, window="on")


def _from_device(A, solver):
    dev = torch.device("cuda", solver.device)
    rp = torch.from_numpy(A.indptr.astype(np.int32)).to(dev)
    ci = torch.from_numpy(A.indices.astype(np.int32)).to(dev)
    va = torch.from_numpy(np.ascontiguousarray(A.data, dtype=np.float64)).to(dev)
    return dist.factor_from_device(A.shape[0], A.nnz, rp, ci, va, solver)


def _single_rank_comm():
    try:
        return dist.Comm(0, 0, 1, lambda raw: raw)
    except _lib.B200Error as e:
        if e.code == _lib.ERR_UNSUPPORTED:
            pytest.skip(f"cs_b200_create_bcast needs NCCL, which the library cannot load: {e}")
        raise


def _entries():
    g, A = _raster()
    return {
        "create": lambda s: cb.B200Factor(A, s),
        "from_device": lambda s: _from_device(A, s),
        "from_raster": lambda s: cb.B200Factor.from_raster(g, s),
        "from_raster_polygons": lambda s: cb.B200Factor.from_raster_polygons(g, None, s)[0],
        "bcast": lambda s: _single_rank_comm().create_factor(A, s),
    }


def _same_levels(H, D):
    """the comparisons of test_device_setup.py::test_hierarchy_device_matches_host"""
    assert len(H) == len(D) >= 3
    for l, (h, d) in enumerate(zip(H, D)):
        assert abs(h["omega"] - d["omega"]) <= 1e-12 * h["omega"], l
        for name in ("A", "P", "R"):
            if h[name] is None:
                assert d[name] is None
                continue
            assert h[name].shape == d[name].shape and h[name].nnz == d[name].nnz, (l, name)
            assert np.array_equal(h[name].indptr, d[name].indptr) and np.array_equal(h[name].indices, d[name].indices)
            scale = np.abs(h[name].data).max()
            assert np.abs(h[name].data - d[name].data).max() <= 1e-12 * scale, (l, name)
            assert d[name + "_windowed"] == h[name + "_windowed"], (l, name)
        if d["P"] is not None:
            assert abs(d["R"] - d["P"].T).max() == 0.0
            Ac = (d["R"] @ d["A"] @ d["P"]).tocsr()
            assert abs(Ac - D[l + 1]["A"]).max() <= 1e-12 * abs(Ac).max()
    assert D[-1]["A"].shape[0] <= 200


@pytest.mark.parametrize("entry", ["create", "from_device", "from_raster", "from_raster_polygons", "bcast"])
def test_every_entry_same_hierarchy_from_both_builders(entry):
    make = _entries()[entry]
    csr, lv = {}, {}
    for setup in SETUPS:
        with make(_solver(setup)) as f:
            csr[setup], lv[setup] = f.get_csr(), f.levels()
    assert (csr["host"] != csr["device"]).nnz == 0
    _same_levels(lv["host"], lv["device"])


@pytest.mark.parametrize("entry", ["from_device", "bcast"])
def test_borrowed_and_broadcast_entries_solve(entry):
    _, A = _raster()
    nodes = graph.focal_nodes(A.shape[0], 4, seed=7)
    src, dst = graph.all_pairs(nodes)
    Vref = co.solve_pairs_direct(A, src, dst)
    Rref = Vref[dst, np.arange(len(src))]
    csr = {}
    for setup in SETUPS:
        with _entries()[entry](cb.CUDASolver(setup=setup)) as f:
            csr[setup] = f.get_csr()
            R = f.solve_pairs(src, dst)["R"]
        assert np.abs(R - Rref).max() <= 1e-6 * np.abs(Rref).max(), setup
    assert (csr["host"] != csr["device"]).nnz == 0
    assert abs(csr["device"] - A).max() == 0


@pytest.mark.parametrize("setup", SETUPS)
@pytest.mark.parametrize("polygons", [False, True])
def test_failed_create_reports_and_next_create_succeeds(polygons, setup):
    """An all-zero raster is refused by the assembler, after the handle exists: ERR_ARG, its text in
    cs_b200_last_error(NULL), the same under both builders, and the thread's next create works."""
    lib = _lib.load()
    solver = cb.CUDASolver(setup=setup)
    create = ((lambda g: cb.B200Factor.from_raster_polygons(g, None, solver)[0]) if polygons
              else (lambda g: cb.B200Factor.from_raster(g, solver)))
    with pytest.raises(_lib.B200Error) as e:
        create(np.zeros((40, 30)))
    assert e.value.code == _lib.ERR_ARG
    assert lib.cs_b200_last_error(None) == b"raster has no cell with conductance > 0"
    assert str(e.value) == "raster has no cell with conductance > 0"
    g, A = _raster()
    with create(g) as f:
        assert f.n == A.shape[0]

"""The right-hand side the start pass of a pairs panel forms (kernels.cuh pair_rhs_at / pair_rhs_val, which
k_panel_start evaluates per element) against a numpy rendering of the sequence it replaces: B zero-filled,
k_pair_rhs (-1 at src, +1 at dst, only where both are >= 0 and differ), R copied from B, R32 = (float) R.  Bit for
bit, the sign of every zero included, for panel widths 1, 2, 4 and 8 in fp64 and fp32, with columns whose src or dst
is negative, columns with src == dst and pairs on the first and last rows.  CPU only: the harness is compiled for
the host with nvcc."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    nvcc = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.isfile(nvcc):
        pytest.skip("nvcc is not available")
    so = str(tmp_path_factory.mktemp("panel_start") / "panel_start_harness.so")
    subprocess.check_call([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-shared",
                           "-Xcompiler", "-fPIC", "-o", so, os.path.join(HERE, "panel_start_harness.cu")])
    lib = C.CDLL(so)
    lib.panel_start_pairs.restype = C.c_int
    lib.panel_start_pairs.argtypes = [C.c_int, C.c_int, C.c_longlong] + [C.c_void_p] * 4
    return lib


def _replaced_sequence(n_pad, kt, src, dst, dtype):
    """memset(B) + k_pair_rhs + memcpy(R <- B) + k_convert(R -> R32)"""
    B = np.zeros((n_pad, kt), dtype=dtype)
    for c in range(kt):
        s, d = int(src[c]), int(dst[c])
        if s >= 0 and d >= 0 and s != d:
            B[s, c] = -1
            B[d, c] = 1
    R = B.copy()
    return R, R.astype(np.float32)


def _columns(rng, n, kt):
    src = rng.integers(0, n, kt)
    dst = rng.integers(0, n, kt)
    special = [(-1, 3), (5, -1), (7, 7), (0, n - 1), (n - 1, 0), (-1, -1)]
    for c in range(kt):
        if rng.random() < 0.5:
            src[c], dst[c] = special[rng.integers(len(special))]
    return src.astype(np.int64), dst.astype(np.int64)


@pytest.mark.parametrize("dtype", [np.float64, np.float32], ids=["fp64", "fp32"])
@pytest.mark.parametrize("kt", [1, 2, 4, 8])
def test_start_pass_writes_what_the_replaced_sequence_wrote(harness, kt, dtype):
    rng = np.random.default_rng(kt)
    for n in (1, 9, 37, 1000):
        n_pad = (n + 3) // 4 * 4
        for _ in range(8):
            src, dst = _columns(rng, n, kt)
            R = np.full((n_pad, kt), np.nan, dtype=dtype)
            R32 = np.full((n_pad, kt), np.nan, dtype=np.float32)
            rc = harness.panel_start_pairs(kt, 1 if dtype == np.float64 else 0, n_pad, src.ctypes.data,
                                           dst.ctypes.data, R.ctypes.data, R32.ctypes.data)
            assert rc == 0
            want_R, want_R32 = _replaced_sequence(n_pad, kt, src, dst, dtype)
            ui = np.uint64 if dtype == np.float64 else np.uint32
            assert np.array_equal(R.view(ui), want_R.view(ui)), (n, src, dst)
            assert np.array_equal(R32.view(np.uint32), want_R32.view(np.uint32)), (n, src, dst)

"""Pair sharding across GPUs (one process per GPU, torch.distributed).

The path shards over *independent focal pairs* against one replicated read-only
matrix -- the same axis the reference parallelises with threads
(src/core.jl:262-272).  Collectives, all outside the solve itself:
  * one broadcast of the CSR arrays from rank 0        (NCCL on GPUs)
  * one all_gather of per-pair resistances / iterations
  * optional all_reduce SUM of cumulative and MAX of max node-current vectors
CPU tests exercise the same code with the gloo backend (tests/test_dist_gloo.py).
"""
from __future__ import annotations

import ctypes as C

import numpy as np


def shard_pairs(npairs, rank, world):
    """Round-robin pair indices of `rank` (equalises count; iteration-count skew is
    reported per rank by the benchmark)."""
    return np.arange(rank, npairs, world, dtype=np.int64)


def broadcast_csr(csr, dist, device, src=0):
    """Broadcast (rowptr int32, colidx int32, vals) from `src`; returns torch tensors
    resident on `device` on every rank.  `csr` is a scipy CSR on rank src, None elsewhere."""
    import torch
    rank = dist.get_rank()
    meta = torch.zeros(3, dtype=torch.int64, device=device)
    if rank == src:
        is64 = 1 if csr.data.dtype == np.float64 else 0
        meta = torch.tensor([csr.shape[0], csr.nnz, is64], dtype=torch.int64, device=device)
    dist.broadcast(meta, src=src)
    n, nnz, is64 = (int(x) for x in meta.tolist())
    vdt = torch.float64 if is64 else torch.float32
    if rank == src:
        rowptr = torch.from_numpy(np.ascontiguousarray(csr.indptr, dtype=np.int32)).to(device)
        colidx = torch.from_numpy(np.ascontiguousarray(csr.indices, dtype=np.int32)).to(device)
        vals = torch.from_numpy(np.ascontiguousarray(csr.data)).to(device)
    else:
        rowptr = torch.empty(n + 1, dtype=torch.int32, device=device)
        colidx = torch.empty(nnz, dtype=torch.int32, device=device)
        vals = torch.empty(nnz, dtype=vdt, device=device)
    for t in (rowptr, colidx, vals):
        dist.broadcast(t, src=src)
    return n, nnz, rowptr, colidx, vals


def factor_from_device(n, nnz, rowptr, colidx, vals, solver, log_transform=False):
    """cs_b200_create_from_device on tensors that already live on solver.device."""
    import torch
    from . import _lib
    from .solver import B200Factor
    lib = _lib.load()
    f = B200Factor.__new__(B200Factor)
    f._lib = lib
    f._h = C.c_void_p()
    f.n = n
    f.dtype = np.dtype(np.float64 if vals.dtype == torch.float64 else np.float32)
    f.io_dtype = f.dtype
    f.solver = solver
    f._keep = (rowptr, colidx, vals)      # the handle borrows these buffers
    opts = B200Factor._opts(solver, log_transform)
    torch.cuda.synchronize()   # the broadcast ran on torch's streams; the library uses its own
    rc = lib.cs_b200_create_from_device(n, nnz, C.c_void_p(rowptr.data_ptr()), C.c_void_p(colidx.data_ptr()),
                                        C.c_void_p(vals.data_ptr()), _lib.dtype_code(f.dtype),
                                        solver.device, C.byref(opts), C.byref(f._h))
    _lib.check(lib, None, rc)
    return f


class Comm:
    """NCCL communicator behind the C ABI (cs_b200_comm_*): what a Julia host would use.  The only
    thing the host language moves is the 128-byte unique id from rank 0 to the other ranks --
    `exchange(id_bytes_or_None) -> id_bytes` (torch.distributed broadcast, MPI, a file ...)."""

    def __init__(self, device, rank, nranks, exchange):
        from . import _lib
        self._lib = lib = _lib.load()
        self.rank, self.nranks, self.device = rank, nranks, device
        ident = (C.c_char * 128)()
        if rank == 0:
            _lib.check(lib, None, lib.cs_b200_comm_unique_id(C.cast(ident, C.c_void_p)))
        raw = exchange(bytes(ident.raw) if rank == 0 else None)
        buf = (C.c_char * 128).from_buffer_copy(raw)
        self._c = C.c_void_p()
        rc = lib.cs_b200_comm_init(device, rank, nranks, C.cast(buf, C.c_void_p), C.byref(self._c))
        self._check(rc, None)

    def _check(self, rc, c):
        if rc != 0:
            from . import _lib
            msg = self._lib.cs_b200_comm_last_error(c)
            raise _lib.B200Error(rc, msg.decode() if msg else f"libcsb200 comm error {rc}")

    def close(self):
        if getattr(self, "_c", None) is not None and self._c.value:
            self._lib.cs_b200_comm_destroy(self._c)
            self._c = C.c_void_p()

    __del__ = close

    def create_factor(self, matrix, solver, root=0, shape=None, log_transform=False):
        """cs_b200_create_bcast: `matrix` (scipy CSR) on the root, None elsewhere; `shape` =
        (n, nnz, is_f64) must be known on every rank (the host broadcasts three integers)."""
        from . import _lib
        from .solver import B200Factor
        f = B200Factor.__new__(B200Factor)
        f._bind(solver)
        opts = B200Factor._opts(solver, log_transform)
        if matrix is not None:
            n, nnz, rp, ci, vals, bits = f._host_csr(matrix)
            args = (_lib._ptr(rp), _lib._ptr(ci), _lib._ptr(vals))
        else:
            n, nnz = int(shape[0]), int(shape[1])
            bits = 32
            args = (None, None, None)
        f.n = n
        rc = self._lib.cs_b200_create_bcast(self._c, root, n, nnz, *args, bits, 0, _lib.dtype_code(f.dtype),
                                            C.byref(opts), C.byref(f._h))
        self._check(rc, self._c)
        return f

    def reduce_currents(self, factor):
        self._check(self._lib.cs_b200_comm_reduce_currents(self._c, factor._h), self._c)

    def gather_pairs(self, local_idx, local_vals, npairs):
        from . import _lib
        idx = np.ascontiguousarray(local_idx, dtype=np.int64)
        val = np.ascontiguousarray(local_vals, dtype=np.float64)
        out = np.empty(npairs, dtype=np.float64)
        rc = self._lib.cs_b200_comm_gather_pairs(self._c, npairs, _lib._ptr(idx), len(idx), _lib._ptr(val), _lib._ptr(out))
        self._check(rc, self._c)
        return out

    def max(self, values):
        from . import _lib
        v = np.ascontiguousarray(values, dtype=np.float64).copy()
        self._check(self._lib.cs_b200_comm_max_double(self._c, _lib._ptr(v), len(v)), self._c)
        return v

    def barrier(self):
        self._check(self._lib.cs_b200_comm_barrier(self._c), self._c)


def gather_pairs(local_idx, local_vals, npairs, dist, device="cpu"):
    """all_gather variable-length (index, value) shards into a dense length-npairs
    vector on every rank."""
    import torch
    world = dist.get_world_size()
    cnt = (npairs + world - 1) // world
    idx = torch.full((cnt,), -1, dtype=torch.int64, device=device)
    val = torch.zeros(cnt, dtype=torch.float64, device=device)
    idx[: len(local_idx)] = torch.as_tensor(np.asarray(local_idx), dtype=torch.int64, device=device)
    val[: len(local_idx)] = torch.as_tensor(np.asarray(local_vals, dtype=np.float64), device=device)
    idxs = [torch.empty_like(idx) for _ in range(world)]
    vals = [torch.empty_like(val) for _ in range(world)]
    dist.all_gather(idxs, idx)
    dist.all_gather(vals, val)
    out = np.zeros(npairs, dtype=np.float64)
    for i, v in zip(idxs, vals):
        i, v = i.cpu().numpy(), v.cpu().numpy()
        ok = i >= 0
        out[i[ok]] = v[ok]
    return out


class _DevArray:
    """__cuda_array_interface__ view of a raw device pointer (for torch.as_tensor)."""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False),
                                         "version": 2}


def reduce_currents(factor, dist):
    """all_reduce the handle's cumulative (SUM) and max (MAX) node-current vectors in
    place on the device, over NCCL."""
    import torch
    dcum, dmax = factor.currents_device_ptrs()
    ts = "<f8" if factor.dtype == np.float64 else "<f4"
    dev = f"cuda:{factor.solver.device}"
    cum = torch.as_tensor(_DevArray(dcum, factor.n, ts), device=dev)
    mx = torch.as_tensor(_DevArray(dmax, factor.n, ts), device=dev)
    dist.all_reduce(cum, op=dist.ReduceOp.SUM)
    dist.all_reduce(mx, op=dist.ReduceOp.MAX)
    torch.cuda.synchronize()

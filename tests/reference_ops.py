"""Float64 references of the operations the CUDA kernels implement, in plain numpy / scipy.

    vcycle(levels, r)             the Jacobi-smoothed V(1,1) cycle the device runs as its preconditioner
    pcg(A, B, precond, rtol, itmax)
                                  the device's PCG recurrence, column by column: deferred x update, stop
                                  test, stall guard and per-column freezing (csrc/kernels.cuh
                                  cg_after_precond, k_cg_*)
    true_relres(A, X, B)          ||B - A X|| / ||B|| per column (the reference's residual gate,
                                  src/core.jl:640-650)
    node_currents(A, v)           per-node currents with the 1e-8 relative zeroing (src/out.jl:178-290)
    stencil_wraps(A)              what the device's stencil-form detection sees in an operator

`levels` is a list of dicts with A, P, R (None on the coarsest level) and omega, as
`B200Factor.levels()` returns them (the fp32 values of a mixed cycle widened to fp64) or as the host
hierarchy harness builds them.
"""
import numpy as np
import scipy.sparse as sp

DENSE_COARSE_LIMIT = 320      # coarsest operators up to this size are solved with a dense pseudo-inverse


def coarse_pinv(A):
    """Pseudo-inverse of a (possibly singular) symmetric coarse operator: eigenvalues below
    1e-10 n lambda_max are the null space (amg_host.hpp dense_pinv)."""
    A = np.asarray(A.toarray() if sp.issparse(A) else A, dtype=np.float64)
    n = A.shape[0]
    w, V = np.linalg.eigh((A + A.T) / 2.0)
    lmax = np.abs(w).max() if n else 0.0
    keep = w > lmax * 1e-10 * max(1, n)
    return (V[:, keep] / w[keep]) @ V[:, keep].T


def vcycle(levels, r, pinv=None):
    """z = M^-1 r for r of shape (n,) or (n, k).  `pinv`: pseudo-inverse of the coarsest operator
    (default: coarse_pinv of levels[-1]["A"]; used only when that level has <= 320 rows)."""
    r = np.asarray(r, dtype=np.float64)
    if pinv is None and levels[-1]["A"].shape[0] <= DENSE_COARSE_LIMIT:
        pinv = coarse_pinv(levels[-1]["A"])
    return _vcycle(levels, pinv, r, 0)


def _vcycle(levels, pinv, b, l):
    L = levels[l]
    A = L["A"]
    dinv = 1.0 / A.diagonal()
    if b.ndim == 2:
        dinv = dinv[:, None]
    om = L["omega"]
    if l == len(levels) - 1:
        if A.shape[0] <= DENSE_COARSE_LIMIT:
            return pinv @ b
        # coarsening stopped above the dense limit: 4 damped-Jacobi sweeps from zero
        x = om * dinv * b
        for _ in range(3):
            x = x + om * dinv * (b - A @ x)
        return x
    x = om * dinv * b
    x = x + L["P"] @ _vcycle(levels, pinv, L["R"] @ (b - A @ x), l + 1)
    return x + om * dinv * (b - A @ x)


ATOL = float(np.sqrt(np.finfo(np.float64).eps))     # the device's default absolute tolerance


def _coldots(U, V):
    """r.z per column, each column its own contiguous fp64 dot (a column's value does not depend on
    the other columns of the panel)."""
    return np.array([np.dot(U[:, c].astype(np.float64), V[:, c].astype(np.float64))
                     for c in range(U.shape[1])])


def pcg(A, B, precond, rtol, itmax, atol=ATOL, stall_limit=40, dtype=np.float64):
    """The device's preconditioned CG recurrence for B of shape (n,) or (n, k), column by column
    (csrc/kernels.cuh cg_after_precond, k_cg_init / k_cg_update_r / k_cg_update_xp, k_cg_update_r0 /
    k_cg_update_xp2, the SP_CG epilogue):

        x = 0, r = b, z = M^-1 r, p = z, rho0 = |r.z|, tol = atol + rtol sqrt(rho0)
        active  <=>  rho0 > 0 and sqrt(rho0) > tol and itmax > 0
        per iteration of an active column:
            alpha = rho / p.Ap  (0 if p.Ap <= 0) ;  r -= alpha Ap ;  z = M^-1 r ;  rho' = |r.z|
            beta = rho' / rho ;  stall guard: rho' < 0.81 best resets the counter, `stall_limit`
            iterations without that freeze the column ;  stop: !(sqrt(rho') > tol) or it >= itmax
            x += alpha p  (the deferred update runs on the stopping iteration too) ;  p = z + beta p
        a frozen column is never touched again.

    `precond(R)` maps an (n, j) panel to M^-1 R (Jacobi: D^-1 R, whose r.z is the device's r.D^-1 r).
    `dtype` is the storage type of x, r, p, z and A p; alpha, beta and the dots stay fp64, as on the
    device.  The device's AMG path uses stall_limit = 40, its Jacobi path 2000.

    Returns (X (n, k), iters (k,), rho (iterations + 1, k), tol (k,)): rho[j, c] is column c's rho
    after iteration j (rho0 at j = 0), NaN where the column had already stopped."""
    dtype = np.dtype(dtype)
    B = np.asarray(B, dtype=dtype)
    B = B.reshape(B.shape[0], -1)
    n, k = B.shape
    X = np.zeros((n, k), dtype=dtype)
    R = B.copy()
    Z = np.asarray(precond(R), dtype=dtype).reshape(n, k)
    P = Z.copy()
    rho = np.abs(_coldots(R, Z))
    tol = atol + rtol * np.sqrt(rho)
    active = (rho > 0) & (np.sqrt(rho) > tol) & (itmax > 0)
    iters = np.zeros(k, dtype=np.int64)
    best, stall = rho.copy(), np.zeros(k, dtype=np.int64)
    hist = [rho.copy()]
    it = 0
    while active.any():
        it += 1
        c = np.nonzero(active)[0]
        AP = np.asarray(A @ P[:, c], dtype=dtype).reshape(n, c.size)
        pap = _coldots(P[:, c], AP)
        alpha = np.where(pap > 0, rho[c] / np.where(pap > 0, pap, 1.0), 0.0)
        Rc = R[:, c] - alpha.astype(dtype) * AP
        Zc = np.asarray(precond(Rc), dtype=dtype).reshape(n, c.size)
        rn = np.abs(_coldots(Rc, Zc))
        beta = np.where(rho[c] > 0, rn / np.where(rho[c] > 0, rho[c], 1.0), 0.0)
        row = np.full(k, np.nan)
        row[c] = rn
        hist.append(row)
        for j, col in enumerate(c):
            iters[col] = it
            if rn[j] < 0.81 * best[col]:
                best[col], stall[col] = rn[j], 0
            else:
                stall[col] += 1
                if stall_limit > 0 and stall[col] >= stall_limit:
                    active[col] = False
            if not (np.sqrt(rn[j]) > tol[col]) or it >= itmax:
                active[col] = False
        rho[c] = rn
        X[:, c] += alpha.astype(dtype) * P[:, c]
        P[:, c] = Zc + beta.astype(dtype) * P[:, c]
        R[:, c] = Rc
    return X, iters, np.array(hist), tol


def true_relres(A, X, B):
    """||B - A X||_2 / ||B||_2 per column, in float64 (0 for a zero column of B)."""
    A = sp.csr_matrix(A, dtype=np.float64)
    X = np.asarray(X, dtype=np.float64).reshape(A.shape[0], -1)
    B = np.asarray(B, dtype=np.float64).reshape(A.shape[0], -1)
    rn = np.linalg.norm(B - A @ X, axis=0)
    bn = np.linalg.norm(B, axis=0)
    return np.where(bn > 0, rn / np.where(bn > 0, bn, 1.0), 0.0)


def node_currents(A, v, threshold=1e-8, margin=1e-6, dv=0.0):
    """Node currents of voltages v (n,) on the Laplacian A -- src/out.jl:178-207 with the zeroing of
    src/out.jl:281-287: branch currents d_ij = |a_ij| (v_i - v_j) over the stored upper triangle,
    zeroed where |d / max(d)| < threshold, then max(inflow, outflow) per node, where the inflow is
    cut against the largest positive branch current and the outflow against the largest negative one.

    Returns (currents, mask).  mask marks the nodes that have a branch whose |d / max| lies within
    `margin` (relative) of the threshold, widened by the branch's own uncertainty |a_ij| dv when the
    compared implementation evaluates v_i - v_j to within dv: there the two implementations may
    legitimately round to opposite sides of the cut."""
    coo = sp.triu(sp.csr_matrix(A, dtype=np.float64), k=1).tocoo()
    coo = sp.coo_matrix((coo.data[coo.data != 0], (coo.row[coo.data != 0], coo.col[coo.data != 0])),
                        shape=coo.shape)
    n = A.shape[0]
    v = np.asarray(v, dtype=np.float64)
    a = np.abs(coo.data)
    d = a * (v[coo.row] - v[coo.col])
    mask = np.zeros(n, dtype=bool)

    def one(b):
        s = np.zeros(n)
        if not len(b):
            return s
        mx = b.max()
        with np.errstate(divide="ignore", invalid="ignore"):
            ratio = np.abs(b / mx)
            b = np.where(ratio < threshold, 0.0, b)
            near = np.abs(ratio - threshold) <= threshold * margin + a * dv / abs(mx)
        mask[coo.row[near]] = True
        mask[coo.col[near]] = True
        np.add.at(s, coo.col, np.maximum(b, 0.0))
        np.add.at(s, coo.row, np.maximum(-b, 0.0))
        return s

    p, q = one(d), one(-d)
    return np.where(p > q, p, q), mask


def stencil_wraps(A):
    """The stencil-form rule of the device (setup_device.cu build_dia) evaluated on the host:
    (nr, entries off the 9 raster diagonals, wrapped entries).  nr = row 0's smallest column
    above 1 (0 when there is no candidate); a wrapped entry sits on a diagonal but its row offset
    dr leaves the raster column, (i mod nr) + dr outside [0, nr)."""
    A = sp.csr_matrix(A)
    n = A.shape[0]
    c0 = A.indices[A.indptr[0]:A.indptr[1]]
    cand = c0[c0 > 1]
    if n < 16 or not len(cand) or cand.min() < 3 or cand.min() >= n:
        return 0, None, None
    nr = int(cand.min())
    coo = A.tocoo()
    off = coo.col.astype(np.int64) - coo.row
    dc = np.where(np.abs(off) <= 1, 0, np.sign(off))
    dr = off - dc * nr
    on = (np.abs(dr) <= 1) & ((np.abs(off) <= 1) | (np.abs(np.abs(off) - nr) <= 1))
    r = coo.row % nr + dr
    wrapped = on & ((r < 0) | (r >= nr))
    return nr, int((~on).sum()), int(wrapped.sum())

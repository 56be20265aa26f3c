"""Float64 references of the operations the CUDA kernels implement, in plain numpy / scipy.

    vcycle(levels, r)             the Jacobi-smoothed V(1,1) cycle the device runs as its preconditioner
    pcg(A, B, precond, rtol, itmax)
                                  the device's PCG recurrence, column by column: deferred x update, stop
                                  test, stall guard and per-column freezing (csrc/kernels.cuh
                                  cg_after_precond, k_cg_*)
    true_relres(A, X, B)          ||B - A X|| / ||B|| per column (the reference's residual gate,
                                  src/core.jl:640-650)
    node_currents(A, v)           per-node currents with the 1e-8 relative zeroing (src/out.jl:178-290)
    advanced_window(g, src, gnd, four, rtol, itmax)
                                  one moving window of the batched advanced-mode kernel
                                  (csrc/advanced_batch.cu): labels, skip rule, reduced systems, Jacobi-PCG,
                                  residual gate, status and node currents
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


def pcg(A, B, precond, rtol, itmax, atol=ATOL, stall_limit=40, dtype=np.float64, iterates=None):
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
    device.  The device's AMG path uses stall_limit = 40, its Jacobi path 2000; 0 switches the guard off.
    `iterates`: a list that receives a copy of X after every iteration.

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
        if iterates is not None:
            iterates.append(X.copy())
    return X, iters, np.array(hist), tol


def true_relres(A, X, B):
    """||B - A X||_2 / ||B||_2 per column, in float64 (0 for a zero column of B)."""
    A = sp.csr_matrix(A, dtype=np.float64)
    X = np.asarray(X, dtype=np.float64).reshape(A.shape[0], -1)
    B = np.asarray(B, dtype=np.float64).reshape(A.shape[0], -1)
    rn = np.linalg.norm(B - A @ X, axis=0)
    bn = np.linalg.norm(B, axis=0)
    return np.where(bn > 0, rn / np.where(bn > 0, bn, 1.0), 0.0)


def node_currents(A, v, threshold=1e-8, margin=1e-6, dv=0.0, finitegrounds=None):
    """Node currents of voltages v (n,) on the Laplacian A -- src/out.jl:178-207 with the zeroing of
    src/out.jl:281-287: branch currents d_ij = |a_ij| (v_i - v_j) over the stored upper triangle,
    zeroed where |d / max(d)| < threshold, then max(inflow, outflow) per node, where the inflow is
    cut against the largest positive branch current and the outflow against the largest negative one.

    `finitegrounds` (n,): the current finitegrounds * v to ground joins the inflow where it is negative
    and the outflow where it is positive, uncut (src/out.jl:193-202).

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
    if finitegrounds is not None:
        fg = np.asarray(finitegrounds, dtype=np.float64) * v
        p = p + np.where(fg < 0, -fg, 0.0)
        q = q + np.where(fg > 0, fg, 0.0)
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


# ---- one moving window of the batched advanced-mode kernel (csrc/advanced_batch.cu) ----------------
NODATA = -9999.0
GATE = 1e-4                                   # src/core.jl:641
WIN_OK, WIN_MAXITER, WIN_RESIDUAL = 0, 1, 2   # a window reports the worst of its components


def window_graph(g, four):
    """Edge weights of a conductance window as a symmetric CSR matrix over its cells (cell r + c nrows,
    column-major): (g_i + g_j) / 2 between valid 4-neighbours, divided by sqrt(2) on the diagonals of
    the 8-neighbour stencil.  A cell is a node when g > 0 (NODATA, 0 and NaN are not).  Returns (W, valid)."""
    g = np.asarray(g, dtype=np.float64)
    nr, nc = g.shape
    with np.errstate(invalid="ignore"):
        valid = g > 0
    idx = np.arange(nr * nc).reshape(nc, nr).T
    rows, cols, vals = [], [], []
    for dr, dc in ((1, 0), (0, 1)) + (() if four else ((1, 1), (-1, 1))):
        ra, rb = slice(max(0, -dr), nr - max(0, dr)), slice(max(0, dr), nr + min(0, dr))
        ca, cb = slice(0, nc - dc), slice(dc, nc)
        ok = valid[ra, ca] & valid[rb, cb]
        w = (g[ra, ca] + g[rb, cb]) / (2.0 * np.sqrt(2.0) if dr and dc else 2.0)
        rows.append(idx[ra, ca][ok])
        cols.append(idx[rb, cb][ok])
        vals.append(w[ok])
    i, j, w = np.concatenate(rows), np.concatenate(cols), np.concatenate(vals)
    W = sp.coo_matrix((np.concatenate([w, w]), (np.concatenate([i, j]), np.concatenate([j, i]))),
                      shape=(nr * nc, nr * nc)).tocsr()
    return W, valid.T.ravel()


def advanced_window(g, src, gnd, four, rtol, itmax, atol=ATOL, iterates=False):
    """One window of compute_omniscape_current as the batched kernel solves it, in float64
    (src/raster/advanced.jl:119-149, 184-221, 274-305; src/out.jl:178-207):

      * nodes are the cells with g > 0, components those of the 4- or 8-neighbour grid, labelled by
        their smallest column-major cell r + c nrows and visited in that order;
      * policy rmvsrc: a source on a grounded cell is dropped; a component is solved unless its sources
        or its grounds sum to exactly 0;
      * the reduced system deletes the Inf-ground cells (held at 0 V) and carries the finite grounds on
        the diagonal unless the finite ground of the component's first cell is -9999;
      * Jacobi-PCG from x = 0 (`pcg` with D^-1 and no stall guard: the kernel has neither that guard nor
        the p.Ap <= 0 one, which a positive definite system never takes, and updates x in place, which
        is the same arithmetic), then the true relative residual of the reduced system against the
        1e-4 gate; RESIDUAL outranks MAXITER (itmax reached with sqrt(rho) still above tol);
      * node currents of the component's own Laplacian and voltages, cut at 1e-8 of the component's
        own maxima, plus the finite-ground currents.

    g, src, gnd: 2-D rasters (float32 values are widened).  Returns a dict: labels (nrows, ncols; -1 =
    not a node), solved (roots, ascending), comps (per solved component: root, cells, keep, A_red, a_local,
    fin, b, x, x_hist when `iterates`, iters, rho, tol, relres, status), volt, cur, mask (rasters),
    iters (sum), relres (max), status, and fail = (root, relres, iters) of the first component with the
    window's status (None when OK)."""
    g, src, gnd = (np.asarray(a, dtype=np.float64) for a in (g, src, gnd))
    nr, nc = g.shape
    n = nr * nc
    flat = lambda a: a.T.ravel()
    unflat = lambda a: a.reshape(nc, nr).T
    W, valid = window_graph(g, four)
    _, comp = sp.csgraph.connected_components(W, directed=False)
    root_of = np.full(comp.max() + 1, n)
    np.minimum.at(root_of, comp, np.arange(n))
    labels = np.where(valid, root_of[comp], -1)

    s0, gr0 = flat(src), flat(gnd)
    s = np.where((s0 != 0) & (gr0 != 0), 0.0, s0)                    # rmvsrc
    gr = np.where(np.isinf(gr0) & (s > 0), 0.0, gr0)
    fin = np.where(np.isfinite(gr0), gr0, 0.0)
    L = (sp.diags(np.asarray(W.sum(axis=1)).ravel()) - W).tocsr()

    volt, cur, mask = np.zeros(n), np.zeros(n), np.zeros(n, dtype=bool)
    out = dict(labels=unflat(labels), solved=[], comps=[], iters=0, relres=0.0, status=WIN_OK, fail=None)
    order = np.argsort(labels, kind="stable")
    order = order[labels[order] >= 0]
    starts = np.nonzero(np.diff(labels[order], prepend=-1))[0]
    for cells in np.split(order, starts[1:]) if len(order) else []:
        root = int(cells[0])
        with np.errstate(invalid="ignore"):
            if s[cells].sum() == 0 or gr[cells].sum() == 0:
                continue
        use_fin = fin[root] != NODATA
        f_local = fin[cells] if use_fin else None
        a_local = L[cells][:, cells].tocsr()
        sel = gr0[cells] != np.inf
        keep = cells[sel]
        A_red = a_local + sp.diags(f_local) if use_fin else a_local
        A_red = A_red.tocsr()[sel][:, sel].tocsr()
        b = s[keep]
        d = A_red.diagonal()
        hist = [] if iterates else None
        X, it, rho, tol = pcg(A_red, b, lambda R: R / d[:, None], rtol, itmax, atol=atol, stall_limit=0,
                              iterates=hist)
        x, it, rho, tol = X[:, 0], int(it[0]), rho[:, 0], float(tol[0])
        relres = float(true_relres(A_red, x, b)[0])
        status = WIN_RESIDUAL if not relres < GATE else \
            WIN_MAXITER if it >= itmax and np.sqrt(rho[-1]) > tol else WIN_OK
        v = np.zeros(len(cells))
        v[sel] = x
        c, m = node_currents(a_local, v, finitegrounds=f_local)
        volt[cells], cur[cells], mask[cells] = v, c, m
        comp_out = dict(root=root, cells=cells, keep=keep, A_red=A_red, a_local=a_local, fin=f_local, b=b, x=x,
                        iters=it, rho=rho, tol=tol, relres=relres, status=status)
        if iterates:
            comp_out["x_hist"] = [h[:, 0] for h in hist]
        out["solved"].append(root)
        out["comps"].append(comp_out)
        out["iters"] += it
        out["relres"] = max(out["relres"], relres)
        if status > out["status"]:
            out["status"], out["fail"] = status, (root, relres, it)
    out.update(volt=unflat(volt), cur=unflat(cur), mask=unflat(mask))
    return out

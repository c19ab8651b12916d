"""Float64 restatement of ``libreco/algorithms/_als.pyx`` (``als_update``): the CG and direct per-row solves with
the reference's early exits and LAPACK's ``info``, for checking the float32 Cython goldens and the GPU kernels.

The exits compare float64 residuals against the same absolute 1e-10, so a case whose residual sits near 1e-10
can exit on one side and not the other; :func:`als_update` returns the residuals it tested for that check."""
import numpy as np


def base_matrix(Y, reg, implicit):
    Y = np.asarray(Y, dtype=np.float64)
    d = Y.shape[1]
    reg32 = float(np.float32(reg))
    return (Y.T @ Y if implicit else np.zeros((d, d))) + reg32 * np.eye(d)


def _row(csr, m):
    s = slice(csr.indptr[m], csr.indptr[m + 1])
    return np.asarray(csr.indices[s]), np.asarray(csr.data[s], dtype=np.float64)


def cholesky_info(A):
    """(L, info): LAPACK spotrf's test, pivot <= 0 or NaN at column j -> info = j + 1."""
    d = A.shape[0]
    L = np.array(A, dtype=np.float64)
    for j in range(d):
        piv = L[j, j] - L[j, :j] @ L[j, :j]
        if not piv > 0:
            return None, j + 1
        L[j, j] = np.sqrt(piv)
        L[j + 1:, j] = (L[j + 1:, j] - L[j + 1:, :j] @ L[j, :j]) / L[j, j]
    return np.tril(L), 0


def als_update(csr, X, Y, reg, task, use_cg=True, cg_steps=3):
    """Returns (X_new float64, residuals): residuals lists every r.r the CG exits compared with 1e-10.
    Raises ValueError with the reference's text on a direct-path failure (smallest failing row)."""
    implicit = task == "ranking"
    Y64 = np.asarray(Y, dtype=np.float64)
    X64 = np.array(X, dtype=np.float64)
    A0 = base_matrix(Y, reg, implicit)
    tested = []
    for m in range(X64.shape[0]):
        idx, val = _row(csr, m)
        Yr = Y64[idx]
        if use_cg:
            x = X64[m].copy()
            if implicit:
                r = -A0 @ x + Yr.T @ (val - (val - 1) * (Yr @ x))
            else:
                r = -A0 @ x + Yr.T @ (val - Yr @ x)
            p = r.copy()
            rsold = r @ r
            tested.append(rsold)
            if rsold < 1e-10:
                continue
            w = (val - 1) if implicit else np.ones_like(val)
            for _ in range(cg_steps):
                Ap = A0 @ p + Yr.T @ (w * (Yr @ p))
                ak = rsold / (p @ Ap)
                x = x + ak * p
                r = r - ak * Ap
                rsnew = r @ r
                tested.append(rsnew)
                if rsnew < 1e-10:
                    break
                p = r + (rsnew / rsold) * p
                rsold = rsnew
            X64[m] = x
        else:
            w = (val - 1) if implicit else np.ones_like(val)
            A = A0 + (Yr * w[:, None]).T @ Yr
            b = Yr.T @ val
            L, info = cholesky_info(A)
            if info:
                raise ValueError(f"cython_lapack.posv failed (err={info}) on row {m}. "
                                 "Try increasing the regularization parameter.")
            X64[m] = np.linalg.solve(L.T, np.linalg.solve(L, b))
    return X64, np.asarray(tested)


def fit(csr_raw, task, use_cg, U0, I0, reg=5.0, alpha=10, n_epochs=2, cg_steps=3):
    """``ALS.fit``'s loop (``als.py:146-168``) on :func:`als_update` in float64 from float32 initial tables;
    returns (U, I) with the mean row appended."""
    import scipy.sparse as sp

    users = sp.csr_matrix(csr_raw, dtype=np.float64, copy=True)
    items = users.T.tocsr()
    if task == "ranking":
        users.data = users.data * alpha + 1
        items.data = items.data * alpha + 1
    U, I = np.asarray(U0, dtype=np.float64), np.asarray(I0, dtype=np.float64)
    for _ in range(n_epochs):
        U, _ = als_update(users, U, I, reg, task, use_cg, cg_steps)
        I, _ = als_update(items, I, U, reg, task, use_cg, cg_steps)
    return np.vstack([U, U.mean(0)]), np.vstack([I, I.mean(0)])

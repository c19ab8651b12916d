"""Swing oracles (``libreco/algorithms/swing.py`` on recfarm ``rust/src/graph.rs``, ``swing.rs``, ``inference.rs``).

* :func:`matrix_scores`: float64 ``S = M^T diag(coef) M`` with a zero diagonal, where row p of the sparse M is the
  common-item indicator of user pair p = (u < v) with ``|C| >= 2`` and ``coef_p = w_u w_v / (alpha + |C| - 1)``.  It
  never loops over target items, so it is independent of the per-target loop it checks.
* :func:`literal_scores`: ``compute_single_swing`` restated loop for loop (fp32 by default), for tiny graphs.
* :func:`topk_lists`, :func:`recommend`, :func:`predict`: the per-item lists and the serving of ``swing.rs``.

R is a scipy CSR (users x items, sorted rows); its stored entries are the interactions, explicit zeros included.
"""
import numpy as np
import scipy.sparse as sp


def _pattern(R):
    R = sp.csr_matrix(R)
    return sp.csr_matrix((np.ones(R.nnz), R.indices, R.indptr), shape=R.shape)


def matrix_scores(R, alpha, chunk=1 << 18):
    """float64 [n_items, n_items] sparse swing scores."""
    B = _pattern(R)
    n_items = B.shape[1]
    w = 1.0 / np.sqrt(np.maximum(np.diff(B.indptr), 1).astype(np.float64))
    G = sp.triu(B @ B.T, k=1).tocoo()
    keep = G.data >= 2
    us, vs, c = G.row[keep], G.col[keep], G.data[keep]
    S = sp.csr_matrix((n_items, n_items))
    for a in range(0, len(us), chunk):
        u, v, cc = us[a:a + chunk], vs[a:a + chunk], c[a:a + chunk]
        M = B[u].multiply(B[v]).tocsr()
        coef = w[u] * w[v] / (float(alpha) + cc - 1.0)
        S = S + (M.T @ sp.diags(coef) @ M).tocsr()
    S = S.tolil()
    S.setdiag(0)
    S = S.tocsr()
    S.eliminate_zeros()
    return S


def literal_scores(R, alpha, dtype=np.float32):
    """Dense [n_items, n_items] scores by graph.rs's loop: per target i, pairs u < v of its users, intersection C,
    term ``w_u * w_v * (alpha + k).recip()`` in ``dtype``, added to every j in C other than i."""
    R = sp.csr_matrix(R)
    RT = R.T.tocsr()
    n_items = R.shape[1]
    one = dtype(1)
    w = one / np.sqrt(np.diff(R.indptr).astype(dtype))
    rows = [R.indices[R.indptr[u]:R.indptr[u + 1]] for u in range(R.shape[0])]
    S = np.zeros((n_items, n_items), dtype=dtype)
    for i in range(n_items):
        users = RT.indices[RT.indptr[i]:RT.indptr[i + 1]]
        for a, u in enumerate(users):
            for v in users[a + 1:]:
                C = np.intersect1d(rows[u], rows[v], assume_unique=True)
                if len(C) < 2:
                    continue
                term = w[u] * w[v] * (one / (dtype(alpha) + dtype(len(C) - 1)))
                for j in C:
                    if j != i:
                        S[i, j] += term
    return S


def topk_lists(S, top_k):
    """Per item: (ids, scores) of its first top_k nonzero scores by (score desc, id asc), and the nonzero count."""
    S = sp.csr_matrix(S)
    out, count = [], np.zeros(S.shape[0], dtype=np.int64)
    for i in range(S.shape[0]):
        ids = S.indices[S.indptr[i]:S.indptr[i + 1]]
        vals = S.data[S.indptr[i]:S.indptr[i + 1]]
        nz = vals != 0
        ids, vals = ids[nz], vals[nz]
        order = np.lexsort((ids, -vals))[:top_k]
        out.append((ids[order].astype(np.int64), vals[order].astype(np.float64)))
        count[i] = len(ids)
    return out, count


def user_scores(R, lists, top_k, user_consumed, u, filter_consumed):
    """{item: score} of swing.rs:203-220 for user u (float64 sums of ``score * label``)."""
    R = sp.csr_matrix(R)
    if u < 0 or u >= R.shape[0]:
        return {}
    consumed = set(user_consumed.get(u, [])) if filter_consumed else set()
    scores = {}
    for e in range(R.indptr[u], R.indptr[u + 1]):
        i, label = R.indices[e], float(R.data[e])
        if i >= len(lists):
            continue
        ids, vals = lists[i]
        for j, s in zip(ids[:top_k], vals[:top_k]):
            if int(j) in consumed:
                continue
            scores[int(j)] = scores.get(int(j), 0.0) + float(s) * label
    return scores


def recommend(R, lists, top_k, user_consumed, users, n_rec, filter_consumed):
    """(recs, additional counts, per-user score dicts): each user's candidates by (score desc, id asc)."""
    recs, extra, dicts = [], [], []
    for u in users:
        sc = user_scores(R, lists, top_k, user_consumed, int(u), filter_consumed)
        ranked = sorted(sc, key=lambda j: (-sc[j], j))[:n_rec]
        recs.append(ranked)
        extra.append(n_rec - len(ranked))
        dicts.append(sc)
    return recs, extra, dicts


def predict(R, lists, top_k, n_users, n_items, users, items, default_pred=0.0):
    """swing.rs:153-185 with compute_pred "ranking": the mean score of item i's first top_k neighbours in row u."""
    R = sp.csr_matrix(R)
    out = []
    for u, i in zip(users, items):
        u, i = int(u), int(i)
        if not (0 <= u < n_users and 0 <= i < n_items) or u >= R.shape[0]:
            out.append(default_pred)
            continue
        row = set(R.indices[R.indptr[u]:R.indptr[u + 1]].tolist())
        ids, vals = lists[i]
        hits = [float(s) for j, s in zip(ids[:top_k], vals[:top_k]) if int(j) in row]
        out.append(float(np.mean(hits)) if hits else default_pred)
    return out

"""UserCF / ItemCF oracles (``libreco/bases/cf_base_rs.py`` on recfarm ``rust/src/similarities.rs``, ``item_cf.rs``,
``user_cf.rs``, ``inference.rs``).

* :func:`matrix_sims`: float64 ``prod = M M^T`` and ``count = B B^T`` (B the binary pattern of the sim-side matrix M),
  ``sq`` the diagonal of ``prod``, then the cosine with compute_cosine's zero rule and the ``min_common`` mask, off the
  diagonal.  It never loops over target rows, so it is independent of the per-target loop it checks.
* :func:`literal_sims`: ``forward_cosine`` restated loop for loop (fp32 by default), for tiny graphs.
* :func:`topk_lists`, :func:`recommend`, :func:`predict`: the per-row lists and the serving of both engines.

The sim side is ``R^T`` (items) for ItemCF and ``R`` (users) for UserCF; R is a scipy CSR (users x items, sorted
rows) whose stored entries are the interactions, explicit zeros included.  A result "pairs" is ``(x1, x2, cosine)``
arrays of every kept ordered pair.
"""
import numpy as np
import scipy.sparse as sp


def sim_side(R, user_based):
    R = sp.csr_matrix(R)
    return R if user_based else R.T.tocsr()


def matrix_sims(M, min_common):
    """Kept ordered pairs (x1, x2, cosine) in float64, sorted by (x1, x2)."""
    M = sp.csr_matrix(M, dtype=np.float64)
    B = sp.csr_matrix((np.ones(M.nnz), M.indices, M.indptr), shape=M.shape)
    count = (B @ B.T).tocoo()
    prod = (M @ M.T).tocsr()
    sq = np.asarray(M.multiply(M).sum(axis=1)).ravel()
    keep = (count.data >= min_common) & (count.row != count.col)
    x1, x2 = count.row[keep].astype(np.int64), count.col[keep].astype(np.int64)
    p = np.asarray(prod[x1, x2]).ravel() if len(x1) else np.zeros(0)
    cos = np.zeros(len(x1))
    nz = (p != 0) & (sq[x1] != 0) & (sq[x2] != 0)
    cos[nz] = p[nz] / (np.sqrt(sq[x1[nz]]) * np.sqrt(sq[x2[nz]]))
    order = np.lexsort((x2, x1))
    return x1[order], x2[order], cos[order]


def literal_sims(M, min_common, dtype=np.float32):
    """forward_cosine (similarities.rs:13-152): sum squares and the merge walk of every x1 < x2, in ``dtype``; both
    orientations of each kept pair."""
    M = sp.csr_matrix(M)
    n_x = M.shape[0]
    rows = [(M.indices[M.indptr[x]:M.indptr[x + 1]], M.data[M.indptr[x]:M.indptr[x + 1]].astype(dtype))
            for x in range(n_x)]
    sq = []
    for _, d in rows:
        ss = dtype(0)
        for v in d:
            ss = dtype(ss + v * v)
        sq.append(ss)
    out = []
    for x1 in range(n_x):
        for x2 in range(x1 + 1, n_x):
            (a, da), (b, db) = rows[x1], rows[x2]
            i = j = 0
            prod, count = dtype(0), 0
            while i < len(a) and j < len(b):
                if a[i] < b[j]:
                    i += 1
                elif a[i] > b[j]:
                    j += 1
                else:
                    prod = dtype(prod + da[i] * db[j])
                    count += 1
                    i += 1
                    j += 1
            if count >= min_common:
                if prod == 0 or sq[x1] == 0 or sq[x2] == 0:
                    c = dtype(0)
                else:
                    c = dtype(prod / dtype(np.sqrt(sq[x1]) * np.sqrt(sq[x2])))
                out += [(x1, x2, c), (x2, x1, c)]
    out.sort(key=lambda t: (t[0], t[1]))
    x1 = np.array([t[0] for t in out], np.int64)
    x2 = np.array([t[1] for t in out], np.int64)
    return x1, x2, np.array([t[2] for t in out], dtype)


def topk_lists(pairs, n_x, k_sim):
    """Per row: (ids, cosines) of its first k_sim kept entries by (cosine desc, id asc), and its kept count."""
    x1, x2, cos = pairs
    out, count = [], np.bincount(x1, minlength=n_x).astype(np.int64)
    starts = np.concatenate([[0], np.cumsum(count)])
    for x in range(n_x):
        ids, vals = x2[starts[x]:starts[x + 1]], np.asarray(cos[starts[x]:starts[x + 1]], np.float64)
        order = np.lexsort((ids, -vals))[:k_sim]
        out.append((ids[order].astype(np.int64), vals[order]))
    return out, count


def _row(C, r):
    return C.indices[C.indptr[r]:C.indptr[r + 1]], C.data[C.indptr[r]:C.indptr[r + 1]].astype(np.float64)


def user_scores(R, lists, k_sim, user_consumed, u, filter_consumed, user_based):
    """{item: score} of item_cf.rs:156-209 / user_cf.rs:151-205 for user u (float64 sums of ``sim * label``)."""
    R = sp.csr_matrix(R)
    if u < 0 or u >= R.shape[0]:
        return {}
    consumed = set(user_consumed.get(u, [])) if filter_consumed else set()
    scores = {}

    def add(j, v):
        if int(j) not in consumed:
            scores[int(j)] = scores.get(int(j), 0.0) + v

    if user_based:
        ids, sims = lists[u]
        for v, s in zip(ids[:k_sim], sims[:k_sim]):
            for i, label in zip(*_row(R, int(v))):
                add(i, float(s) * label)
    else:
        for i, label in zip(*_row(R, u)):
            ids, sims = lists[i]
            for j, s in zip(ids[:k_sim], sims[:k_sim]):
                add(j, float(s) * label)
    return scores


def recommend(R, lists, k_sim, user_consumed, users, n_rec, filter_consumed, user_based):
    """(recs, no_rec_indices, per-user score dicts): each user's candidates by (score desc, id asc)."""
    recs, no_rec, dicts = [], [], []
    for k, u in enumerate(users):
        sc = user_scores(R, lists, k_sim, user_consumed, int(u), filter_consumed, user_based)
        recs.append(sorted(sc, key=lambda j: (-sc[j], j))[:n_rec])
        if not sc:
            no_rec.append(k)
        dicts.append(sc)
    return recs, no_rec, dicts


def compute_pred(task, sims, labels, dtype=np.float64):
    """inference.rs:48-71 in ``dtype``, terms in the given order."""
    sims, labels = np.asarray(sims, dtype), np.asarray(labels, dtype)
    with np.errstate(divide="ignore", invalid="ignore"):
        total = dtype(0)
        for s in sims:
            total = dtype(total + s)
        if task == "ranking":
            return dtype(total / dtype(len(sims)))
        out = dtype(0)
        for s, lab in zip(sims, labels):
            out = dtype(out + dtype(lab * s) / total)
        return out


def predict(R, lists, k_sim, task, users, items, default_pred, user_based, dtype=np.float64):
    """item_cf.rs:361-396 / user_cf.rs:814-849: the query's first k_sim neighbours intersected with the other CSR's
    row, in neighbour order (cosine desc, the order recfarm's heap pops them); default_pred for an id outside range or
    an empty intersection."""
    R = sp.csr_matrix(R)
    n_users, n_items = R.shape
    other = R.T.tocsr() if user_based else R
    out = []
    for u, i in zip(users, items):
        u, i = int(u), int(i)
        if not (0 <= u < n_users and 0 <= i < n_items):
            out.append(default_pred)
            continue
        q, r = (u, i) if user_based else (i, u)
        idx, lab = _row(other, r)
        labels = dict(zip(idx.tolist(), lab.tolist()))
        ids, sims = lists[q]
        hit = [(float(s), labels[int(j)]) for j, s in zip(ids[:k_sim], sims[:k_sim]) if int(j) in labels]
        out.append(float(compute_pred(task, [h[0] for h in hit], [h[1] for h in hit], dtype)) if hit
                   else default_pred)
    return out

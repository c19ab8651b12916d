"""Float64 restatement of ``libreco/algorithms/_bpr.pyx`` (``bpr_update``) and of the two negative streams, for
checking the float32 Cython goldens and the GPU kernel.

* :func:`update`: the Cython's per-sample update for sgd / momentum / adam (``_bpr.pyx:116-399``), given the
  negatives, in float64 and in the Cython's order (all three gradients from the values before the sample).
* :func:`reference_negatives`: the Cython's own negatives when it is compiled without OpenMP.  ``prange`` is then a
  plain loop, sample ``i`` draws from generator ``t = i % num_threads``, which is ``std::mt19937((seed + 11 t) % 7)``
  through libstdc++'s ``uniform_int_distribution<long>(0, n_items - 1)``: Lemire's multiply-and-reject on one 32-bit
  output per try, redrawn while the item is in the user's CSR row.  ``numpy.random.RandomState(s)``'s MT19937 is
  ``std::mt19937(s)``.
* :func:`device_negatives`: the device sampler of ``csrc/bpr.cu`` bit for bit: one Philox4x32-10 draw keyed by
  (seed, epoch, sample index), ``r = bounded(., n_items - c_u)``, and the r-th item not in the row.
* :func:`ranking_metrics`: recall@k and ndcg@k of embedding tables on held-out pairs, consumed items excluded.
"""
import numpy as np

from oracle.sampling import philox4x32_10

OPTIMIZERS = ("sgd", "momentum", "adam")
STATE_NAMES = {"sgd": (), "momentum": ("u_velocity", "i_velocity"),
               "adam": ("u_1st_mom", "i_1st_mom", "u_2nd_mom", "i_2nd_mom")}


def update(optimizer, users, items, negs, U, I, lr, reg, epoch, states=None, momentum=0.9, rho1=0.9, rho2=0.999):
    """One ``bpr_update`` epoch in float64 on copies; returns (U, I, states dict)."""
    U, I = np.array(U, dtype=np.float64), np.array(I, dtype=np.float64)
    st = {k: np.array(v, dtype=np.float64) for k, v in (states or {}).items()}
    e = U.shape[1] - 1
    if optimizer == "adam":
        c1, c2 = 1.0 - rho1 ** epoch, 1.0 - rho2 ** epoch
    for u, p, n in zip(np.asarray(users).tolist(), np.asarray(items).tolist(), np.asarray(negs).tolist()):
        uu, pp, nn = U[u].copy(), I[p].copy(), I[n].copy()
        g = 1.0 / (1.0 + np.exp(uu @ (pp - nn)))
        gu = g * (pp[:e] - nn[:e]) - reg * uu[:e]
        gp = g * uu - reg * pp
        gn = -g * uu - reg * nn
        if optimizer == "sgd":
            gp[e], gn[e] = g - reg * pp[e], -g - reg * nn[e]
            U[u, :e] += lr * gu
            I[p] += lr * gp
            I[n] += lr * gn
        elif optimizer == "momentum":
            vu, vi = st["u_velocity"], st["i_velocity"]
            vu[u, :e] = momentum * vu[u, :e] + lr * gu
            U[u, :e] += vu[u, :e]
            vi[p] = momentum * vi[p] + lr * gp
            I[p] += vi[p]
            vi[n] = momentum * vi[n] + lr * gn
            I[n] += vi[n]
        else:
            for W, M, H, r, cols, grad in ((U, st["u_1st_mom"], st["u_2nd_mom"], u, slice(0, e), gu),
                                           (I, st["i_1st_mom"], st["i_2nd_mom"], p, slice(None), gp),
                                           (I, st["i_1st_mom"], st["i_2nd_mom"], n, slice(None), gn)):
                M[r, cols] = rho1 * M[r, cols] + (1.0 - rho1) * grad
                H[r, cols] = rho2 * H[r, cols] + (1.0 - rho2) * grad ** 2
                W[r, cols] += lr * (M[r, cols] / c1) / (np.sqrt(H[r, cols] / c2) + 1e-8)
    return U, I, st


class _MT:
    """One ``std::mt19937(seed)`` with libstdc++'s ``uniform_int_distribution`` on [0, n)."""

    def __init__(self, seed):
        self.bits = np.random.RandomState(seed & 0xFFFFFFFF)._bit_generator
        self.buf, self.pos = [], 0

    def raw(self):
        if self.pos == len(self.buf):
            self.buf, self.pos = self.bits.random_raw(4096).tolist(), 0
        self.pos += 1
        return self.buf[self.pos - 1]

    def below(self, n):
        prod = self.raw() * n
        low = prod & 0xFFFFFFFF
        if low < n:
            threshold = (1 << 32) % n
            while low < threshold:
                prod = self.raw() * n
                low = prod & 0xFFFFFFFF
        return prod >> 32


def _c_mod(a, m):
    """C's ``%`` (truncating) on integers."""
    r = abs(a) % m
    return r if a >= 0 else -r


def reference_negatives(users, indptr, indices, n_items, seed, num_threads=1):
    """The serial Cython build's negatives for one ``bpr_update`` call (int64 [n])."""
    gens = [_MT(_c_mod(seed + 11 * t, 7)) for t in range(num_threads)]
    rows = {}
    out = np.empty(len(users), dtype=np.int64)
    for i, u in enumerate(np.asarray(users).tolist()):
        if u not in rows:
            rows[u] = set(np.asarray(indices[indptr[u]:indptr[u + 1]]).tolist())
        gen, cons = gens[i % num_threads], rows[u]
        n = gen.below(n_items)
        while n in cons:
            n = gen.below(n_items)
        out[i] = n
    return out


def device_draws(n, seed, epoch, m):
    """bounded(Philox4x32-10((s, 0, epoch) under (seed, epoch)), m) for s < n; m int64 [n] (the range per sample)."""
    s = np.arange(n, dtype=np.uint64)
    seed, epoch = int(seed) & 0xFFFFFFFFFFFFFFFF, int(epoch) & 0xFFFFFFFFFFFFFFFF
    k0, k1 = seed & 0xFFFFFFFF, ((seed >> 32) ^ (epoch >> 32)) & 0xFFFFFFFF
    r0, r1, _, _ = philox4x32_10((s & np.uint64(0xFFFFFFFF)).astype(np.uint32), (s >> np.uint64(32)).astype(np.uint32),
                                 np.zeros(n, np.uint32), np.full(n, epoch & 0xFFFFFFFF, np.uint32), k0, k1)
    m = np.asarray(m, dtype=np.uint64)
    # high 64 bits of ((r0 << 32) | r1) * m for m < 2^32: (r0 m + (r1 m >> 32)) >> 32, exact in uint64
    hi = r0.astype(np.uint64) * m + ((r1.astype(np.uint64) * m) >> np.uint64(32))
    return (hi >> np.uint64(32)).astype(np.int64)


def device_negatives(users, indptr, indices, n_items, seed, epoch):
    """``csrc/bpr.cu``'s negatives (int64 [n]; -1 for a user whose row holds every item)."""
    users = np.asarray(users, dtype=np.int64)
    indptr = np.asarray(indptr, dtype=np.int64)
    deg = indptr[users + 1] - indptr[users]
    m = n_items - deg
    r = device_draws(len(users), seed, epoch, np.maximum(m, 1))
    out = np.empty(len(users), dtype=np.int64)
    for i, u in enumerate(users.tolist()):
        if m[i] <= 0:
            out[i] = -1
            continue
        row = np.asarray(indices[indptr[u]:indptr[u + 1]], dtype=np.int64)
        out[i] = r[i] + np.searchsorted(row - np.arange(row.size), r[i], side="right")
    return out


def ranking_metrics(U, I, train_indptr, train_indices, eval_users, eval_items, k=10):
    """(recall@k, ndcg@k) averaged over the users with held-out items: scores U[u] . I over every item, the user's
    training items removed, top k by score (ties to the lower id)."""
    U, I = np.asarray(U, dtype=np.float64), np.asarray(I, dtype=np.float64)
    eval_users, eval_items = np.asarray(eval_users), np.asarray(eval_items)
    order = np.argsort(eval_users, kind="stable")
    eu, ei = eval_users[order], eval_items[order]
    users, starts = np.unique(eu, return_index=True)
    ends = np.r_[starts[1:], eu.size]
    scores = U[users] @ I.T
    for r, u in enumerate(users.tolist()):
        scores[r, train_indices[train_indptr[u]:train_indptr[u + 1]]] = -np.inf
    top = np.argsort(-scores, axis=1, kind="stable")[:, :k]
    disc = 1.0 / np.log2(np.arange(2, k + 2))
    recall, ndcg = [], []
    for r in range(users.size):
        rel = set(ei[starts[r]:ends[r]].tolist())
        hit = np.array([t in rel for t in top[r].tolist()], dtype=np.float64)
        recall.append(hit.sum() / len(rel))
        ndcg.append((hit * disc).sum() / disc[:min(len(rel), k)].sum())
    return float(np.mean(recall)), float(np.mean(ndcg))

"""Serial restatement of the skip-gram semantics of ``csrc/skipgram.cu`` / ``librecommender_b200.skipgram``
(DESIGN.md §4, "Skip-gram training"), for checking the kernels and the host tables.

* The streams: Philox4x32-10 (``oracle.sampling.philox4x32_10``) keyed by (seed, pass, position) with the stream tag
  in counter word 2 — keep decisions per raw token, reduced windows per kept slot, negatives per (slot, context
  offset, draw), walk steps per (walk, step).
* Host tables written independently of the library: the Huffman tree (heapq over (count, index)), gensim's
  cumulative negative table, the keep probability.
* :func:`train`: one or more epochs in a chosen dtype (float64 is the oracle), serial, in the kernel's order.
* :func:`ranking_metrics` is ``_bpr_oracle``'s.
"""
import heapq

import numpy as np

from _bpr_oracle import ranking_metrics  # noqa: F401  (re-exported for the skip-gram tests)
from oracle.sampling import philox4x32_10

TAG_KEEP, TAG_WINDOW, TAG_NEG, TAG_WALK = 0, 1, 2, 3
MAX_EXP = 6.0


def draws(pos, tag, sub, seed, pass_):
    """(r0, r1) uint32 arrays of the draws at positions ``pos`` (array) with sub-index ``sub`` (array or scalar)."""
    pos = np.asarray(pos, dtype=np.uint64)
    sub = np.asarray(sub, dtype=np.uint64)
    c2 = ((np.uint64(tag) << np.uint64(28)) | sub).astype(np.uint32)
    k0 = seed & 0xFFFFFFFF
    k1 = ((seed >> 32) ^ (pass_ >> 32)) & 0xFFFFFFFF
    r0, r1, _, _ = philox4x32_10((pos & np.uint64(0xFFFFFFFF)).astype(np.uint32), (pos >> np.uint64(32)).astype(np.uint32),
                                 c2, np.uint32(pass_ & 0xFFFFFFFF), k0, k1)
    return r0, r1


def bounded(r0, r1, n):
    """High 64 bits of ((r0 << 32) | r1) * n for 0 < n < 2^32, vectorised."""
    a, b, n = np.asarray(r0, np.uint64), np.asarray(r1, np.uint64), np.asarray(n, np.uint64)
    return ((a * n + ((b * n) >> np.uint64(32))) >> np.uint64(32)).astype(np.int64)


def keep_decisions(tokens, keep_thr, seed, pass_):
    r0, _ = draws(np.arange(len(tokens)), TAG_KEEP, 0, seed, pass_)
    return r0.astype(np.uint64) < np.asarray(keep_thr, np.uint64)[np.asarray(tokens)]


def compact(indptr, tokens, keep):
    """Per sentence: (slot of its first kept token = indptr[s], kept item ids)."""
    out = []
    for s in range(len(indptr) - 1):
        b, e = int(indptr[s]), int(indptr[s + 1])
        out.append((b, np.asarray(tokens[b:e])[keep[b:e]]))
    return out


def reduced_windows(slots, window, seed, pass_):
    r0, r1 = draws(slots, TAG_WINDOW, 0, seed, pass_)
    return bounded(r0, r1, window)


def negative_draws(slot, offsets, window, negative, cum, vocab_items, seed, pass_):
    """[len(offsets), negative] item ids drawn for one centre slot."""
    offsets = np.asarray(offsets, dtype=np.int64)
    sub = ((offsets[:, None] + window) << 4) | np.arange(negative)[None, :]
    r0, r1 = draws(np.full(sub.shape, slot), TAG_NEG, sub, seed, pass_)
    r = bounded(r0, r1, int(cum[-1]))
    idx = np.searchsorted(np.asarray(cum, np.int64), r, side="left")
    return np.asarray(vocab_items)[idx]


def walks(g_indptr, g_dst, n_items, n_walks, walk_length, seed, pass_):
    """List of walks (lists of item ids), walk w = round * n_items + start item."""
    out = []
    for w in range(n_walks * n_items):
        cur = w % n_items
        walk = [cur]
        while len(walk) < walk_length:
            b, e = int(g_indptr[cur]), int(g_indptr[cur + 1])
            if e == b:
                break
            r0, r1 = draws([w], TAG_WALK, len(walk), seed, pass_)
            cur = int(g_dst[b + int(bounded(r0, r1, e - b)[0])])
            walk.append(cur)
        out.append(walk)
    return out


def huffman_paths(counts):
    """Per vocabulary index: (points, codes) root first; inner node k has index V + k, points are index - V."""
    V = len(counts)
    heap = [(int(c), i) for i, c in enumerate(counts)]
    heapq.heapify(heap)
    children = {}
    for k in range(V - 1):
        _, a = heapq.heappop(heap)
        c2, b = heapq.heappop(heap)
        children[V + k] = (a, b)
        heapq.heappush(heap, (_ + c2, V + k))
    paths = [None] * V
    stack = [(2 * V - 2, [], [])] if V > 1 else []
    while stack:
        node, pts, cds = stack.pop()
        if node < V:
            paths[node] = (pts, cds)
            continue
        a, b = children[node]
        stack.append((a, pts + [node - V], cds + [0]))
        stack.append((b, pts + [node - V], cds + [1]))
    if V == 1:
        paths[0] = ([], [])
    return paths


def cum_table(counts):
    """gensim's make_cum_table in plain Python floats."""
    total = sum(float(c) ** 0.75 for c in counts)
    cum, acc = [], 0.0
    for c in counts:
        acc += float(c) ** 0.75
        cum.append(round(acc / total * (2 ** 31 - 1)))
    return np.array(cum, dtype=np.int64)


def keep_probability(counts, sample=1e-3):
    c = np.asarray(counts, dtype=np.float64)
    t = sample * c.sum()
    return np.minimum(1.0, (np.sqrt(c / t) + 1.0) * t / c)


def vocab_first_appearance(tokens):
    seen, items, counts = {}, [], []
    for t in np.asarray(tokens).tolist():
        if t not in seen:
            seen[t] = len(items)
            items.append(t)
            counts.append(0)
        counts[seen[t]] += 1
    return np.array(items, dtype=np.int64), np.array(counts, dtype=np.int64)


def train(dtype, corpora, syn0, syn1neg, syn1, vocab_items, counts, keep_thr, hs, window, seed, words_total,
          negative=5, alpha0=0.025, min_alpha=1e-4, first_pass=1):
    """Serial epochs in ``dtype`` over ``corpora`` (a list of (indptr, tokens), one per epoch, pass first_pass + e);
    returns copies of (syn0, syn1neg, syn1)."""
    syn0, syn1neg = np.array(syn0, dtype=dtype), np.array(syn1neg, dtype=dtype)
    syn1 = None if syn1 is None else np.array(syn1, dtype=dtype)
    cum = cum_table(counts)
    paths = huffman_paths(counts) if hs else None
    vidx = {int(w): v for v, w in enumerate(np.asarray(vocab_items).tolist())}
    n_epochs = len(corpora)
    one, six = dtype(1), dtype(MAX_EXP)
    for e, (indptr, tokens) in enumerate(corpora):
        pass_ = first_pass + e
        keep = keep_decisions(tokens, keep_thr, seed, pass_)
        for beg, kept in compact(indptr, tokens, keep):
            n = kept.size
            if n == 0:
                continue
            prog = min(1.0, (e * words_total + beg) / (n_epochs * words_total))
            alpha = dtype(alpha0 - (alpha0 - min_alpha) * prog)
            bs = reduced_windows(beg + np.arange(n), window, seed, pass_)
            for i in range(n):
                wi, q, reach = int(kept[i]), beg + i, window - int(bs[i])
                js = [j for j in range(max(0, i - reach), min(n - 1, i + reach) + 1) if j != i]
                if not js:
                    continue
                negs = negative_draws(q, np.array(js) - i, window, negative, cum, vocab_items, seed, pass_)
                for jj, j in enumerate(js):
                    wj = int(kept[j])
                    h = syn0[wj].copy()
                    if hs:
                        work = np.zeros_like(h)
                        pts, cds = paths[vidx[wi]]
                        for p, c in zip(pts, cds):
                            f = h @ syn1[p]
                            if f <= -six or f >= six:
                                continue
                            g = (one - dtype(c) - one / (one + np.exp(-f))) * alpha
                            work += g * syn1[p]
                            syn1[p] += g * h
                        syn0[wj] += work
                        h = syn0[wj].copy()
                    work = np.zeros_like(h)
                    for dd in range(negative + 1):
                        if dd == 0:
                            target, label = wi, one
                        else:
                            target, label = int(negs[jj, dd - 1]), dtype(0)
                            if target == wi:
                                continue
                        f = h @ syn1neg[target]
                        if f <= -six or f >= six:
                            continue
                        g = (label - one / (one + np.exp(-f))) * alpha
                        work += g * syn1neg[target]
                        syn1neg[target] += g * h
                    syn0[wj] += work
    return syn0, syn1neg, syn1

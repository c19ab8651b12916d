"""Skip-gram training on the device: what gensim's ``Word2Vec(sg=1)`` does for the reference's ``Item2Vec`` and
``DeepWalk`` (``libreco/bases/gensim_base.py:65-70``, ``algorithms/item2vec.py:70-83``, ``algorithms/deepwalk.py``),
on the kernels of ``csrc/skipgram.cu``.

* :class:`SkipGramTrainer` is this library's API, shaped like ``BPRTrainer``: a consumed CSR in, ``fit``, device
  ``embeddings()`` that serve through ``recommend_from_embedding``.  The corpus (or DeepWalk's walk graph), the
  tables, the Huffman arrays and the negative table stay on the device across epochs; DeepWalk's walks are drawn on
  the device every epoch.
* :class:`Word2Vec` is the subset of gensim's class that the reference calls.  ``dropin.install(libreco,
  gensim=True)`` binds it in place of gensim's, so the reference's own ``Item2Vec(...).fit`` / ``DeepWalk(...).fit``
  train here with or without gensim installed.
* :func:`pool_users` is ``GensimBase.set_embeddings``'s user loop (``gensim_base.py:96-108``): the mean of the
  consumed item rows, duplicates included, as one CSR SpMM.

The semantics (DESIGN.md §4, "Skip-gram training") follow gensim 4.x as far as it is known without running it:
first-appearance vocabulary, ``default_rng(seed)`` initial vectors, heapq Huffman tree, the unigram^0.75 cumulative
table, ``sample = 1e-3`` downsampling, reduced windows, HS then NS on every pair, |f| >= 6 skipped.  Two differences
are deliberate: the exact logistic replaces gensim's 1000-entry table, and the learning rate steps per sentence,
not per job of about 10 000 words.  Random draws are Philox4x32-10 keyed by (seed, pass, position), not gensim's
streams, so results are not gensim's bit for bit.
"""
from __future__ import annotations

import heapq
import pickle

import numpy as np

from . import _lib

MAX_EMBED = 128
MAX_WINDOW = 4096
MAX_SENTENCE = 10000
ALPHA, MIN_ALPHA, SAMPLE, NEGATIVE, NS_EXPONENT = 0.025, 1e-4, 1e-3, 5, 0.75
DOMAIN = 2 ** 31 - 1
MODES = {"item2vec": 0, "deepwalk": 1}        # the value is hs
GUIDE_BUCKETS = 1 << 16


# ---- host-side vocabulary, tables and trees ------------------------------------------------------------------------
def corpus_csr(sentences):
    """Sentence CSR (indptr int64, tokens int32) of an iterable of item-id sequences, each cut to its first
    ``MAX_SENTENCE`` tokens."""
    seqs = [np.asarray(s, dtype=np.int64)[:MAX_SENTENCE] for s in sentences]
    lens = np.array([s.size for s in seqs], dtype=np.int64)
    indptr = np.zeros(lens.size + 1, dtype=np.int64)
    np.cumsum(lens, out=indptr[1:])
    tokens = np.concatenate(seqs).astype(np.int32) if seqs and indptr[-1] else np.zeros(0, dtype=np.int32)
    return indptr, tokens


def truncate_csr(indptr, tokens):
    """The CSR with every sentence cut to its first ``MAX_SENTENCE`` tokens."""
    indptr, tokens = np.asarray(indptr, dtype=np.int64), np.asarray(tokens)
    lens = np.minimum(np.diff(indptr), MAX_SENTENCE)
    if np.all(lens == np.diff(indptr)):
        return indptr, tokens.astype(np.int32)
    out = np.zeros_like(indptr)
    np.cumsum(lens, out=out[1:])
    pos = np.arange(int(out[-1]), dtype=np.int64) - np.repeat(out[:-1], lens) + np.repeat(indptr[:-1], lens)
    return out, tokens[pos].astype(np.int32)


def vocabulary(tokens):
    """(items int32 [V] in order of first appearance, counts int64 [V]): ``build_vocab`` with ``min_count=1``,
    ``sorted_vocab=0``."""
    tokens = np.asarray(tokens)
    uniq, first, counts = np.unique(tokens, return_index=True, return_counts=True)
    order = np.argsort(first, kind="stable")
    return uniq[order].astype(np.int32), counts[order].astype(np.int64)


def initial_vectors(vocab_items, n_items, d, seed):
    """gensim's ``prep_vectors``: ``(default_rng(seed).random((V, d), float32) * 2 - 1) / d`` in vocabulary order,
    scattered to item-id rows (items outside the vocabulary stay zero)."""
    v = np.random.default_rng(seed).random((len(vocab_items), d), dtype=np.float32)
    v *= np.float32(2.0)
    v -= np.float32(1.0)
    v /= np.float32(d)
    out = np.zeros((n_items, d), dtype=np.float32)
    out[vocab_items] = v
    return out


def huffman(counts):
    """Huffman codes over the vocabulary: pop the two smallest (count, index); the first is the left child (code
    0); inner node k is index V + k.  Returns (ptr int64 [V+1], points int32, codes int8), each path root first;
    points are inner-node rows of syn1 (index - V)."""
    counts = np.asarray(counts, dtype=np.int64)
    V = counts.size
    if V < 2:
        return np.zeros(V + 1, dtype=np.int64), np.zeros(0, dtype=np.int32), np.zeros(0, dtype=np.int8)
    heap = [(int(c), i) for i, c in enumerate(counts.tolist())]
    heapq.heapify(heap)
    parent = np.zeros(2 * V - 1, dtype=np.int64)
    bit = np.zeros(2 * V - 1, dtype=np.int8)
    for k in range(V - 1):
        c1, a = heapq.heappop(heap)
        c2, b = heapq.heappop(heap)
        parent[a], parent[b] = V + k, V + k
        bit[b] = 1
        heapq.heappush(heap, (c1 + c2, V + k))
    root = 2 * V - 2
    # walk every leaf up to the root at once; column t of the stacks is the t-th step above the leaf
    cur = np.arange(V, dtype=np.int64)
    steps_p, steps_c = [], []
    alive = np.ones(V, dtype=bool)
    while alive.any():
        steps_c.append(np.where(alive, bit[cur], -1))
        cur = np.where(alive, parent[cur], cur)
        steps_p.append(np.where(alive, cur - V, -1))
        alive &= cur != root
    P, C = np.stack(steps_p, 1), np.stack(steps_c, 1)
    depth = (C >= 0).sum(1)
    ptr = np.zeros(V + 1, dtype=np.int64)
    np.cumsum(depth, out=ptr[1:])
    # reverse each row's valid prefix: root first
    col = depth[:, None] - 1 - np.arange(P.shape[1])[None, :]
    valid = col >= 0
    rows = np.repeat(np.arange(V), depth)
    cols = col[valid]
    return ptr, P[rows, cols].astype(np.int32), C[rows, cols].astype(np.int8)


def negative_table(counts):
    """gensim's ``make_cum_table``: cum[i] = round(sum_{k<=i} c_k^0.75 / sum c^0.75 * (2^31 - 1)), uint32."""
    pw = np.asarray(counts, dtype=np.float64) ** NS_EXPONENT
    return np.round(np.cumsum(pw) / pw.sum() * DOMAIN).astype(np.uint32)


def negative_guide(cum, buckets=GUIDE_BUCKETS):
    """guide[k] = bisect_left(cum, k * step), step = ceil(cum[-1] / buckets): the search range of a draw."""
    last = int(cum[-1])
    buckets = max(1, min(int(buckets), last))
    step = -(-last // buckets)
    return np.searchsorted(cum, np.arange(buckets + 1, dtype=np.int64) * step, side="left").astype(np.int32), buckets


def keep_thresholds(vocab_items, counts, n_items, sample=SAMPLE):
    """Per item, round(min(1, p_w) 2^32) with p_w = (sqrt(c_w / t) + 1) t / c_w, t = sample * total raw tokens."""
    c = np.asarray(counts, dtype=np.float64)
    t = sample * c.sum()
    p = (np.sqrt(c / t) + 1.0) * t / c
    thr = np.where(p >= 1.0, 2.0 ** 32, np.round(p * 2.0 ** 32)).astype(np.uint64)
    out = np.zeros(n_items, dtype=np.uint64)
    out[vocab_items] = thr
    return out


def walk_graph(indptr, indices, n_items):
    """DeepWalk's graph (``deepwalk.py:79-84``) as a CSR over items: an edge (items[k], items[k+1]) for every
    consecutive pair of every consumed row, kept with multiplicity, in row order within each source."""
    indptr, indices = np.asarray(indptr, dtype=np.int64), np.asarray(indices, dtype=np.int64)
    n = indices.size
    ok = np.ones(max(n - 1, 0), dtype=bool)
    ends = indptr[1:-1] - 1                      # last entry of every row but the final one
    ok[ends[(ends >= 0) & (ends < n - 1)]] = False
    src, dst = indices[:-1][ok], indices[1:][ok]
    order = np.argsort(src, kind="stable")
    g_indptr = np.zeros(n_items + 1, dtype=np.int64)
    np.cumsum(np.bincount(src, minlength=n_items), out=g_indptr[1:])
    return g_indptr, dst[order].astype(np.int32)


def graph_from_dict(graph, n_items):
    """The CSR of the reference's ``defaultdict(list)`` graph, sources in id order, each list kept verbatim."""
    keys = sorted(k for k in graph if len(graph[k]))
    lens = np.zeros(n_items, dtype=np.int64)
    for k in keys:
        lens[int(k)] = len(graph[k])
    g_indptr = np.zeros(n_items + 1, dtype=np.int64)
    np.cumsum(lens, out=g_indptr[1:])
    dst = (np.concatenate([np.asarray(graph[k], dtype=np.int64) for k in keys]) if keys
           else np.zeros(0, dtype=np.int64))
    if dst.size and (dst.min() < 0 or dst.max() >= n_items):
        raise ValueError(f"graph holds items outside [0, {n_items})")
    return g_indptr, dst.astype(np.int32)


# ---- device launches -----------------------------------------------------------------------------------------------
def _u64(seed):
    return int(seed) & 0xFFFFFFFFFFFFFFFF


def walks(g_indptr, g_dst, n_items, n_walks, walk_length, seed, pass_):
    """Device walks of one pass: (indptr int64 [n_walks n_items + 1], tokens int32)."""
    import torch

    dev = g_indptr.device
    total = int(n_walks) * int(n_items)
    L = min(int(walk_length), MAX_SENTENCE)
    lens = torch.empty(total, dtype=torch.int64, device=dev)
    _lib.check(_lib.lib.b200_item_walks(_lib.ptr(g_indptr), _lib.ptr(g_dst), int(n_items), int(n_walks), L,
                                        _u64(seed), int(pass_), _lib.ptr(lens), None, None, _lib.current_stream()))
    indptr = torch.zeros(total + 1, dtype=torch.int64, device=dev)
    torch.cumsum(lens, 0, out=indptr[1:])
    tokens = torch.empty(max(int(indptr[-1]), 1), dtype=torch.int32, device=dev)
    _lib.check(_lib.lib.b200_item_walks(_lib.ptr(g_indptr), _lib.ptr(g_dst), int(n_items), int(n_walks), L,
                                        _u64(seed), int(pass_), None, _lib.ptr(indptr), _lib.ptr(tokens),
                                        _lib.current_stream()))
    return indptr, tokens[:int(indptr[-1])]


def subsample(indptr, tokens, n_items, keep_thr, seed, pass_, record=False):
    """Keep decisions and in-place compaction of one pass: (kept_tokens, kept_sent, kept_len[, keep uint8])."""
    import torch

    dev = indptr.device
    T, S = int(tokens.numel()), int(indptr.numel()) - 1
    kept = torch.empty(max(T, 1), dtype=torch.int32, device=dev)
    sent = torch.empty(max(T, 1), dtype=torch.int32, device=dev)
    klen = torch.empty(max(S, 1), dtype=torch.int32, device=dev)
    keep = torch.empty(max(T, 1), dtype=torch.uint8, device=dev) if record else None
    _lib.check(_lib.lib.b200_skipgram_subsample(
        _lib.ptr(indptr), _lib.ptr(tokens), S, int(n_items), _lib.ptr(keep_thr), _u64(seed), int(pass_),
        _lib.ptr(kept), _lib.ptr(sent), _lib.ptr(klen), _lib.ptr(keep), _lib.current_stream()))
    return (kept, sent, klen) + ((keep[:T],) if record else ())


class Tables:
    """The per-vocabulary device arrays an epoch reads: negative table and guide, and for HS the Huffman paths
    scattered to item ids."""

    def __init__(self, vocab_items, counts, n_items, hs, device):
        import torch

        self.vocab_items = np.asarray(vocab_items, dtype=np.int32)
        self.counts = np.asarray(counts, dtype=np.int64)
        self.V = int(self.vocab_items.size)
        cum = negative_table(self.counts)
        guide, self.buckets = negative_guide(cum)
        self.cum_last = int(cum[-1])
        t = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=device)  # noqa: E731
        self.neg_cum, self.neg_items, self.neg_guide = t(cum), t(self.vocab_items), t(guide)
        self.keep_thr = t(keep_thresholds(self.vocab_items, self.counts, n_items))
        self.hs = int(hs)
        self.hs_ptr = self.hs_points = self.hs_codes = None
        if hs:
            ptr, points, codes = huffman(self.counts)
            lens = np.zeros(n_items, dtype=np.int64)
            lens[self.vocab_items] = np.diff(ptr)
            item_ptr = np.zeros(n_items + 1, dtype=np.int64)
            np.cumsum(lens, out=item_ptr[1:])
            # vocabulary row v's path moves to item vocab_items[v]'s slot: gather the paths in item order
            order = np.argsort(self.vocab_items, kind="stable")
            plen = np.diff(ptr)[order]
            src = np.repeat(ptr[:-1][order], plen) + np.arange(int(plen.sum())) - np.repeat(np.cumsum(plen) - plen, plen)
            self.hs_ptr, self.hs_points, self.hs_codes = t(item_ptr), t(points[src]), t(codes[src])


def epoch(indptr, kept, sent, klen, n_items, syn0, syn1neg, syn1, tables, window, alpha0, min_alpha, words_before,
          words_total, seed, pass_, negative=NEGATIVE, max_inflight=0, record=False):
    """One epoch over a compacted corpus; with ``record`` returns (window_out, neg_out) as device tensors."""
    import torch

    dev = indptr.device
    T, S = int(kept.numel()), int(indptr.numel()) - 1
    T = int(indptr[-1]) if S else 0
    wout = nout = None
    if record:
        wout = torch.full((max(T, 1),), -1, dtype=torch.int32, device=dev)
        nout = torch.full((max(T, 1) * (2 * window + 1) * negative,), -1, dtype=torch.int32, device=dev)
    _lib.check(_lib.lib.b200_skipgram_epoch(
        _lib.ptr(indptr), S, _lib.ptr(kept), _lib.ptr(sent), _lib.ptr(klen), T, int(n_items), _lib.ptr(syn0),
        _lib.ptr(syn1neg), _lib.ptr(syn1), int(syn0.shape[1]), tables.hs, _lib.ptr(tables.hs_ptr),
        _lib.ptr(tables.hs_points), _lib.ptr(tables.hs_codes), _lib.ptr(tables.neg_cum), _lib.ptr(tables.neg_items),
        tables.V, tables.cum_last, _lib.ptr(tables.neg_guide), tables.buckets, int(window), int(negative),
        float(alpha0), float(min_alpha), float(words_before), float(words_total), _u64(seed), int(pass_),
        _lib.ptr(wout), _lib.ptr(nout), int(max_inflight), _lib.current_stream()))
    if record:
        return wout[:T], nout[:T * (2 * window + 1) * negative].view(T, 2 * window + 1, negative)
    return None


def pool_users(indptr, indices, items):
    """Device ``[n_users, d]``: the mean of each user's consumed item rows of ``items``, duplicates included
    (``gensim_base.py:103-106``), as ``b200_spmm_csr`` with values ``1 / len(row)``; an empty row gives zeros."""
    import torch

    from .lightgcn import SpmmGraph

    dev = items.device
    indptr = torch.as_tensor(np.asarray(indptr, dtype=np.int64), device=dev)
    col = torch.as_tensor(np.asarray(indices, dtype=np.int32), device=dev)
    deg = indptr[1:] - indptr[:-1]
    inv = torch.where(deg > 0, 1.0 / deg.clamp(min=1).to(torch.float32), torch.zeros_like(deg, dtype=torch.float32))
    val = torch.repeat_interleave(inv, deg)
    if col.numel() == 0:
        return torch.zeros((deg.numel(), items.shape[1]), dtype=torch.float32, device=dev)
    return SpmmGraph(indptr, col.contiguous(), val.contiguous()).spmm(items.contiguous())


def _check_ids(name, a, n):
    if a.size and (a.min() < 0 or a.max() >= n):
        raise ValueError(f"{name} holds item ids outside [0, {n})")


class SkipGramTrainer:
    """Item2Vec (``mode="item2vec"``: the consumed rows are the sentences, negative sampling) or DeepWalk
    (``mode="deepwalk"``: ``n_walks`` walks of at most ``walk_length`` items from every item over the graph of
    consecutive consumed pairs, hierarchical softmax and negative sampling), trained on the device.

    ``consumed``: a ``ConsumedCSR`` (``consumed.as_csr``), a scipy CSR or ``(indptr, indices)`` with rows in
    consumption order.  ``graph``: optional ``(indptr, dst)`` walk graph that replaces the one built from ``consumed``
    (DeepWalk only).  ``max_inflight``: centres in flight (0: the library default, 1: the serial schedule)."""

    def __init__(self, consumed, n_items, mode="item2vec", embed_size=16, window=5, n_epochs=10, seed=42,
                 norm_embed=False, n_walks=10, walk_length=10, max_inflight=0, graph=None, corpus=None, device=None):
        import torch

        if mode not in MODES:
            raise ValueError(f"mode must be 'item2vec' or 'deepwalk', got {mode!r}")
        if not 1 <= int(embed_size) <= MAX_EMBED:
            raise ValueError(f"embed_size {embed_size} outside [1, {MAX_EMBED}]")
        if not 1 <= int(window) <= MAX_WINDOW:
            raise ValueError(f"window {window} outside [1, {MAX_WINDOW}]")
        if int(n_epochs) < 0 or int(max_inflight) < 0:
            raise ValueError("n_epochs and max_inflight must be >= 0")
        self.n_items, self.mode, self.hs = int(n_items), mode, MODES[mode]
        if self.n_items < 1:
            raise ValueError("n_items must be positive")
        self.d, self.window, self.n_epochs, self.seed = int(embed_size), int(window), int(n_epochs), int(seed)
        self.norm_embed, self.max_inflight = bool(norm_embed), int(max_inflight)
        self.n_walks, self.walk_length = int(n_walks), int(walk_length)
        self.device = torch.device(device) if device is not None else _lib.require_cuda()
        self.consumed = None
        if consumed is not None:
            ind = getattr(consumed, "idx", None)
            indptr, indices = ((consumed.indptr, ind) if ind is not None else
                               (consumed.indptr, consumed.indices) if hasattr(consumed, "indices") else consumed)
            indptr, indices = np.asarray(indptr, dtype=np.int64), np.asarray(indices, dtype=np.int64)
            if indptr.ndim != 1 or indptr.size < 1 or indptr[0] != 0 or np.any(np.diff(indptr) < 0) \
                    or int(indptr[-1]) != indices.size:
                raise ValueError("consumed must be a CSR: indptr from 0, non-decreasing, ending at len(indices)")
            _check_ids("consumed", indices, self.n_items)
            self.consumed = (indptr, indices.astype(np.int32))
        t = lambda a: torch.as_tensor(np.ascontiguousarray(a), device=self.device)  # noqa: E731
        if mode == "deepwalk":
            if self.n_walks < 1 or self.walk_length < 1:
                raise ValueError("n_walks and walk_length must be >= 1")
            if graph is None:
                if self.consumed is None:
                    raise ValueError("deepwalk needs consumed rows or a graph")
                graph = walk_graph(*self.consumed, self.n_items)
            g_indptr, g_dst = (np.asarray(a) for a in graph)
            if g_indptr.shape != (self.n_items + 1,) or int(g_indptr[-1]) != g_dst.size:
                raise ValueError("graph must be a CSR over n_items sources")
            _check_ids("graph", g_dst, self.n_items)
            self.g_indptr, self.g_dst = t(g_indptr.astype(np.int64)), t(np.r_[g_dst, 0].astype(np.int32))
            indptr, tokens = walks(self.g_indptr, self.g_dst, self.n_items, self.n_walks, self.walk_length,
                                   self.seed, 0)
            vocab_tokens = tokens.cpu().numpy()
            self.corpus = None
        else:
            if corpus is None:
                if self.consumed is None:
                    raise ValueError("item2vec needs consumed rows or a corpus")
                corpus = self.consumed
            indptr, tokens = truncate_csr(*corpus)
            _check_ids("corpus", tokens, self.n_items)
            vocab_tokens = tokens
            self.corpus = (t(indptr), t(np.r_[tokens, 0].astype(np.int32))[:tokens.size])
        if vocab_tokens.size == 0:
            raise ValueError("the corpus is empty: no vocabulary to train")
        self.corpus_count = int(indptr.numel() - 1 if hasattr(indptr, "numel") else indptr.size - 1)
        self.words_total = int(vocab_tokens.size)
        vocab_items, counts = vocabulary(vocab_tokens)
        self.tables = Tables(vocab_items, counts, self.n_items, self.hs, self.device)
        self.syn0 = t(initial_vectors(vocab_items, self.n_items, self.d, self.seed))
        self.syn1neg = torch.zeros_like(self.syn0)
        self.syn1 = (torch.zeros((max(self.tables.V - 1, 1), self.d), dtype=torch.float32, device=self.device)
                     if self.hs else None)
        self.passes_done = 0

    def epoch_corpus(self, pass_):
        """The sentence CSR of a pass: the fixed corpus, or DeepWalk's fresh walks."""
        if self.mode == "deepwalk":
            return walks(self.g_indptr, self.g_dst, self.n_items, self.n_walks, self.walk_length, self.seed, pass_)
        return self.corpus

    def epoch(self, index, n_epochs, record=False):
        """Training pass ``index + 1`` of a schedule of ``n_epochs`` (alpha decays over all of them)."""
        pass_ = self.passes_done + 1
        indptr, tokens = self.epoch_corpus(pass_)
        kept, sent, klen = subsample(indptr, tokens, self.n_items, self.tables.keep_thr, self.seed, pass_)
        out = epoch(indptr, kept, sent, klen, self.n_items, self.syn0, self.syn1neg, self.syn1, self.tables,
                    self.window, ALPHA, MIN_ALPHA, index * self.words_total, n_epochs * self.words_total,
                    self.seed, pass_, max_inflight=self.max_inflight, record=record)
        self.passes_done = pass_
        return out

    def fit(self, n_epochs=None):
        """``n_epochs`` passes (default: the constructor's), alpha from 0.025 down to 1e-4 over them."""
        n = self.n_epochs if n_epochs is None else int(n_epochs)
        for e in range(n):
            self.epoch(e, n)
        return self

    def item_vectors(self):
        """Device ``[n_items, d]``: syn0, L2-normalised per row when ``norm_embed``."""
        I = self.syn0.clone()
        if self.norm_embed:
            _lib.check(_lib.lib.b200_l2_normalize_rows(_lib.ptr(I), I.stride(0), I.shape[0], self.d,
                                                       _lib.current_stream()))
        return I

    def embeddings(self):
        """Device ``(U, I)`` with the mean row appended (``assign_embedding_oov``)."""
        import torch

        if self.consumed is None:
            raise ValueError("embeddings() needs the consumed rows")
        I = self.item_vectors()
        U = pool_users(*self.consumed, I)
        return (torch.cat([U, U.mean(0, keepdim=True)]), torch.cat([I, I.mean(0, keepdim=True)]))


# ---- gensim's Word2Vec, the subset the reference calls -----------------------------------------------------------
class _KeyedVectors:
    def __init__(self, vectors):
        self.vectors = vectors

    def get_vector(self, key, norm=False):
        v = self.vectors[int(key)]
        if norm:
            n = np.linalg.norm(v)
            return v / n if n > 0 else v
        return v


class Word2Vec:
    """``gensim.models.Word2Vec`` as ``gensim_base.py``, ``item2vec.py`` and ``deepwalk.py`` use it: skip-gram
    (``sg=1``), ``min_count=1``, ``sorted_vocab=0``; ``hs=0`` is Item2Vec's negative sampling, ``hs=1`` DeepWalk's
    hierarchical softmax plus negative sampling.  ``workers`` is accepted and ignored.  The corpus must be one of
    the reference's two corpus objects: Item2Vec's (``item_seqs``) or DeepWalk's (``graph``, ``n_items``,
    ``n_walks``, ``walk_length``; its walks are drawn on the device and it is never iterated)."""

    def __init__(self, sentences=None, vector_size=100, window=5, sg=0, hs=0, negative=5, seed=1, min_count=5,
                 workers=3, sorted_vocab=1, max_inflight=0, **unsupported):
        if unsupported:
            raise NotImplementedError(f"Word2Vec arguments not supported here: {sorted(unsupported)}")
        if sentences is not None:
            raise NotImplementedError("pass the corpus to build_vocab, as the reference does")
        if sg != 1:
            raise NotImplementedError("only skip-gram (sg=1) is implemented")
        if hs not in (0, 1) or negative != NEGATIVE:
            raise NotImplementedError(f"only hs in (0, 1) with negative={NEGATIVE} is implemented")
        if min_count != 1 or sorted_vocab != 0:
            raise NotImplementedError("only min_count=1, sorted_vocab=0 is implemented")
        del workers
        self.vector_size, self.window, self.sg, self.hs, self.negative = int(vector_size), int(window), 1, hs, negative
        self.seed, self.min_count, self.sorted_vocab, self.max_inflight = int(seed), 1, 0, int(max_inflight)
        self.trainer = None
        self.corpus_count = 0
        self.wv = None

    def _trainer(self, corpus):
        if hasattr(corpus, "item_seqs"):
            if self.hs:
                raise NotImplementedError("Item2Vec's corpus is trained with hs=0")
            indptr, tokens = corpus_csr(corpus.item_seqs)
            n_items = int(tokens.max()) + 1 if tokens.size else 1
            return SkipGramTrainer(None, n_items, "item2vec", self.vector_size, self.window, seed=self.seed,
                                   max_inflight=self.max_inflight, corpus=(indptr, tokens))
        if all(hasattr(corpus, a) for a in ("graph", "n_items", "n_walks", "walk_length")):
            if not self.hs:
                raise NotImplementedError("DeepWalk's corpus is trained with hs=1")
            n_items = int(corpus.n_items)
            return SkipGramTrainer(None, n_items, "deepwalk", self.vector_size, self.window, seed=self.seed,
                                   n_walks=corpus.n_walks, walk_length=corpus.walk_length,
                                   max_inflight=self.max_inflight, graph=graph_from_dict(corpus.graph, n_items))
        raise TypeError(f"unsupported corpus {type(corpus).__name__}: expected the reference's Item2Vec corpus "
                        "(item_seqs) or DeepWalk corpus (graph, n_items, n_walks, walk_length)")

    def build_vocab(self, corpus_iterable, update=False):
        if update:
            raise NotImplementedError("build_vocab(update=True) (retraining a loaded model) is not implemented")
        self.trainer = self._trainer(corpus_iterable)
        self.corpus_count = self.trainer.corpus_count
        self._sync()

    def train(self, corpus_iterable=None, total_examples=None, epochs=None, **_):
        if self.trainer is None:
            raise RuntimeError("call build_vocab before train (a loaded model cannot be trained further)")
        self.trainer.fit(int(epochs))
        self._sync()

    def _sync(self):
        self.wv = _KeyedVectors(self.trainer.syn0.cpu().numpy())

    def save(self, path):
        t = self.trainer
        state = dict(params=dict(vector_size=self.vector_size, window=self.window, hs=self.hs,
                                 negative=self.negative, seed=self.seed, corpus_count=self.corpus_count),
                     syn0=self.wv.vectors if self.wv is not None else None)
        if t is not None:
            state.update(syn1neg=t.syn1neg.cpu().numpy(), syn1=None if t.syn1 is None else t.syn1.cpu().numpy(),
                         vocab_items=t.tables.vocab_items, counts=t.tables.counts)
        with open(path, "wb") as f:
            pickle.dump(state, f, protocol=4)

    @classmethod
    def load(cls, path):
        with open(path, "rb") as f:
            state = pickle.load(f)
        p = state["params"]
        self = cls(vector_size=p["vector_size"], window=p["window"], sg=1, hs=p["hs"], negative=p["negative"],
                   seed=p["seed"], min_count=1, sorted_vocab=0)
        self.corpus_count = p["corpus_count"]
        self.wv = None if state["syn0"] is None else _KeyedVectors(state["syn0"])
        self.arrays = {k: state.get(k) for k in ("syn1neg", "syn1", "vocab_items", "counts")}
        return self


def set_embeddings(model):
    """``GensimBase.set_embeddings`` on the device: item rows from the trained model (normalised when
    ``model.norm_embed``), each user row the mean of the consumed item rows; sets the same numpy attributes."""
    import torch

    from .consumed import as_csr

    dev = _lib.require_cuda()
    vecs = model.gensim_model.wv.vectors
    n = int(model.n_items)
    if vecs.shape[0] < n:
        raise ValueError(f"the trained model holds {vecs.shape[0]} item vectors, the data {n}")
    I = torch.as_tensor(np.ascontiguousarray(vecs[:n], dtype=np.float32), device=dev).clone()
    if model.norm_embed:
        _lib.check(_lib.lib.b200_l2_normalize_rows(_lib.ptr(I), I.stride(0), I.shape[0], I.shape[1],
                                                   _lib.current_stream()))
    csr = as_csr(model.user_consumed, int(model.n_users))
    U = pool_users(csr.indptr, csr.idx, I)
    model.item_embeds_np = I.cpu().numpy()
    model.user_embeds_np = U.cpu().numpy()

"""GPU: YouTubeRetrieval training (librecommender_b200/training.py::YouTubeRetrievalTrainer).

* the unique candidate sampler (``b200_unique_candidates``) against its host restatement
  (``tests/_youtube_retrieval_train_oracle.py``), ids and ``num_tries`` exactly, both kinds;
* one batch (loss and every gradient) against torch float64 autograd given the device's candidates, for both losses
  x ``norm_embed`` x ``use_bn``, with and without user fields: repeated labels, accidental hits, histories built by
  ``b200_interacted_seqs`` (position 0 -> length 1 with the pad id) against the reference's windows (position 0 ->
  empty), S not a multiple of 4;
* several steps, ``step_graph``, ``reg`` and ``lr_decay``, the export into ``feat_models.YouTubeRetrieval`` and the
  ``weights_io`` round trip, the ``ValueError``s, one step at 1 M items."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _youtube_retrieval_train_oracle as yo  # noqa: E402

pytestmark = pytest.mark.gpu

# GPU bounds (calibrated in test_youtube_retrieval_train_cpu.py: a float32 restatement meets each with 4x to spare)
LOSS_REL = 2e-5
GRAD_REL, GRAD_ABS = 3e-4, 6e-6


def make_case(seed, n_users=150, n_items=300, K=8, hidden=(32, 16), use_bn=True, fields=True, B=200, T=5):
    """(spec, weights, consumed, batch) — the batch rows are (user, label = one of the user's consumed items at a
    random position), some labels repeated; ``ref`` windows per the reference (``get_sparse_interacted``)."""
    from librecommender_b200 import synthetic as syn

    rng = np.random.default_rng(seed)
    spec = syn.make_spec(rng, n_users, n_items, [7, 12] if fields else [], [5], 1 if fields else 0, 1)
    emb = syn.make_embeddings(rng, spec, K, linear=False)
    nu = 1 + len(spec["user_sparse_col_index"]) + len(spec["user_dense_col_index"])
    H = hidden[-1]
    w = dict(seq_embeds=syn._glorot(rng, (n_items, K)), item_embeds=syn._glorot(rng, (n_items, H)),
             item_biases=rng.normal(0, 0.1, n_items).astype(np.float32), mlp=syn.make_mlp(rng, nu * K, hidden, use_bn))
    if fields:
        w["sparse_embeds"], w["dense_embeds"] = emb["sparse_embeds"], emb["dense_embeds"]
    consumed = {u: rng.choice(n_items, size=int(rng.integers(1, 3 * T)), replace=False).tolist()
                for u in range(n_users)}
    users = rng.integers(0, n_users, B)
    pos = np.array([rng.integers(0, len(consumed[u])) for u in users])
    pos[:10] = 0                                                    # empty histories
    users[10:15] = users[15:20]                                     # repeated labels
    pos[10:15] = pos[15:20]
    items = np.array([consumed[u][p] for u, p in zip(users, pos)])
    return spec, w, consumed, (users, items)


def reference_windows(consumed, users, items, T, n_items):
    """get_sparse_interacted, mode "recent": the at most T items before the label's first occurrence; position 0 gives
    an empty history (length 0)."""
    seqs = np.full((len(users), T), n_items, dtype=np.int32)
    lens = np.zeros(len(users), dtype=np.int32)
    for r, (u, i) in enumerate(zip(users, items)):
        p = consumed[u].index(i)
        h = consumed[u][max(0, p - T):p]
        seqs[r, :len(h)] = h
        lens[r] = len(h)
    return seqs, lens


def device_batch(consumed, users, items, T, n_items):
    import torch

    from librecommender_b200.collate import DeviceSequenceBuilder
    from librecommender_b200.consumed import ConsumedCSR

    sb = DeviceSequenceBuilder(ConsumedCSR.from_dict(consumed, len(consumed)), T, n_items)
    u, i = torch.as_tensor(users).cuda(), torch.as_tensor(items).cuda()
    seqs, lens = sb(u, i)
    return u, i, seqs, lens


def trainer_name(k, ref):
    if k.startswith("W"):
        return "Wt" + k[1:], ref.T
    return k, ref


def assert_grads(tr, ref_g):
    gmax = max(np.abs(v).max() for v in ref_g.values())
    for k, ref in ref_g.items():
        name, ref_t = trainer_name(k, ref)
        got = tr.grads[name].cpu().numpy().astype(np.float64).reshape(ref_t.shape)
        err = np.abs(got - ref_t).max()
        assert err <= GRAD_REL * np.abs(ref_t).max() + GRAD_ABS * gmax, (k, float(err), float(np.abs(ref_t).max()))


def sampler_call(kind, n_items, S, seed, step):
    import torch

    from librecommender_b200 import _lib

    owner = torch.full((n_items,), -1, dtype=torch.int32, device="cuda")
    out = torch.empty(S, dtype=torch.int64, device="cuda")
    tries = torch.empty(1, dtype=torch.int64, device="cuda")
    step_d = torch.full((1,), step, dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib.b200_unique_candidates(kind, n_items, S, seed, _lib.ptr(step_d), _lib.ptr(owner),
                                               owner.numel() * 4, _lib.ptr(out), _lib.ptr(tries),
                                               _lib.current_stream()))
    return out.cpu().numpy(), int(tries.cpu()[0]), owner


@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("S,n_items", [(1, 1), (1, 1_000_000), (255, 255), (255, 256), (255, 5000),
                                       (8192, 8192), (8192, 20_000), (8192, 1_000_000)])
def test_sampler_matches_host_restatement(kind, S, n_items):
    ref, ref_tries, ambiguous = yo.unique_candidates(kind, n_items, S, 42, 3)
    got, tries, owner = sampler_call(kind, n_items, S, 42, 3)
    if ambiguous:
        pytest.skip(f"{ambiguous} log-uniform draws within 4 ulp of an integer boundary of exp")
    assert tries == ref_tries
    np.testing.assert_array_equal(got, ref)
    assert len(np.unique(got)) == S and got.min() >= 0 and got.max() < n_items
    assert bool((owner == -1).all()), "the workspace is left free"
    if S < n_items:
        nxt, _, _ = sampler_call(kind, n_items, S, 42, 4)
        assert not np.array_equal(nxt, got), "consecutive steps draw the same candidates"


CASES = [("sampled_softmax", False, True, True, 0, 255), ("sampled_softmax", True, False, True, 1, 37),
         ("sampled_softmax", False, False, False, 0, 290), ("sampled_softmax", True, True, False, 1, 128),
         ("nce", False, True, True, 1, 255), ("nce", True, False, True, 0, 37),
         ("nce", False, False, False, 1, 101), ("nce", True, True, False, 0, 290)]


@pytest.mark.parametrize("loss_type,norm,use_bn,fields,kind,S", CASES)
def test_one_batch_matches_float64(loss_type, norm, use_bn, fields, kind, S):
    import torch

    from librecommender_b200.training import YouTubeRetrievalTrainer

    T, n_items = 5, 300
    spec, w, consumed, (users, items) = make_case(7 + S, use_bn=use_bn, fields=fields, T=T, n_items=n_items)
    u, i, seqs, lens = device_batch(consumed, users, items, T, n_items)
    ref_seqs, ref_lens = reference_windows(consumed, users, items, T, n_items)
    ln = lens.cpu().numpy()
    assert (ln[ref_lens == 0] == 1).all() and (ref_lens == 0).sum() >= 10      # position 0: length 1, the pad id
    assert (ref_lens == T).any()                                                # histories longer than T are cut
    tr = YouTubeRetrievalTrainer(spec, w, loss_type, batch_size=len(users), num_sampled_per_batch=S,
                                 sampler="uniform" if kind == 0 else "log_uniform", norm_embed=norm, use_bn=use_bn)
    loss = float(tr.forward_backward(u, i, seqs, lens))
    ids, tries = tr.sampled.cpu().numpy(), int(tr.num_tries.cpu()[0])
    ref_ids, ref_tries, _ = yo.unique_candidates(kind, n_items, S, 42, 0)
    np.testing.assert_array_equal(ids, ref_ids)
    assert tries == ref_tries
    assert np.isin(items, ids).any(), "the batch has accidental hits"
    st = yo.init_state(w, use_bn)
    ref_loss, ref_g, _, _ = yo.forward_backward(st, spec, users, items, ref_seqs, ref_lens, ids, tries, loss_type, kind,
                                               norm)
    assert abs(loss - ref_loss) <= LOSS_REL * max(1.0, abs(ref_loss)), (loss, ref_loss)
    assert_grads(tr, ref_g)
    torch.cuda.synchronize()


@pytest.mark.parametrize("loss_type", ["sampled_softmax", "nce"])
def test_steps_export_and_reload(tmp_path, loss_type):
    import torch

    from librecommender_b200 import weights_io as wio
    from librecommender_b200.feat_models import YouTubeRetrieval, recent_sequences
    from librecommender_b200.training import YouTubeRetrievalTrainer
    from oracle import tf_models as tm

    T, n_items, lr = 5, 300, 1e-2
    spec, w, consumed, (users, items) = make_case(21, T=T, n_items=n_items)
    u, i, seqs, lens = device_batch(consumed, users, items, T, n_items)
    ref_seqs, ref_lens = reference_windows(consumed, users, items, T, n_items)
    tr = YouTubeRetrievalTrainer(spec, w, loss_type, batch_size=len(users), num_sampled_per_batch=64, lr=lr)
    st = yo.init_state(w, True)
    seen = []
    for step in range(3):
        loss = float(tr.step(u, i, seqs, lens))
        ids, tries = tr.sampled.cpu().numpy(), int(tr.num_tries.cpu()[0])
        seen.append(ids.copy())
        ref = yo.train_step(st, spec, users, items, ref_seqs, ref_lens, ids, tries, lr, loss_type=loss_type)
        assert abs(loss - ref) <= 1e-3 * max(1.0, abs(ref)) * (step + 1), (step, loss, ref)
        if step == 0:
            for k, v in st["params"].items():
                name, ref_t = trainer_name(k, v)
                got = tr.params[name].cpu().numpy().astype(np.float64).reshape(ref_t.shape)
                assert np.abs(got - ref_t).max() <= 2e-2 * lr + 1e-6, (k, float(np.abs(got - ref_t).max()))
    assert not np.array_equal(seen[0], seen[1])
    for name, (mm, mv) in tr.moving.items():
        np.testing.assert_allclose(mm.cpu().numpy(), st["moving"][name][0], rtol=1e-3, atol=1e-4)
        np.testing.assert_allclose(mv.cpu().numpy(), st["moving"][name][1], rtol=1e-3, atol=1e-4)
    w2 = tr.export_weights()
    useqs, ulens = recent_sequences(consumed, spec["n_users"], n_items, T)
    model = YouTubeRetrieval(spec, w2, useqs, ulens)
    ids_u = np.arange(spec["n_users"])
    got = model.user_vectors(ids_u).cpu().numpy()
    ref = tm.youtube_retrieval_user_vectors(w2, spec, ids_u, useqs, ulens, False, dtype=np.float64)
    assert np.abs(got - ref).max() <= 3e-5 * max(1.0, np.abs(ref).max())
    np.savez(tmp_path / "m_tf_variables.npz", **wio.youtube_retrieval_tf_variables(w2))
    back = wio.load_reference_tf_model(str(tmp_path), "m", "YouTubeRetrieval", 2, True)
    for k in ("seq_embeds", "item_embeds", "item_biases", "sparse_embeds", "dense_embeds"):
        np.testing.assert_array_equal(back[k], w2[k])
    for a, b in zip(back["mlp"]["kernels"] + back["mlp"]["biases"], w2["mlp"]["kernels"] + w2["mlp"]["biases"]):
        np.testing.assert_array_equal(a, b)
    for j, bn in enumerate([back["mlp"]["bn_in"]] + back["mlp"]["bns"]):
        ref_bn = ([w2["mlp"]["bn_in"]] + w2["mlp"]["bns"])[j]
        for k in ("gamma", "beta", "mean", "var"):
            np.testing.assert_array_equal(bn[k], ref_bn[k])
    torch.cuda.synchronize()


@pytest.mark.parametrize("loss_type", ["sampled_softmax", "nce"])
def test_step_graph_matches_step(loss_type):
    from librecommender_b200.training import YouTubeRetrievalTrainer

    T, n_items = 5, 300
    spec, w, consumed, (users, items) = make_case(33, T=T, n_items=n_items)
    u, i, seqs, lens = device_batch(consumed, users, items, T, n_items)
    a = YouTubeRetrievalTrainer(spec, w, loss_type, batch_size=len(users), num_sampled_per_batch=101, lr=1e-2)
    b = YouTubeRetrievalTrainer(spec, w, loss_type, batch_size=len(users), num_sampled_per_batch=101, lr=1e-2)
    for step in range(3):
        la = float(a.step(u, i, seqs, lens))
        ids_a = a.sampled.cpu().numpy()
        lb = float(b.step_graph(u, i, seqs, lens))
        np.testing.assert_array_equal(b.sampled.cpu().numpy(), ids_a)        # replays draw this step's candidates
        assert abs(la - lb) <= 1e-5 * max(1.0, abs(la)), (step, la, lb)
    assert b.graph_launches_per_step > 0
    for k in a.params:
        x, y = a.params[k].cpu().numpy(), b.params[k].cpu().numpy()
        assert np.abs(x - y).max() <= 1e-5 + 1e-4 * np.abs(x).max(), k


def test_reg_and_lr_decay():
    from librecommender_b200.training import YouTubeRetrievalTrainer, set_regularisation

    T, n_items, lr, reg = 5, 300, 1e-2, 1e-3
    spec, w, consumed, (users, items) = make_case(45, T=T, n_items=n_items, use_bn=False)
    u, i, seqs, lens = device_batch(consumed, users, items, T, n_items)
    ref_seqs, ref_lens = reference_windows(consumed, users, items, T, n_items)
    tr = set_regularisation(YouTubeRetrievalTrainer(spec, w, "nce", batch_size=len(users), num_sampled_per_batch=64,
                                                    use_bn=False, lr=lr), reg, True, 1, 0.5)
    st = yo.init_state(w, False)
    for step in range(2):
        loss = float(tr.step(u, i, seqs, lens))
        ids, tries = tr.sampled.cpu().numpy(), int(tr.num_tries.cpu()[0])
        ref = yo.train_step(st, spec, users, items, ref_seqs, ref_lens, ids, tries, lr, reg=reg, decay_steps=1,
                            decay_rate=0.5, loss_type="nce")
        assert abs(loss - ref) <= 1e-3 * max(1.0, abs(ref)) * (step + 1)
    for k, v in st["params"].items():
        name, ref_t = trainer_name(k, v)
        got = tr.params[name].cpu().numpy().astype(np.float64).reshape(ref_t.shape)
        assert np.abs(got - ref_t).max() <= 4e-2 * lr + 1e-6, (k, float(np.abs(got - ref_t).max()))


def test_value_errors_launch_nothing():
    from librecommender_b200 import _lib
    from librecommender_b200 import synthetic as syn
    from librecommender_b200.training import YouTubeRetrievalTrainer

    spec, w, _, _ = make_case(3, n_items=300)
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match="loss_type"):
        YouTubeRetrievalTrainer(spec, w, "bpr")
    with pytest.raises(ValueError, match="num_sampled"):
        YouTubeRetrievalTrainer(spec, w, batch_size=256, num_sampled_per_batch=301)
    with pytest.raises(ValueError, match="num_sampled"):
        YouTubeRetrievalTrainer(dict(spec, n_items=70_000), w, batch_size=65_537)
    with pytest.raises(ValueError, match="rows"):
        YouTubeRetrievalTrainer(spec, dict(w, item_embeds=w["item_embeds"][:-1]))
    rng = np.random.default_rng(1)
    ms = syn.make_multi_sparse_spec(rng, 150, 300, [7], [5], [("user", 9, 3)])
    with pytest.raises(ValueError, match="combiner"):
        YouTubeRetrievalTrainer(ms, w)
    assert _lib.launch_count() == n0


def test_one_step_at_catalogue_scale():
    import torch

    from librecommender_b200 import synthetic as syn
    from librecommender_b200.training import YouTubeRetrievalTrainer

    rng = np.random.default_rng(9)
    n_users, n_items, K, B, T = 20_000, 1_000_000, 64, 8192, 10
    spec = syn.make_spec(rng, n_users, n_items, [30], [], 1, 0)
    emb = syn.make_embeddings(rng, spec, K, linear=False)
    w = dict(seq_embeds=syn._glorot(rng, (n_items, K)), item_embeds=syn._glorot(rng, (n_items, K)),
             item_biases=np.zeros(n_items, np.float32), sparse_embeds=emb["sparse_embeds"],
             dense_embeds=emb["dense_embeds"], mlp=syn.make_mlp(rng, 3 * K, (128, 64, K), True))
    tr = YouTubeRetrievalTrainer(spec, w, "sampled_softmax", batch_size=B)
    users = torch.as_tensor(rng.integers(0, n_users, B)).cuda()
    items = torch.as_tensor(rng.integers(0, n_items, B)).cuda()
    lens = torch.as_tensor(rng.integers(0, T + 1, B).astype(np.int32)).cuda()
    seqs = torch.as_tensor(rng.integers(0, n_items, (B, T)).astype(np.int32)).cuda()
    seqs = torch.where(torch.arange(T, device="cuda")[None] < lens[:, None], seqs, torch.full_like(seqs, n_items))
    l0 = float(tr.step(users, items, seqs, lens))
    ids0 = tr.sampled.cpu().numpy()
    ref, tries, amb = yo.unique_candidates(0, n_items, B, 42, 0)
    np.testing.assert_array_equal(ids0, ref)
    assert int(tr.num_tries.cpu()[0]) == tries
    l1 = float(tr.step_graph(users, items, seqs, lens))
    assert np.isfinite(l0) and np.isfinite(l1) and l1 < l0 + 1.0
    # with near-zero logits the softmax loss starts at about log(1 + S)
    assert abs(l0 - np.log(1 + B)) < 1.0, l0

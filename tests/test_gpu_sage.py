"""GraphSage / PinSage inference on the device: neighbour ids, weights and lengths bit for bit against the restated
Philox streams of ``tests/_sage_oracle.py`` at every level, a chi-square test of one-walk transitions, the encoder on
the reference's recorded messages against the reference's outputs, ``set_embeddings`` shapes / OOV rows / batching,
serving against the exact fp32 path, C1 recall@10 against the reference's own tables, and the ``sage=True`` drop-in
on the live reference."""
import numpy as np
import pytest
from scipy import stats

import _sage_oracle as orc
from test_sage_cpu import CASES, data_info, feats, golden, message, state_dict

pytestmark = pytest.mark.gpu


def engine(data, kind, paradigm, **kw):
    from librecommender_b200 import sage

    z = golden()
    di = data_info(z, data)
    sd = state_dict(z, f"{data}_{kind}_{paradigm}")
    layers = kw.get("num_layers", 2)              # the goldens have 2 layers: drop the second or repeat it
    for name in ("w_linears", "q_linears"):
        for part in ("weight", "bias"):
            if f"{name}.1.{part}" not in sd:
                continue
            layer1 = sd.pop(f"{name}.1.{part}")
            for layer in range(1, layers):
                sd[f"{name}.{layer}.{part}"] = layer1
    cls = sage.GraphSage if kind == "graphsage" else sage.PinSage
    return cls(di, sd, paradigm=paradigm, **kw), di, sd, z


@pytest.mark.parametrize("kind,layers,nn,walks,wl,p", [
    ("graphsage", 2, 3, 0, 0, 0.5), ("graphsage", 3, 5, 0, 0, 0.5), ("graphsage", 1, 32, 0, 0, 0.5),
    ("pinsage", 2, 3, 10, 2, 0.5), ("pinsage", 3, 4, 8, 4, 0.3), ("pinsage", 1, 32, 64, 4, 0.1),
])
def test_neighbors_match_the_restated_streams_bit_for_bit(kind, layers, nn, walks, wl, p):
    kw = dict(num_layers=layers, num_neighbors=nn, seed=1234567890123)
    if kind == "pinsage":
        kw.update(num_walks=walks, neighbor_walk_len=wl, termination_prob=p)
    eng, di, _, _ = engine("pure", kind, "i2i", **kw)
    n_i = di["n_items"]
    roots = np.unique(np.r_[np.arange(0, n_i, max(1, n_i // (60 if layers < 3 else 12))), n_i - 1])
    g = orc.Graph(di["user_consumed"], di["item_consumed"], di["n_users"], n_i)
    want = orc.sample(kind, g, kw["seed"], roots, layers, nn, walks, wl, p)
    got = eng.neighbors(roots)
    assert len(got) == layers
    for level, (w, h) in enumerate(zip(want, got)):
        if kind == "graphsage":
            np.testing.assert_array_equal(h, w, err_msg=f"level {level}")
        else:
            for a, b, name in zip(h, w, ("ids", "weights", "lens")):
                np.testing.assert_array_equal(a, b, err_msg=f"level {level} {name}")


def test_one_walk_transitions_follow_the_csr_probabilities():
    """One slot, many independent paths of one root: the taken neighbour of item v is n != v with probability
    p(n) (1 - p(v)^11) / (1 - p(v)) and v itself with p(v)^11, p the exact one-walk transition from the CSRs."""
    import torch

    from librecommender_b200 import _lib

    eng, di, _, _ = engine("pure", "graphsage", "i2i", num_neighbors=1)
    uc, ic = di["user_consumed"], di["item_consumed"]
    deg = np.array([len(ic[i]) for i in range(di["n_items"])])
    v = int(np.argsort(deg)[-40])
    p = {}
    for u in ic[v]:
        for n in uc[u]:
            p[n] = p.get(n, 0.0) + 1.0 / len(ic[v]) / len(uc[u])
    pv = p.get(v, 0.0)
    M = 200_000
    roots = torch.tensor([v], dtype=torch.int32, device=eng.device)
    nodes = torch.full((M,), v, dtype=torch.int32, device=eng.device)
    out = torch.empty((M, 1), dtype=torch.int32, device=eng.device)
    _lib.check(_lib.lib.b200_sage_neighbors(*[_lib.ptr(a) for a in eng.graph], _lib.ptr(roots), _lib.ptr(nodes), M, M,
                                            0, 1, 99, _lib.ptr(out), _lib.current_stream()))
    got = out.cpu().numpy().reshape(-1)
    keys = sorted(p)
    expect = np.array([(pv ** 11 if n == v else p[n] * (1 - pv ** 11) / (1 - pv)) for n in keys]) * M
    counts = np.array([(got == n).sum() for n in keys])
    assert counts.sum() == M
    big = expect >= 5                                  # pool the rare neighbours into one cell
    obs = np.r_[counts[big], counts[~big].sum()]
    exp = np.r_[expect[big], expect[~big].sum()]
    keep = exp > 0
    assert stats.chisquare(obs[keep], exp[keep]).pvalue > 1e-4


@pytest.mark.parametrize("data,kind,paradigm", CASES)
def test_encoder_on_recorded_messages_matches_the_reference(data, kind, paradigm):
    """The reference computes in float32 on the CPU; here fp32 SIMT (or 3xTF32, fp32-accurate) dense layers with
    other reduction orders.  Each output goes through at most 5 dense layers of at most (F + 1) d = 64 inputs: the
    rounding of both sides is below 64 * 2^-24 * 5 ~ 2e-5 of the magnitudes involved, so 1e-4 relative to the
    largest output leaves a margin of 5."""
    eng, di, sd, z = engine(data, kind, paradigm)
    case = f"{data}_{kind}_{paradigm}"
    items, nbs, offs, wts = message(z, case, kind)
    got = eng.encode_message(items, nbs, offs, wts).cpu().numpy()
    ref = z[f"{case}_msg_out"]
    tol = 1e-4 * max(1.0, np.abs(ref).max())
    np.testing.assert_allclose(got, ref, rtol=0, atol=tol)
    np.testing.assert_allclose(got, orc.encode(kind, sd, items, nbs, offs, wts, 2, feats(di)), rtol=0, atol=tol)
    if paradigm == "u2i":
        U = eng.user_embeddings().cpu().numpy()
        users = z[f"{case}_users"]
        ref_u = z[f"{case}_user_rows"]
        np.testing.assert_allclose(U[users], ref_u, rtol=0, atol=1e-4 * max(1.0, np.abs(ref_u).max()))


@pytest.mark.parametrize("kind", ["graphsage", "pinsage"])
def test_device_levels_encode_like_their_message(kind):
    """The padded device levels give the same rows as the same neighbours passed in the reference's form."""
    eng, di, _, _ = engine("feat", kind, "i2i")
    roots = np.arange(0, di["n_items"], 13)
    levels = eng.neighbors(roots)
    nbs, offs, wts = orc.padded_to_message(kind, roots, levels)
    a = eng.encode_message(roots, nbs, offs, wts).cpu().numpy()
    import torch

    b = eng._encode_roots(torch.as_tensor(roots.astype(np.int32)).to(eng.device)).cpu().numpy()
    np.testing.assert_allclose(a, b, rtol=0, atol=1e-5 * max(1.0, np.abs(a).max()))


@pytest.mark.parametrize("kind", ["graphsage", "pinsage"])
@pytest.mark.parametrize("paradigm", ["i2i", "u2i"])
def test_set_embeddings_shapes_oov_and_batching(kind, paradigm, monkeypatch):
    from librecommender_b200 import sage

    eng, di, _, _ = engine("feat", kind, paradigm)
    U, I = eng.set_embeddings()
    n_u, n_i, d = di["n_users"], di["n_items"], eng.d
    assert tuple(U.shape) == (n_u + 1, d) and tuple(I.shape) == (n_i + 1, d)
    assert np.isfinite(U.cpu().numpy()).all() and np.isfinite(I.cpu().numpy()).all()
    np.testing.assert_allclose(I[-1].cpu().numpy(), I[:-1].mean(0).cpu().numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(U[-1].cpu().numpy(), U[:-1].mean(0).cpu().numpy(), rtol=1e-5, atol=1e-6)
    if paradigm == "i2i":
        uc = di["user_consumed"]
        Ih = I.cpu().numpy().astype(np.float64)
        want = np.stack([Ih[uc[u]].mean(0) for u in range(n_u)])
        np.testing.assert_allclose(U[:-1].cpu().numpy(), want, rtol=1e-5, atol=1e-6)
    # same seed, other chunking of the roots: the same bits (d = 8: every dense layer on the SIMT kernel)
    monkeypatch.setattr(sage, "ROWS_PER_CHUNK", 97 * eng.num_neighbors ** eng.num_layers)
    again = engine("feat", kind, paradigm)[0].item_embeddings()
    assert torch_equal(again, I[:-1])
    other = engine("feat", kind, paradigm, seed=43)[0].item_embeddings()
    assert not torch_equal(other, I[:-1])


def torch_equal(a, b):
    return bool((a == b).all())


@pytest.mark.parametrize("kind", ["graphsage", "pinsage"])
def test_recommend_user_matches_the_exact_path(kind):
    eng, di, _, _ = engine("pure", kind, "i2i")
    eng.set_embeddings()
    users = np.arange(di["n_users"])
    got = eng.recommend_user(users, 10)
    ref = eng.scorer.recommend(users.tolist(), 10, True, False, path="exact")
    assert (got == ref).mean() > 0.999
    for u in users[:50]:
        assert not set(got[u].tolist()) & set(di["user_consumed"][u])
    U, I = (t.cpu().numpy().astype(np.float64) for t in eng.tables_d)
    pr = eng.predict([0, 1, di["n_users"]], [2, 3, di["n_items"]])
    want = 1 / (1 + np.exp(-np.array([U[0] @ I[2], U[1] @ I[3], U[-1] @ I[-1]])))
    np.testing.assert_allclose(pr, want, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("kind", ["graphsage", "pinsage"])
def test_c1_recall_within_15_percent_of_the_reference(kind):
    """C1 pure i2i, whose golden keeps the whole fitted tables.  After one epoch, recall@10 moves by tens of percent
    with the walks alone (the reference's own set_embeddings under 5 walk seeds; here 5 Philox seeds), so the mean
    recall over 5 seeds must lie within 15 % of the reference's mean, widened by two standard errors of the
    difference of the two means."""
    from _bpr_oracle import ranking_metrics

    z = golden()
    ref = z[f"pure_{kind}_i2i_ref_metrics_walk_seeds"][:, 0]
    got = []
    for seed in range(len(ref)):
        eng, di, _, _ = engine("pure", kind, "i2i", seed=seed)
        U, I = (t.cpu().numpy() for t in eng.set_embeddings())
        n_u, n_i = di["n_users"], di["n_items"]
        got.append(ranking_metrics(U[:n_u], I[:n_i], z["pure_uc_indptr"], z["pure_uc_items"], z["pure_eval_users"],
                                   z["pure_eval_items"])[0])
    got = np.asarray(got)
    se = np.sqrt(got.var(ddof=1) / got.size + ref.var(ddof=1) / ref.size)
    assert abs(got.mean() - ref.mean()) <= 0.15 * ref.mean() + 2 * se, (got, ref)


@pytest.mark.parametrize("kind", ["graphsage", "pinsage"])
def test_dropin_on_the_live_reference(kind):
    import os

    from oracle import make_ref

    if not os.path.isdir(os.path.join(os.path.dirname(make_ref.__file__), "_ref")):
        pytest.skip("oracle/_ref is absent")
    from oracle.ref_loader import load_reference

    load_reference()
    import random

    import pandas as pd
    import torch

    from libreco.algorithms import GraphSage, PinSage
    from libreco.data import DatasetPure, split_by_ratio_chrono
    from oracle.ref_loader import sample_data_path

    from librecommender_b200 import dropin, sage

    df = pd.read_csv(sample_data_path(), sep="::", names=["user", "item", "label", "time"], engine="python")
    train, _ = split_by_ratio_chrono(df, test_size=0.2)
    train_data, di = DatasetPure.build_trainset(train)
    torch.manual_seed(0)
    random.seed(0)
    np.random.seed(0)
    cls = GraphSage if kind == "graphsage" else PinSage
    model = cls("ranking", di, embed_size=8, n_epochs=1, batch_size=2048, device="cpu")
    dropin.install(losses=False, lightgcn=False, sage=True)     # training stays on the reference's CPU path
    try:
        model.fit(train_data, neg_sampling=True, verbose=0)
    finally:
        dropin.uninstall()
    assert model.item_embeds_np.shape == (di.n_items + 1, 8)
    assert model.user_embeds_np.shape == (di.n_users + 1, 8)
    I = sage.engine_for(model).item_embeddings().cpu().numpy()
    np.testing.assert_array_equal(model.item_embeds_np[:-1], I)
    recs = model.recommend_user(1, 10)
    assert len(next(iter(recs.values()))) == 10

"""GPU: SIM training (csrc/sim_train.cu, the dual-sequence collator, training.SIMTrainer) against the float64 step
oracle of tests/_sim_train_oracle.py (parity unpinned, see its header), evaluated on the device's own GSU selection.
Loss and gradients are held to GPU_RTOL of each gradient's largest float64 entry; test_sim_train_cpu.py shows float32
meets that bound with 4x to spare on the same cases."""
import os
import random
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _sim_oracle as so  # noqa: E402
import _sim_train_oracle as sto  # noqa: E402
from test_sim_train_cpu import GPU_RTOL  # noqa: E402

from oracle import tf_models as tm  # noqa: E402

pytestmark = pytest.mark.gpu
G = np.load(os.path.join(os.path.dirname(__file__), "golden", "dual_sequences.npz"))
L_, S_, K_SEL = 24, 6, 6


def _dev(a, dtype=None):
    import torch

    t = torch.as_tensor(np.asarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


# ---- collation ---------------------------------------------------------------------------------------------------
def _golden_csr():
    from librecommender_b200.consumed import ConsumedCSR

    indptr, idx = G["indptr"], G["idx"]
    cons = {u: [int(i) for i in idx[indptr[u]:indptr[u + 1]]] for u in range(len(indptr) - 1)}
    return ConsumedCSR.from_dict(cons, len(cons)), cons


@pytest.mark.parametrize("shape", [tuple(s) for s in G["shapes"]], ids=str)
def test_dual_builder_parity_mode_equals_the_reference(shape):
    from librecommender_b200.collate import DeviceDualSequenceBuilder, interacted_positions_host

    L, S = shape
    csr, cons = _golden_csr()
    random.seed(4321)
    pos = interacted_positions_host(cons, G["users"], G["items"])
    b = DeviceDualSequenceBuilder(csr, L, S, int(G["n_items"]))
    got = b(_dev(G["users"]), _dev(G["items"]), _dev(pos))
    for t, key in zip(got, ("long", "long_lens", "short", "short_lens")):
        np.testing.assert_array_equal(t.cpu().numpy(), G[f"{key}_{L}_{S}"])


def test_dual_builder_fast_mode_windows():
    """Philox positions: the short window ends at the drawn position and the long one right before it, lengths lie
    in their bounds, padding fills the rest; same (seed, step) repeats exactly."""
    import torch

    from librecommender_b200.collate import DeviceDualSequenceBuilder

    csr, cons = _golden_csr()
    L, S, pad = 20, 5, int(G["n_items"])
    users = np.concatenate([G["users"], G["users"]])
    items = np.full(len(users), pad + 7)                  # never consumed: every position is a draw
    b1, b2 = DeviceDualSequenceBuilder(csr, L, S, pad, seed=3), DeviceDualSequenceBuilder(csr, L, S, pad, seed=3)
    out = b1(_dev(users), _dev(items))
    assert all(torch.equal(a, c) for a, c in zip(out, b2(_dev(users), _dev(items))))
    ls, ll, ss, sl = (t.cpu().numpy() for t in out)
    assert ((ll >= 1) & (ll <= L)).all() and ((sl >= 1) & (sl <= S)).all()
    for j, u in enumerate(users):
        c = cons[int(u)]
        # the position the windows imply (item ids never equal the pad id)
        if ss[j, 0] == pad:
            p = 0
        elif sl[j] < S:
            p = int(sl[j])
        elif ls[j, 0] == pad:
            p = S
        elif ll[j] < L:
            p = S + int(ll[j])
        else:
            p = next(q for q in range(L + S, len(c))
                     if c[q - S:q] == list(ss[j]) and c[q - S - L:q - S] == list(ls[j]))
        assert p < len(c)
        ref = sto.dual_windows(cons, [u], [p], pad, L, S)
        for got, want in zip((ls[j], ll[j], ss[j], sl[j]), ref):
            np.testing.assert_array_equal(got, np.asarray(want).reshape(np.shape(got)))


# ---- GSU ------------------------------------------------------------------------------------------------------
def _engine(spec, w, seqs, k=so.TOPK_DEFAULT):
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.feat_models import SIM

    return SIM(spec, wio.sim_weights(w), *seqs, search_topk=k)


@pytest.mark.parametrize("c", so.CASES, ids=so.case_id)
def test_gsu_kernel_selects_what_the_inference_rows_kernel_selects(c):
    import torch

    from librecommender_b200 import _lib

    rng, spec, w, _, seqs = so.make_case(c)
    model = _engine(spec, w, seqs)
    users, items, _, _ = so.case_rows(rng, spec, R=600)
    _, pos = model.attention_rows(users, items)
    u = _dev(users, torch.int64)
    ls, ll = model.long_seqs[u].contiguous(), model.long_lens[u].contiguous()
    R, k, K = len(users), model.topk, model.K
    sel = torch.empty((R, k), dtype=torch.int32, device="cuda")
    pooled = torch.empty((R, K), dtype=torch.float32, device="cuda")
    it = _dev(items, torch.int64)
    _lib.check(_lib.lib.b200_sim_gsu_forward(_lib.ptr(model.Gp), model.Gp.stride(0), K, _lib.ptr(it), _lib.ptr(ls),
                                             ls.stride(0), _lib.ptr(ll), model.L, k, R, _lib.ptr(sel), _lib.ptr(pooled),
                                             K, _lib.current_stream()))
    np.testing.assert_array_equal(sel.cpu().numpy(), pos.cpu().numpy())
    Gp = so.item_table(w, spec, np.float64)
    lsn, lln = seqs[0][users], seqs[1][users]
    scores = so.gsu_scores(Gp, items, lsn, lln)
    margin, sk = so.gsu_margin(scores, lln, k)
    clear = margin > 1e-4 * np.maximum(1.0, sk)
    assert (~clear).mean() < 0.02
    assert (sel.cpu().numpy()[clear] == so.gsu_select(scores, k)[clear]).all()
    inside = np.arange(model.L)[None, :] < np.clip(lln, 0, None)[:, None]
    want = (Gp[lsn] * inside[:, :, None]).sum(1)
    err = np.abs(pooled.cpu().numpy() - want).max()
    assert err <= 1e-5 * max(1.0, np.abs(Gp).max() * model.L), err


# ---- ESU ------------------------------------------------------------------------------------------------------
def _esu_ref(q, ks, vs, valid, H, do):
    """float64 (O, dQ, dK, dV) of the per-head masked attention core."""
    import torch

    R, k, K = ks.shape
    hd = K // H
    t = [torch.tensor(a, dtype=torch.float64, requires_grad=True) for a in (q, ks, vs)]
    qh = t[0].reshape(R, H, hd)
    a = torch.einsum("rhd,rthd->rht", qh, t[1].reshape(R, k, H, hd)) / np.sqrt(hd)
    a = torch.where(torch.as_tensor(valid)[:, None, :], a, torch.full_like(a, -np.inf))
    o = torch.einsum("rht,rthd->rhd", torch.softmax(a, -1), t[2].reshape(R, k, H, hd)).reshape(R, K)
    (o * torch.as_tensor(do)).sum().backward()
    return [o.detach().numpy()] + [x.grad.numpy() for x in t]


@pytest.mark.parametrize("K,H,k", [(8, 1, 1), (8, 2, 32), (16, 4, 10), (24, 2, 7), (32, 1, 32), (48, 4, 17),
                                   (64, 2, 32), (64, 1, 5), (64, 4, 3)])
def test_esu_kernels_against_float64(K, H, k):
    import torch

    from librecommender_b200 import _lib

    rng = np.random.default_rng(K * 100 + H * 10 + k)
    R, L = 300, 64
    q, do = rng.standard_normal((R, K)).astype(np.float32), rng.standard_normal((R, K)).astype(np.float32)
    ks, vs = (rng.standard_normal((R, k, K)).astype(np.float32) for _ in range(2))
    sel = np.sort(np.stack([rng.choice(L, k, replace=False) for _ in range(R)]), axis=1).astype(np.int32)
    lens = rng.integers(1, L + 1, R).astype(np.int32)
    lens[:10] = 1
    sel[~(sel < lens[:, None]).any(1), 0] = 0          # at least one visible key (lens >= 1)
    valid = sel < lens[:, None]
    Q, Ks, Vs, Sel, Ln, dO = (_dev(a) for a in (q, ks.reshape(R * k, K), vs.reshape(R * k, K), sel, lens, do))
    f32 = dict(dtype=torch.float32, device="cuda")

    def run():
        O, P = torch.empty((R, K), **f32), torch.empty(R * H * k, **f32)
        _lib.check(_lib.lib.b200_sim_esu_forward(_lib.ptr(Q), K, _lib.ptr(Ks), _lib.ptr(Vs), K, _lib.ptr(Sel),
                                                 _lib.ptr(Ln), R, K, H, k, _lib.ptr(O), K, _lib.ptr(P), None))
        dQ, dK, dV = torch.empty((R, K), **f32), torch.empty((R * k, K), **f32), torch.empty((R * k, K), **f32)
        _lib.check(_lib.lib.b200_sim_esu_backward(_lib.ptr(Q), K, _lib.ptr(Ks), _lib.ptr(Vs), K, _lib.ptr(Sel),
                                                  _lib.ptr(Ln), R, K, H, k, _lib.ptr(P), _lib.ptr(dO), K, _lib.ptr(dQ),
                                                  K, _lib.ptr(dK), _lib.ptr(dV), K, None))
        return [x.cpu().numpy() for x in (O, dQ, dK.reshape(R, k, K), dV.reshape(R, k, K), P.reshape(R, H, k))]

    got = run()
    ref = _esu_ref(q, ks, vs, valid, H, do)
    for g, r in zip(got[:4], ref):
        assert np.abs(g - r).max() <= 1e-5 * max(1.0, np.abs(r).max()) * np.sqrt(k), np.abs(g - r).max()
    hidden = ~valid
    assert not got[2][hidden].any() and not got[3][hidden].any()
    assert not got[4].transpose(0, 2, 1)[hidden].any()
    again = run()
    assert all(np.array_equal(a, b) for a, b in zip(got, again))


# ---- one step ---------------------------------------------------------------------------------------------------
STEP_CASES = [
    ("ids", 16, 2, True, "keras", 1.0, 1.0, "cross_entropy"),
    ("ids", 16, 2, True, "legacy", 0.3, 0.8, "focal"),
    ("feat", 8, 4, False, "keras", 0.0, 1.0, "cross_entropy"),
    ("feat", 16, 1, True, "legacy", 1.0, 1.0, "focal"),
    ("multi", 16, 2, True, "keras", 0.3, 0.8, "cross_entropy"),
    ("multi", 8, 2, False, "legacy", 0.0, 1.0, "focal"),
]


def _trainer(case, **kw):
    from librecommender_b200.training import SIMTrainer

    layout, K, H, bn, ver, a, b, loss = case
    spec, w, consumed, rows = sto.make_train_case(layout, K, H, bn, ver, L=L_, S=S_, k=K_SEL)
    tr = SIMTrainer(spec, w, search_topk=K_SEL, alpha=a, beta=b, loss_type=loss, use_bn=bn, **kw)
    st = sto.init_state(w, bn, K_SEL, alpha=a, beta=b, loss_type=loss)
    return tr, st, spec, w, rows


def _batch(rows):
    import torch

    users, items, ls, ll, ss, sl, _, _, labels = rows
    return (_dev(users, torch.int64), _dev(items, torch.int64), _dev(ls), _dev(ll), _dev(ss), _dev(sl),
            _dev(labels, torch.float32))


def _raw_grads(tr):
    """The trainer's gradients in the oracle's flat names (through the export layout)."""
    saved = tr.params
    tr.params = tr.grads
    try:
        raw = tr.export_weights()
    finally:
        tr.params = saved
    return sto.init_state(raw, tr.use_bn, tr.topk)["params"]


def _forward_backward(tr, b):
    import torch

    users, items, ls, ll, ss, sl, labels = b
    L, S = ls.shape[1], ss.shape[1]
    tr.forward(users, items, ls, ll.clamp(1, L).contiguous(), ss, sl.clamp(1, S).contiguous())
    sel = tr._cache["sel"].cpu().numpy()
    loss = float(tr.backward(labels))
    torch.cuda.synchronize()
    return loss, sel


@pytest.mark.parametrize("case", STEP_CASES, ids=lambda c: "-".join(map(str, c)))
def test_one_step_loss_and_gradients_match_the_oracle(case):
    tr, st, spec, w, rows = _trainer(case)
    loss, sel = _forward_backward(tr, _batch(rows))
    users, items, ls, ll, ss, sl, sparse, dense, labels = rows
    l64, _, g64, _, sel64, margin, sk = sto.forward_backward(st, spec, users, items, ls, ll, ss, sl, sparse, dense,
                                                             labels, sel=sel)
    clear = margin > 1e-4 * np.maximum(1.0, sk)
    ref_sel = so.gsu_select(so.gsu_scores(so.item_table(w, spec, np.float64), items, ls, np.clip(ll, 1, L_)), K_SEL)
    assert (sel[clear] == ref_sel[clear]).all()
    assert abs(loss - l64) <= GPU_RTOL * abs(l64)
    got = _raw_grads(tr)
    for k, ref in g64.items():
        scale = max(np.abs(ref).max(), 1e-30)
        err = np.abs(got[k] - ref).max()
        assert err <= GPU_RTOL * scale, (k, err, scale)
    if case[5] == 0.0:
        assert not any(got[k].any() for k in got if k.startswith(("fs_", "first_stage_out")))


def test_adam_steps_follow_the_oracle_and_graph_replay_equals_step():
    case = STEP_CASES[1]
    tr, st, spec, _, rows = _trainer(case, lr=1e-2)
    tr_g, _, _, _, _ = _trainer(case, lr=1e-2)
    users, items, ls, ll, ss, sl, sparse, dense, labels = rows
    b = _batch(rows)
    for _ in range(3):
        _, sel = _forward_backward(tr, b)
        tr._adam_update()
        tr._cache = None
        sto.train_step(st, spec, users, items, ls, ll, ss, sl, sparse, dense, labels, 1e-2, sel=sel)
        tr_g.step_graph(*b)
    got = sto.init_state(tr.export_weights(), tr.use_bn, K_SEL)["params"]
    for k, ref in st["params"].items():
        assert np.abs(got[k] - ref).max() <= 1e-3 * max(np.abs(ref).max(), 1e-3), k
    tr2, _, _, _, _ = _trainer(case, lr=1e-2)
    for _ in range(3):
        tr2.step(*b)
    for k in tr2.params:
        np.testing.assert_allclose(tr_g.params[k].cpu().numpy(), tr2.params[k].cpu().numpy(), rtol=1e-5, atol=1e-6)


def test_reg_and_lr_decay_take_effect():
    from librecommender_b200.training import set_regularisation

    case = STEP_CASES[0]
    tr, st, spec, _, rows = _trainer(case)
    set_regularisation(tr, reg=0.05, lr_decay=True, decay_steps=1, decay_rate=0.5)
    users, items, ls, ll, ss, sl, sparse, dense, labels = rows
    b = _batch(rows)
    for _ in range(2):
        _, sel = _forward_backward(tr, b)
        tr._adam_update()
        tr._cache = None
        sto.train_step(st, spec, users, items, ls, ll, ss, sl, sparse, dense, labels, 1e-3, reg=0.05, decay_steps=1,
                       decay_rate=0.5, sel=sel)
    plain, _, _, _, _ = _trainer(case)
    for _ in range(2):
        plain.step(*b)
    for k in ("user_embeds", "item_embeds"):
        got = tr.params[k].cpu().numpy()
        assert np.abs(got - st["params"][k]).max() <= 1e-3 * np.abs(st["params"][k]).max(), k
        assert not np.allclose(got, plain.params[k].cpu().numpy(), rtol=0, atol=1e-7), k


# ---- export ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", [STEP_CASES[0], STEP_CASES[3], STEP_CASES[4]], ids=lambda c: "-".join(map(str, c)))
def test_export_serves_what_the_oracle_computes(case, tmp_path):
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.feat_models import SIM, recent_dual_sequences

    tr, st, spec, w, rows = _trainer(case)
    for _ in range(2):
        tr.step(*_batch(rows))
    raw = tr.export_weights()
    rng = np.random.default_rng(0)
    consumed = so.make_consumed(rng, spec["n_users"], spec["n_items"], L_, S_, K_SEL)
    seqs = recent_dual_sequences(consumed, spec["n_users"], spec["n_items"], L_, S_)
    model = SIM(spec, wio.sim_weights(raw), *seqs, search_topk=K_SEL)
    users, items, _, _ = so.case_rows(rng, spec, R=300)
    _, pos = model.attention_rows(users, items)
    z = model.logits(users, items).cpu().numpy()
    sparse, dense = tm.row_features(spec, users, items)
    raw64 = dict(raw, multi_sparse=None) if case[0] == "multi" else raw
    ref, _, _, _ = so.sim_forward(raw64, spec, users, items, *seqs, K_SEL, sparse, dense, sel=pos.cpu().numpy())
    assert np.abs(z - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())
    tv = wio.sim_tf_variables(raw)
    np.savez(tmp_path / "m_tf_variables.npz", **tv)
    back = wio.load_reference_tf_model(str(tmp_path), "m", "SIM", len(raw["mlp"]["kernels"]), case[3],
                                       num_heads=case[2])
    for k in ("seq_proj", "user_embeds", "item_embeds", "first_stage_out_kernel"):
        np.testing.assert_array_equal(np.asarray(back[k]).reshape(np.shape(raw[k])), raw[k])
    for a, c in zip(back["mlp"]["kernels"] + back["first_stage_mlp"]["kernels"],
                    raw["mlp"]["kernels"] + raw["first_stage_mlp"]["kernels"]):
        np.testing.assert_array_equal(a, c)


# ---- errors -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bad", ["L", "S", "topk", "K", "heads", "mlp", "fs_mlp"])
def test_errors_raise_before_any_launch(bad):
    from librecommender_b200 import _lib
    from librecommender_b200 import synthetic as syn
    from librecommender_b200.training import SIMTrainer

    spec, w, _, rows = sto.make_train_case("ids", 16, 2, True, "keras", L=L_, S=S_, k=K_SEL)
    b = list(_batch(rows))
    n0 = _lib.launch_count()
    rng = np.random.default_rng(3)
    with pytest.raises(ValueError):
        if bad in ("L", "S"):
            tr = SIMTrainer(spec, w, search_topk=K_SEL)
            n0 = _lib.launch_count()
            i = 2 if bad == "L" else 4
            b[i] = b[i].repeat(1, 300 if bad == "L" else 70)
            tr.step(*b)
        elif bad == "topk":
            SIMTrainer(spec, w, search_topk=33)
        elif bad == "K":
            SIMTrainer(spec, syn.make_sim_weights(rng, spec, 72, 2, (8, 4), True, "keras"))
        elif bad == "heads":
            SIMTrainer(spec, dict(w, num_heads=3))
        elif bad == "mlp":
            SIMTrainer(spec, dict(w, mlp=sto.make_train_case("feat", 16, 2, True, "keras")[1]["mlp"]))
        else:
            SIMTrainer(spec, dict(w, first_stage_mlp=w["mlp"]))
    assert _lib.launch_count() == n0

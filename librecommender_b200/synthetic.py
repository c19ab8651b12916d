"""Synthetic feature layouts and glorot-style random weights in the reference's conventions (one shared
sparse table with per-field offsets and an OOV slot per field, unique tables with an extra OOV row;
``libreco/feature/sparse.py:106-119``, ``data/data_info.py:399-413``).  Pure data generators — used by the
tests, by ``bench.py --config ...`` and by the profiling drivers; no model arithmetic lives here."""
from __future__ import annotations

import numpy as np


# ----------------------------------------------------------------------------------------------
def make_spec(rng, n_users, n_items, user_sparse_sizes, item_sparse_sizes, n_user_dense, n_item_dense,
              interleave=True):
    """Feature layout in the reference's convention: one shared sparse table with per-field offsets
    and an OOV slot at the end of each field; unique tables carry an extra OOV row."""
    fs = len(user_sparse_sizes) + len(item_sparse_sizes)
    order = list(rng.permutation(fs)) if interleave else list(range(fs))
    ucol = sorted(order[: len(user_sparse_sizes)])
    icol = sorted(order[len(user_sparse_sizes):])
    sizes = {}
    for j, f in enumerate(ucol):
        sizes[f] = user_sparse_sizes[j]
    for j, f in enumerate(icol):
        sizes[f] = item_sparse_sizes[j]
    offsets, off = {}, 0
    for f in range(fs):
        offsets[f] = off
        off += sizes[f] + 1                       # + OOV slot
    def uniq(n_rows, cols):
        t = np.zeros((n_rows + 1, len(cols)), dtype=np.int32)
        for j, f in enumerate(cols):
            t[:n_rows, j] = offsets[f] + rng.integers(0, sizes[f], size=n_rows)
            t[n_rows, j] = offsets[f] + sizes[f]  # OOV row -> the field's oov index
        return t
    fd = n_user_dense + n_item_dense
    dorder = list(rng.permutation(fd)) if interleave else list(range(fd))
    udc = sorted(dorder[:n_user_dense])
    idc = sorted(dorder[n_user_dense:])
    spec = dict(
        n_users=n_users, n_items=n_items, n_sparse=fs, n_dense=fd, sparse_vocab=off,
        user_sparse_col_index=ucol, item_sparse_col_index=icol,
        user_dense_col_index=udc, item_dense_col_index=idc,
        user_sparse_unique=uniq(n_users, ucol) if ucol else None,
        item_sparse_unique=uniq(n_items, icol) if icol else None,
        user_dense_unique=rng.standard_normal((n_users + 1, len(udc))).astype(np.float32) if udc else None,
        item_dense_unique=rng.standard_normal((n_items + 1, len(idc))).astype(np.float32) if idc else None,
    )
    return spec


def make_multi_sparse_spec(rng, n_users, n_items, user_sparse_sizes, item_sparse_sizes, groups,
                           n_user_dense=1, n_item_dense=1, pad_frac=0.3):
    """Layout with multi-sparse fields in the reference's convention (feature/multi_sparse.py:73-95,
    feature/sparse.py:106-119): plain sparse columns first, then every multi-sparse field's
    sub-columns consecutively; the sub-columns of one field share one vocabulary range and one OOV
    slot (= the padding value of missing sub-features).  `groups` = [(side, vocab, length), ...]."""
    spec = make_spec(rng, n_users, n_items, user_sparse_sizes, item_sparse_sizes, n_user_dense, n_item_dense,
                     interleave=False)
    fs0 = spec["n_sparse"]
    off = spec["sparse_vocab"]
    ucol, icol = list(spec["user_sparse_col_index"]), list(spec["item_sparse_col_index"])
    uu = [spec["user_sparse_unique"]] if ucol else []
    iu = [spec["item_sparse_unique"]] if icol else []
    f_off, f_len, f_oov = [], [], []
    col = fs0
    for side, vocab, ln in groups:
        n_rows = n_users if side == "user" else n_items
        oov = off + vocab
        t = off + rng.integers(0, vocab, size=(n_rows + 1, ln))
        t[rng.random((n_rows + 1, ln)) < pad_frac] = oov          # padded (missing) sub-features
        t[n_rows, :] = oov                                          # OOV row
        t[: min(3, n_rows), :] = oov                                # rows with no feature at all -> div_no_nan
        (uu if side == "user" else iu).append(t.astype(np.int32))
        (ucol if side == "user" else icol).extend(range(col, col + ln))
        f_off.append(col); f_len.append(ln); f_oov.append(oov)
        col += ln
        off += vocab + 1
    spec.update(n_sparse=col, sparse_vocab=off, user_sparse_col_index=ucol, item_sparse_col_index=icol,
                user_sparse_unique=np.concatenate(uu, axis=1) if uu else None,
                item_sparse_unique=np.concatenate(iu, axis=1) if iu else None,
                multi_sparse_combine_info=dict(field_offset=f_off, field_len=f_len, feat_oov=np.array(f_oov)))
    return spec


def _glorot(rng, shape):
    fan_in, fan_out = (shape[0], shape[1]) if len(shape) == 2 else (shape[0], 1)
    lim = np.sqrt(6.0 / (fan_in + fan_out))
    return rng.uniform(-lim, lim, size=shape).astype(np.float32)


def _rand_bn(rng, n):
    return dict(gamma=rng.uniform(0.5, 1.5, n).astype(np.float32), beta=rng.normal(0, 0.1, n).astype(np.float32),
                mean=rng.normal(0, 0.1, n).astype(np.float32), var=rng.uniform(0.5, 1.5, n).astype(np.float32))


def make_mlp(rng, din, hidden, use_bn):
    dims = [din] + list(hidden)
    mlp = dict(kernels=[_glorot(rng, (dims[i], dims[i + 1])) for i in range(len(hidden))],
               biases=[rng.normal(0, 0.05, dims[i + 1]).astype(np.float32) for i in range(len(hidden))])
    if use_bn:
        mlp["bn_in"] = _rand_bn(rng, din)
        mlp["bns"] = [_rand_bn(rng, dims[i + 1]) for i in range(len(hidden) - 1)]
    return mlp


def make_embeddings(rng, spec, K, linear):
    w = dict(user_embeds=_glorot(rng, (spec["n_users"] + 1, K)), item_embeds=_glorot(rng, (spec["n_items"] + 1, K)))
    if spec["n_sparse"]:
        w["sparse_embeds"] = _glorot(rng, (spec["sparse_vocab"], K))
    if spec["n_dense"]:
        w["dense_embeds"] = _glorot(rng, (spec["n_dense"], K))
    if linear:
        w["user_linear"] = _glorot(rng, (spec["n_users"] + 1, 1)).reshape(-1)
        w["item_linear"] = _glorot(rng, (spec["n_items"] + 1, 1)).reshape(-1)
        if spec["n_sparse"]:
            w["sparse_linear"] = rng.uniform(-0.05, 0.05, spec["sparse_vocab"]).astype(np.float32)
        if spec["n_dense"]:
            w["dense_linear"] = rng.uniform(-0.5, 0.5, spec["n_dense"]).astype(np.float32)
    return w


def make_fm_weights(rng, spec, K, use_bn=True):
    w = make_embeddings(rng, spec, K, linear=True)
    F = 2 + spec["n_sparse"] + spec["n_dense"]
    w.update(lin_kernel=_glorot(rng, (F, 1)).reshape(-1), lin_bias=np.float32(0.03),
             pw_kernel=_glorot(rng, (K, 1)).reshape(-1), pw_bias=np.float32(-0.02))
    if use_bn:
        w["fm_bn"] = _rand_bn(rng, K)
    return w


def make_deepfm_weights(rng, spec, K, hidden=(128, 64, 32), use_bn=True):
    w = make_embeddings(rng, spec, K, linear=True)
    F = 2 + spec["n_sparse"] + spec["n_dense"]
    w.update(lin_kernel=_glorot(rng, (F, 1)).reshape(-1), lin_bias=np.float32(0.01),
             mlp=make_mlp(rng, F * K, hidden, use_bn),
             out_kernel=_glorot(rng, (1 + K + hidden[-1], 1)).reshape(-1), out_bias=np.float32(0.05))
    return w


def make_seq_weights(rng, spec, K, hidden=(64, 32), use_bn=True, din=True):
    w = make_embeddings(rng, spec, K, linear=False)
    F = 2 + spec["n_sparse"] + spec["n_dense"]
    if din:
        Kp = K * (1 + len(spec["item_sparse_col_index"]) + len(spec["item_dense_col_index"]))
        w["attention"] = dict(k1=_glorot(rng, (4 * Kp, 16)), b1=rng.normal(0, 0.05, 16).astype(np.float32),
                              k2=_glorot(rng, (16, 1)).reshape(-1), b2=np.float32(0.02))
        din_w = F * K + Kp
    else:
        din_w = (F + 1) * K
    w["mlp"] = make_mlp(rng, din_w, hidden, use_bn)
    w["out_kernel"] = _glorot(rng, (hidden[-1], 1)).reshape(-1)
    w["out_bias"] = np.float32(-0.01)
    return w


def make_two_tower_weights(rng, spec, K, hidden=(64, 32), use_bn=True):
    w = make_embeddings(rng, spec, K, linear=False)
    w["item_embeds"] = w["item_embeds"][: spec["n_items"]]          # two_tower.py:266-271: no OOV row
    nu = 1 + len(spec["user_sparse_col_index"]) + len(spec["user_dense_col_index"])
    ni = 1 + len(spec["item_sparse_col_index"]) + len(spec["item_dense_col_index"])
    w["user_tower"] = make_mlp(rng, nu * K, hidden, use_bn)
    w["item_tower"] = make_mlp(rng, ni * K, hidden, use_bn)
    w["user_dense_cols"] = list(spec["user_dense_col_index"])
    w["item_dense_cols"] = list(spec["item_dense_col_index"])
    return w


def _mha_raw(rng, scheme, d_in, D, H):
    """One ``multi_head_attention`` layer's raw variables of `scheme` (``weights_io._mha_tf_shapes``), each drawn
    glorot over its 2-D view, in the order query, key, value, output."""
    from .weights_io import _mha_2d, _mha_tf_shapes

    raw = _mha_tf_shapes(scheme, d_in, D, H)
    return {n: _glorot(rng, shp).reshape(raw[n]) for n, shp in _mha_2d(scheme, d_in, D).items()}


def make_autoint_weights(rng, spec, K, att_embed_size=(8, 8, 8), num_heads=2, use_residual=True, version="keras",
                         combiner="sqrtn"):
    """AutoInt variables in the raw shapes of the graph TensorFlow `version` builds (layers/attention.py:67-138):
    "keras" (>= 2.10) query / key / value [K, H, hd] and attention_output [H, hd, K]; "legacy" q, k [K, D],
    v [D, D] (applied to the projected keys) and out [D, K].  ``weights_io.autoint_weights`` turns them into
    the engine's dict.  F counts a multi-sparse group as one field unless ``combiner == "normal"``."""
    from .weights_io import autoint_head_dims, autoint_scheme

    scheme = autoint_scheme(version)
    w = make_embeddings(rng, spec, K, linear=False)
    n_sparse = spec["n_sparse"]
    info = spec.get("multi_sparse_combine_info")
    if info is not None and combiner != "normal":
        n_sparse = int(info["field_offset"][0]) + len(info["field_offset"])
    F = 2 + n_sparse + spec["n_dense"]
    H = int(num_heads)
    mha = [_mha_raw(rng, scheme, K, H * hd, H) for hd in autoint_head_dims(att_embed_size)]
    w.update(autoint_scheme=scheme, autoint_mha=mha, num_heads=H, use_residual=bool(use_residual),
             out_kernel=_glorot(rng, (F * K, 1)), out_bias=np.float32(0.02).reshape(1))
    return w


def make_transformer_weights(rng, spec, K, num_heads=1, n_layers=1, max_seq_len=10, hidden=(128, 64, 32), use_bn=True,
                             positional_embedding="trainable", use_causal_mask=False, feat_agg_mode="concat",
                             version="keras", combiner="sqrtn"):
    """Transformer variables (libreco/algorithms/transformer.py:203-339) in the raw shapes of the graph TensorFlow
    `version` builds: "keras" query / key / value [D, H, hd] and attention_output [H, hd, D], "legacy" q, k, v, out
    [D, D] (v applied to the projected keys); FFN [D, 4D], [4D, D]; RMS scales; the trainable positional table
    [T, K] unless `positional_embedding` is sinusoidal.  D = K' + K with K' = K (1 + item sparse columns + item dense
    columns) in concat mode, K in elementwise mode.  ``weights_io.transformer_weights`` turns them into the engine's
    dict.  F counts a multi-sparse group as one field unless ``combiner == "normal"``."""
    from .weights_io import autoint_scheme

    scheme = autoint_scheme(version)
    w = make_embeddings(rng, spec, K, linear=False)
    n_sparse = spec["n_sparse"]
    info = spec.get("multi_sparse_combine_info")
    if info is not None and combiner != "normal":
        n_sparse = int(info["field_offset"][0]) + len(info["field_offset"])
    F = 2 + n_sparse + spec["n_dense"]
    n_is, n_id = len(spec["item_sparse_col_index"]), len(spec["item_dense_col_index"])
    Kp = K * (1 + n_is + n_id) if feat_agg_mode == "concat" else K
    D, H = Kp + K, int(num_heads)
    scale = lambda n: rng.uniform(0.5, 1.5, n).astype(np.float32)      # noqa: E731
    layers = []
    for _ in range(n_layers):
        lw = _mha_raw(rng, scheme, D, D, H)
        lw.update(rms_att=scale(D), rms_ffn=scale(D), ffn1=_glorot(rng, (D, 4 * D)), ffn2=_glorot(rng, (4 * D, D)))
        layers.append(lw)
    w.update(tfm_scheme=scheme, tfm_layers=layers, rms_last=scale(D), rms_item=scale(Kp), num_heads=H,
             use_causal_mask=bool(use_causal_mask), feat_agg_mode=feat_agg_mode,
             mlp=make_mlp(rng, F * K + D, hidden, use_bn), out_kernel=_glorot(rng, (hidden[-1], 1)),
             out_bias=np.float32(0.03).reshape(1))
    if positional_embedding not in ("sinusoidal", "sin", "sinusoid"):
        w["positional_encoding"] = _glorot(rng, (max_seq_len, K))
    if feat_agg_mode == "elementwise":
        for side, n in (("sparse", n_is), ("dense", n_id)):
            if n:
                w[f"ln_{side}"] = dict(scale=scale(K), bias=rng.normal(0, 0.1, K).astype(np.float32))
    return w


def make_sim_weights(rng, spec, K, num_heads=2, hidden=(200, 80), use_bn=True, version="keras", combiner="sqrtn"):
    """SIM variables (libreco/algorithms/sim.py:193-304) in the raw shapes of the graph TensorFlow `version` builds:
    the sequence projection ``seq_proj`` [K', K] with K' = K (1 + item sparse columns + item dense columns), the
    attention over width K ("keras" [K, H, hd] / [H, hd, K], "legacy" [K, K], v applied to the projected keys), the
    first stage (``first_stage_mlp`` on [target, pooled long sequence] and its head) and the second stage ``mlp`` on
    [long_out, short_out, user, item, sparse.., dense..] with its head.  ``weights_io.sim_weights`` turns them into
    the engine's dict.  F counts a multi-sparse group as one field unless ``combiner == "normal"``."""
    from .weights_io import autoint_scheme

    scheme = autoint_scheme(version)
    w = make_embeddings(rng, spec, K, linear=False)
    n_sparse = spec["n_sparse"]
    info = spec.get("multi_sparse_combine_info")
    if info is not None and combiner != "normal":
        n_sparse = int(info["field_offset"][0]) + len(info["field_offset"])
    F = 2 + n_sparse + spec["n_dense"]
    Kp = K * (1 + len(spec["item_sparse_col_index"]) + len(spec["item_dense_col_index"]))
    w.update(sim_scheme=scheme, num_heads=int(num_heads), seq_proj=_glorot(rng, (Kp, K)),
             sim_mha=_mha_raw(rng, scheme, K, K, int(num_heads)),
             first_stage_mlp=make_mlp(rng, 2 * K, hidden, use_bn), first_stage_out_kernel=_glorot(rng, (hidden[-1], 1)),
             first_stage_out_bias=np.float32(0.01).reshape(1), mlp=make_mlp(rng, (F + 2) * K, hidden, use_bn),
             out_kernel=_glorot(rng, (hidden[-1], 1)), out_bias=np.float32(-0.02).reshape(1))
    return w


def make_rnn4rec_weights(rng, n_items, K, hidden_units=(16,), rnn_type="gru", use_layer_norm=False, scheme="keras"):
    """RNN4Rec variables (libreco/algorithms/rnn4rec.py:151-237, layers/recurrent.py:4-63) in the raw shapes of the
    graph `scheme` names: "keras" GRU ``kernel [in, 3H]``, ``recurrent_kernel [H, 3H]``, ``bias [2, 3H]``, keras LSTM
    ``[in, 4H]``, ``[H, 4H]``, ``[4H]`` (+ LayerNorm gamma / beta with `use_layer_norm`); "legacy" GRU ``gates_*``
    ``[in+H, 2H]`` / ``candidate_*`` ``[in+H, H]``, LSTM ``[in+H, 4H]``.  ``seq_embeds`` [n_items+1, hidden_units[0]]
    (the pad row is an ordinary row), ``item_embeds`` [n_items, K], ``item_biases``, the head ``dense_kernel``
    [H_last, K] and ``dense_bias``.  Biases are non-zero so that their placement is tested.
    ``weights_io.rnn4rec_weights`` turns them into the engine's dict."""
    hidden_units = [int(h) for h in hidden_units]
    small = lambda *s: (rng.standard_normal(s) * 0.1).astype(np.float32)      # noqa: E731
    layers, d = [], hidden_units[0]
    for H in hidden_units:
        if scheme == "keras":
            G = 3 if rnn_type == "gru" else 4
            lw = dict(kernel=_glorot(rng, (d, G * H)), recurrent_kernel=_glorot(rng, (H, G * H)),
                      bias=small(2, G * H) if rnn_type == "gru" else small(G * H))
            if use_layer_norm:
                lw.update(gamma=rng.uniform(0.5, 1.5, H).astype(np.float32), beta=small(H))
        elif scheme == "legacy":
            if rnn_type == "gru":
                lw = dict(gates_kernel=_glorot(rng, (d + H, 2 * H)), gates_bias=small(2 * H),
                          candidate_kernel=_glorot(rng, (d + H, H)), candidate_bias=small(H))
            else:
                lw = dict(kernel=_glorot(rng, (d + H, 4 * H)), bias=small(4 * H))
        else:
            raise ValueError(f"unknown RNN4Rec naming scheme `{scheme}`")
        layers.append(lw)
        d = H
    return dict(rnn_scheme=scheme, rnn_type=rnn_type, use_layer_norm=bool(use_layer_norm and scheme == "keras"),
                seq_embeds=_glorot(rng, (n_items + 1, hidden_units[0])), item_embeds=_glorot(rng, (n_items, K)),
                item_biases=small(n_items), rnn_layers=layers, dense_kernel=_glorot(rng, (d, K)), dense_bias=small(K))


def _conv_kernel(rng, w, c_in, c_out):
    lim = np.sqrt(6.0 / (w * c_in + w * c_out))          # Keras glorot_uniform of a Conv1D kernel [w, in, out]
    return rng.uniform(-lim, lim, size=(w, c_in, c_out)).astype(np.float32)


def _conv_model_tables(rng, n_users, n_items, K):
    """The four embedding-scope tables of Caser / WaveNet: ``user_embeds`` [n_users+1, K] (the last row is the OOV
    row ``set_embeddings`` overwrites), ``seq_embeds`` [n_items+1, K] (the pad row, an ordinary random row distinct
    from the others), ``item_embeds`` [n_items, 2K], ``item_biases`` [n_items]."""
    return dict(user_embeds=_glorot(rng, (n_users + 1, K)), seq_embeds=_glorot(rng, (n_items + 1, K)),
                item_embeds=_glorot(rng, (n_items, 2 * K)),
                item_biases=(rng.standard_normal(n_items) * 0.1).astype(np.float32))


def make_caser_weights(rng, n_users, n_items, K, max_seq_len=10, nh_filters=2, nv_filters=4):
    """Caser variables (libreco/algorithms/caser.py:162-221) in their raw shapes: the four tables, ``convs`` = the
    horizontal Conv1D layers {kernel [h, K, nh], bias [nh]} for h = 1..T, ``vertical`` {kernel [1, T, nv], bias [nv]},
    the head ``dense_kernel`` [T*nh + K*nv, K], ``dense_bias`` [K].  Biases are non-zero and of both signs, so that
    ReLU zeros and the max-pool positions are exercised.  ``weights_io.caser_weights`` packs them."""
    T, nh, nv = int(max_seq_len), int(nh_filters), int(nv_filters)
    bias = lambda n: (rng.standard_normal(n) * 0.1).astype(np.float32)      # noqa: E731
    w = _conv_model_tables(rng, n_users, n_items, K)
    w.update(convs=[dict(kernel=_conv_kernel(rng, h, K, nh), bias=bias(nh)) for h in range(1, T + 1)],
             vertical=dict(kernel=_conv_kernel(rng, 1, T, nv), bias=bias(nv)),
             dense_kernel=_glorot(rng, (T * nh + K * nv, K)), dense_bias=bias(K))
    return w


def make_wavenet_weights(rng, n_users, n_items, K, n_filters=16, n_blocks=1, n_layers_per_block=4, dilated=True):
    """WaveNet variables (libreco/algorithms/wave_net.py:166-222) in their raw shapes: the four tables, ``convs`` =
    the causal Conv1D layers {kernel [2, C_in, F], bias [F]}, ``out_conv`` {kernel [1, F, F], bias [F]}, the head
    ``dense_kernel`` [F, K], ``dense_bias`` [K], and ``dilations`` (``weights_io.wavenet_dilations``).  Biases are
    non-zero and of both signs.  ``weights_io.wavenet_weights`` packs them."""
    from .weights_io import wavenet_dilations

    F = int(n_filters)
    dil = wavenet_dilations(n_blocks, n_layers_per_block, dilated)
    bias = lambda n: (rng.standard_normal(n) * 0.1).astype(np.float32)      # noqa: E731
    w = _conv_model_tables(rng, n_users, n_items, K)
    w.update(convs=[dict(kernel=_conv_kernel(rng, 2, K if i == 0 else F, F), bias=bias(F)) for i in range(len(dil))],
             out_conv=dict(kernel=_conv_kernel(rng, 1, F, F), bias=bias(F)),
             dense_kernel=_glorot(rng, (F, K)), dense_bias=bias(K), dilations=dil)
    return w

"""Weight interchange with the reference's on-disk formats (SURVEY.md §8b "Weight interchange",
Appendix C) — pure host code:

* ``<model_name>.npz`` with ``user_embed`` / ``item_embed`` (``EmbedBase.save(inference_only=True)``,
  ``libreco/bases/embed_base.py:289-295``; read back by ``EmbedBase.load``, :323-330);
* ``<model_name>_tf_variables.npz`` keyed by TF variable name (``utils/save_load.py:70-98``): the
  embedding-scope names are fixed by the reference's graph code, the un-named ``tf_dense`` /
  batch-norm variables carry TensorFlow's auto-generated names, so those go through an explicit
  name map;
* ``<model_name>_default_recs.npz`` (``utils/save_load.py:39-48``).
"""
from __future__ import annotations

import os

import numpy as np

EMBEDDING_SCOPE = {
    "user_embeds": "embedding/user_embeds_var:0", "item_embeds": "embedding/item_embeds_var:0",
    "sparse_embeds": "embedding/sparse_embeds_var:0", "dense_embeds": "embedding/dense_embeds_var:0",
    "user_linear": "embedding/user_linear_var:0", "item_linear": "embedding/item_linear_var:0",
    "sparse_linear": "embedding/sparse_linear_var:0", "dense_linear": "embedding/dense_linear_var:0",
}


def save_embed_model(path, model_name, user_embed, item_embed):
    """Write what ``EmbedBase.save(path, model_name, inference_only=True)`` writes for the variables."""
    os.makedirs(path, exist_ok=True)
    np.savez_compressed(os.path.join(path, model_name), user_embed=np.asarray(user_embed, dtype=np.float32),
                        item_embed=np.asarray(item_embed, dtype=np.float32))


def load_embed_model(path, model_name):
    """(user_embed, item_embed) of a reference-saved embed model (last rows = OOV)."""
    v = np.load(os.path.join(path, f"{model_name}.npz"))
    return v["user_embed"], v["item_embed"]


def to_tf_variables(weights, extra_names=None):
    """Engine weight dict -> ``{tf variable name: array}``.  Tables use the fixed embedding-scope
    names; every other entry needs a name in `extra_names` ({engine key: tf name}).  Shapes follow the
    reference's ``var_shape``s: ``user_linear_var`` / ``item_linear_var`` are ``[V, 1]``
    (``fm.py:181-196``), ``sparse_linear_var`` / ``dense_linear_var`` stay 1-D
    (``[sparse_feature_size]`` / ``[dense_field_size]``, ``fm.py:219-249``, ``deepfm.py:224-256``)."""
    out = {}
    for k, name in EMBEDDING_SCOPE.items():
        if weights.get(k) is not None:
            a = np.asarray(weights[k], dtype=np.float32)
            if k in ("user_linear", "item_linear"):
                a = a.reshape(-1, 1)
            elif k in ("sparse_linear", "dense_linear"):
                a = a.reshape(-1)
            out[name] = a
    for k, name in (extra_names or {}).items():
        out[name] = np.asarray(weights[k], dtype=np.float32)
    return out


def save_tf_variables(path, model_name, weights, extra_names=None):
    os.makedirs(path, exist_ok=True)
    np.savez_compressed(os.path.join(path, f"{model_name}_tf_variables"), **to_tf_variables(weights, extra_names))


def load_tf_variables(path, model_name, extra_names=None):
    """Inverse of :func:`save_tf_variables` (also reads files written by the reference)."""
    from .feat_models import from_tf_variables

    npz = np.load(os.path.join(path, f"{model_name}_tf_variables.npz"))
    w = from_tf_variables(npz)
    for k, name in (extra_names or {}).items():
        w[k] = npz[name]
    return w


def save_default_recs(path, model_name, default_recs):
    np.savez_compressed(os.path.join(path, f"{model_name}_default_recs"), default_recs=np.asarray(default_recs))


def load_default_recs(path, model_name):
    return np.load(os.path.join(path, f"{model_name}_default_recs.npz"))["default_recs"]


# ------------------------------------------------------------------------------------------------
# TensorFlow auto-generated variable names of the un-named layers
# ------------------------------------------------------------------------------------------------
# The reference never names its heads: ``tf_dense(units=1)`` (layers/dense.py:52-80) becomes a
# ``tf.keras.layers.Dense`` / ``tf.layers.dense`` whose variables TensorFlow names ``dense``,
# ``dense_1``, ... in CREATION ORDER; ``tf.layers.batch_normalization`` likewise
# (``batch_normalization``, ``batch_normalization_1``, ...), prefixed by the enclosing
# ``tf.variable_scope`` — ``dense_nn`` opens ``<name>`` (default "mlp") and names its Dense layers
# ``<name>_layer<i>`` (layers/dense.py:28-33).  The creation order per model is read off the graph
# builders: fm.py:152-171, deepfm.py:158-174, din.py:205-218 (+ the "attention" dense_nn,
# layers/attention.py:47-53), youtube_ranking.py:208-217, two_tower.py:400-409, autoint.py:160-168 (+
# multi_head_attention, layers/attention.py:67-138, whose graph depends on the TensorFlow version), transformer.py:
# 203-339 (multi_head_attention and the two FFN tf_dense per layer, layers/transformer.py:147-166, then the head).  No TensorFlow exists in
# this environment, so this table is RESTATED from TensorFlow's documented uniquifying rule and is
# unverified against a real checkpoint; ``resolve_tf_names`` therefore checks every expected name AND
# shape against the file and reports exactly what is missing instead of guessing.
def _bn_names(prefix):
    return {k: f"{prefix}/{v}:0" for k, v in (("gamma", "gamma"), ("beta", "beta"), ("mean", "moving_mean"),
                                             ("var", "moving_variance"))}


def _mlp_names(scope, n_layers, use_bn):
    names = {"kernels": [f"{scope}/{scope}_layer{i}/kernel:0" for i in range(1, n_layers + 1)],
             "biases": [f"{scope}/{scope}_layer{i}/bias:0" for i in range(1, n_layers + 1)]}
    if use_bn:
        names["bn_in"] = _bn_names(f"{scope}/batch_normalization")
        names["bns"] = [_bn_names(f"{scope}/batch_normalization_{i}") for i in range(1, n_layers)]
    return names


def _dense_name(i):
    return "dense" if i == 0 else f"dense_{i}"


def autoint_head_dims(att_embed_size):
    """``attention_config`` (libreco/tfops/configs.py:6-17): head size per attention layer; None / 0 -> (8, 8, 8),
    an int -> one layer."""
    if not att_embed_size:
        return [8, 8, 8]
    if isinstance(att_embed_size, (int, np.integer)):
        return [int(att_embed_size)]
    if isinstance(att_embed_size, (list, tuple)):
        return [int(v) for v in att_embed_size]
    raise ValueError("att_embed_size must be int or list")


def autoint_scheme(version):
    """Which graph ``multi_head_attention`` (layers/attention.py:67-138) built: "keras" for TensorFlow >= 2.10
    (``tf.keras.layers.MultiHeadAttention``), "legacy" before.  Takes a scheme name or a TF version string."""
    if version in _MHA_VARS:
        return version
    parts = [int(p) for p in str(version).split(".")[:2] if p.isdigit()]
    return "keras" if tuple(parts + [0, 0][len(parts):]) >= (2, 10) else "legacy"


# ------------------------------------------------------------------------------------------------
# One ``multi_head_attention`` layer (layers/attention.py:67-138), shared by AutoInt and Transformer.  X [rows, d_in],
# width D = H * hd, no biases.  "keras" (TF >= 2.10, tf.keras.layers.MultiHeadAttention): query / key / value
# [d_in, H, hd] and attention_output [H, hd, d_in].  "legacy": four tf_dense created as q, k, v, out: query / key
# [d_in, D], value [D, D] and output [D, d_in]; ``values = tf_dense(D)(keys)`` acts on the PROJECTED keys
# (attention.py:104-106), so V = (X Wk) Wv'.
# ------------------------------------------------------------------------------------------------
_MHA_VARS = {"keras": ("query", "key", "value", "attention_output"), "legacy": ("query", "key", "value", "output")}


def _check_mha_scheme(scheme, who):
    if scheme not in _MHA_VARS:
        raise ValueError(f"{who}: unknown naming scheme `{scheme}`")


def _mha_tf_names(scheme, prefix, layer, first_dense):
    """TF variable names of attention layer `layer` (0-based) under the scope `prefix`: keras
    ``{prefix}multi_head_attention[_layer]/{query,key,value,attention_output}/kernel:0``, legacy
    ``{prefix}dense_{first_dense + j}/kernel:0`` for q, k, v, out."""
    if scheme == "keras":
        scope = f"{prefix}multi_head_attention{'' if layer == 0 else f'_{layer}'}"
        return {k: f"{scope}/{k}/kernel:0" for k in _MHA_VARS[scheme]}
    return {k: f"{prefix}{_dense_name(first_dense + j)}/kernel:0" for j, k in enumerate(_MHA_VARS[scheme])}


def _mha_tf_shapes(scheme, d_in, D, H):
    """Raw shapes of one layer's variables (any scheme other than "keras" reads as legacy)."""
    if scheme == "keras":
        hd = D // H
        return dict(query=(d_in, H, hd), key=(d_in, H, hd), value=(d_in, H, hd), attention_output=(H, hd, d_in))
    return dict(query=(d_in, D), key=(d_in, D), value=(D, D), output=(D, d_in))


def _mha_2d(scheme, d_in, D):
    """The 2-D shapes the trainers hold one layer's variables in, columns head-major: [d_in, D] projections ([D, D]
    for the legacy value) and the [D, d_in] output.  Reshaping to :func:`_mha_tf_shapes` is the inverse."""
    return dict(zip(_MHA_VARS[scheme], ((d_in, D), (d_in, D), (D, D) if scheme == "legacy" else (d_in, D), (D, d_in))))


def _mha_engine(lw, scheme):
    """One layer's raw variables -> the engines' {wq, wk, wv [d_in, D], wo [D, d_in]}: keras kernels flattened; legacy
    the effective value map Wk Wv', multiplied in float64 and then cast."""
    f32 = lambda a: np.asarray(a, dtype=np.float32)      # noqa: E731
    if scheme == "keras":
        d_in, D = np.shape(lw["query"])[0], int(np.prod(np.shape(lw["query"])[1:]))
        return dict(wq=f32(lw["query"]).reshape(d_in, D), wk=f32(lw["key"]).reshape(d_in, D),
                    wv=f32(lw["value"]).reshape(d_in, D), wo=f32(lw["attention_output"]).reshape(D, d_in))
    wk = f32(lw["key"])
    return dict(wq=f32(lw["query"]), wk=wk, wv=(wk.astype(np.float64) @ np.asarray(lw["value"], dtype=np.float64)
                                                ).astype(np.float32), wo=f32(lw["output"]))


def default_tf_names(model_name, n_hidden, use_bn, use_tf_attention=False, n_layers=None, scheme="keras",
                     positional_embedding="trainable", feat_agg_mode="concat", item_sparse=False, item_dense=False,
                     rnn_type="gru", use_layer_norm=False):
    """{engine weight key: TF variable name (or nested dict / list of names)} for the auto-named
    variables of `model_name` in {"FM", "DeepFM", "DIN", "YouTubeRanking", "TwoTower", "AutoInt", "Transformer",
    "RNN4Rec", "Caser", "WaveNet", "SIM"}.

    SIM (sim.py:193-304, creation order: the sequence projection, the first stage, the attention, the second stage):
    ``dense/kernel:0`` (``seq_proj``), the ``first_stage_mlp`` stack and its head ``dense_1``; "keras"
    ``multi_head_attention/{query,key,value,attention_output}/kernel:0`` and the head ``dense_2``; "legacy" q, k, v,
    out ``dense_2`` .. ``dense_5`` and the head ``dense_6``; the ``second_stage_mlp`` stack (under ``mlp``).  Returned
    under ``seq_proj``, ``first_stage_mlp``, ``first_stage_out_kernel`` / ``_bias``, ``sim_mha``, ``mlp``,
    ``out_kernel`` and ``out_bias``.

    Caser (caser.py:194-220; `n_layers` = max_seq_len T): the horizontal ``conv1d[_i]/{kernel,bias}:0`` for
    i = 0..T-1 under ``convs``, the vertical ``conv1d_T`` under ``vertical``, the head ``dense/{kernel,bias}:0``.
    WaveNet (wave_net.py:198-221; `n_layers` = n_blocks * n_layers_per_block): the causal ``conv1d[_i]`` under
    ``convs``, the 1x1 ``conv1d_{n_layers}`` under ``out_conv``, the head ``dense``.  Both also use the four
    ``CONV_TABLE_KEYS`` of ``DYN_EMBED_TABLES``.

    RNN4Rec (rnn4rec.py:151-237 with layers/recurrent.py:4-63; `n_layers` = len(hidden_units)): "keras" layer i is
    ``{t}[_i]/{t}_cell/{kernel,recurrent_kernel,bias}:0`` (t = gru or lstm) plus, with `use_layer_norm`,
    ``layer_normalization[_i]/{gamma,beta}:0``; "legacy" cell i is ``rnn/multi_rnn_cell/cell_{i}/gru_cell/{gates,
    candidate}/{kernel,bias}:0`` or ``.../lstm_cell/{kernel,bias}:0``.  Both: the head ``dense/{kernel,bias}:0``.
    Returned under ``rnn_layers`` (per layer {kernel, recurrent_kernel, bias[, gamma, beta]} or {gates_kernel,
    gates_bias, candidate_kernel, candidate_bias} or {kernel, bias}), ``dense_kernel`` and ``dense_bias``.  Keras
    cell scopes differ between Keras versions: `extra_names` overrides them.

    Transformer (transformer.py:203-339; layer l = 1..L opens ``transformer_layer{l}``): per layer
    ``rms_norm_att/scale:0``, ``rms_norm_ffn/scale:0``, the attention and the two bias-free FFN ``tf_dense``.  "keras":
    ``multi_head_attention[_{l-1}]/{query,key,value,attention_output}/kernel:0`` and FFN ``dense_{2(l-1)}``,
    ``dense_{2(l-1)+1}``, the head ``dense_{2L}``; "legacy": q, k, v, out, ffn1, ffn2 are ``dense_{6(l-1)}`` ..
    ``dense_{6(l-1)+5}`` and the head ``dense_{6L}``.  Both: ``rms_norm_last/scale:0``, ``rms_norm_item/scale:0``,
    ``transformer/positional_encoding:0`` (trainable positions only; the sinusoidal table is not saved), the
    ``mlp`` stack, and in elementwise mode ``elementwise_{sparse,dense}_feats/layer_norm/{scale,bias}:0`` for the
    sides with item features.  Returned under ``tfm_layers`` (per layer {query, key, value, attention_output | output,
    rms_att, rms_ffn, ffn1, ffn2}), ``rms_last``, ``rms_item``, ``positional_encoding``, ``ln_sparse`` / ``ln_dense``,
    ``mlp``, ``out_kernel``, ``out_bias``.

    AutoInt (autoint.py:160-168, one ``multi_head_attention`` per layer, then ``tf_dense(1)``) has two schemes:
    "keras" (TF >= 2.10): ``multi_head_attention[_i]/{query,key,value,attention_output}/kernel:0`` and the head
    ``dense/{kernel,bias}:0``; "legacy": four bias-free ``tf_dense`` per layer created as q, k, v, out, so layer l
    owns ``dense_{4l}`` .. ``dense_{4l+3}`` and the head is ``dense_{4L}``.  Returned under ``autoint_mha``
    (per-layer {query, key, value, attention_output | output}), ``out_kernel``, ``out_bias``."""
    if model_name == "RNN4Rec":
        return _rnn4rec_names(scheme, rnn_type, n_layers, use_layer_norm)
    if model_name == "SIM":
        return _sim_names(scheme, n_hidden, use_bn)
    if model_name in ("Caser", "WaveNet"):
        return _conv_names(model_name, n_layers)
    if model_name == "Transformer":
        _check_mha_scheme(scheme, "Transformer")
        layers = []
        for i in range(n_layers):
            sc = f"transformer_layer{i + 1}"
            lw = _mha_tf_names(scheme, f"{sc}/", i, 6 * i)
            ffn = 2 * i if scheme == "keras" else 6 * i + 4
            lw.update(rms_att=f"{sc}/rms_norm_att/scale:0", rms_ffn=f"{sc}/rms_norm_ffn/scale:0",
                      ffn1=f"{sc}/{_dense_name(ffn)}/kernel:0", ffn2=f"{sc}/{_dense_name(ffn + 1)}/kernel:0")
            layers.append(lw)
        head = _dense_name((2 if scheme == "keras" else 6) * n_layers)
        out = {"tfm_layers": layers, "rms_last": "rms_norm_last/scale:0", "rms_item": "rms_norm_item/scale:0",
               "mlp": _mlp_names("mlp", n_hidden, use_bn), "out_kernel": f"{head}/kernel:0", "out_bias": f"{head}/bias:0"}
        if positional_embedding not in ("sinusoidal", "sin", "sinusoid"):
            out["positional_encoding"] = "transformer/positional_encoding:0"
        if feat_agg_mode == "elementwise":
            for side, present in (("sparse", item_sparse), ("dense", item_dense)):
                if present:
                    out[f"ln_{side}"] = {k: f"elementwise_{side}_feats/layer_norm/{k}:0" for k in ("scale", "bias")}
        return out
    if model_name == "AutoInt":
        _check_mha_scheme(scheme, "AutoInt")
        head = _dense_name(0 if scheme == "keras" else 4 * n_layers)
        return {"autoint_mha": [_mha_tf_names(scheme, "", i, 4 * i) for i in range(n_layers)],
                "out_kernel": f"{head}/kernel:0", "out_bias": f"{head}/bias:0"}
    if model_name == "FM":
        out = {"lin_kernel": "dense/kernel:0", "lin_bias": "dense/bias:0",
               "pw_kernel": "dense_1/kernel:0", "pw_bias": "dense_1/bias:0"}
        if use_bn:
            out["fm_bn"] = _bn_names("batch_normalization")
        return out
    if model_name == "DeepFM":
        return {"lin_kernel": "dense/kernel:0", "lin_bias": "dense/bias:0", "mlp": _mlp_names("mlp", n_hidden, use_bn),
                "out_kernel": "dense_1/kernel:0", "out_bias": "dense_1/bias:0"}
    if model_name == "DIN":
        out = {"mlp": _mlp_names("mlp", n_hidden, use_bn), "out_kernel": "dense/kernel:0", "out_bias": "dense/bias:0"}
        if not use_tf_attention:
            out["attention"] = {"k1": "attention/attention_layer1/kernel:0", "b1": "attention/attention_layer1/bias:0",
                                "k2": "attention/attention_layer2/kernel:0", "b2": "attention/attention_layer2/bias:0"}
        return out
    if model_name == "YouTubeRanking":
        return {"mlp": _mlp_names("mlp", n_hidden, use_bn), "out_kernel": "dense/kernel:0", "out_bias": "dense/bias:0"}
    if model_name == "TwoTower":
        return {"user_tower": _mlp_names("user_tower", n_hidden, use_bn),
                "item_tower": _mlp_names("item_tower", n_hidden, use_bn)}
    raise ValueError(f"no TensorFlow name table for model `{model_name}`")


def resolve_tf_names(npz, names, shapes=None):
    """Read the (possibly nested) name table out of `npz`; a missing variable raises a ``KeyError`` that
    lists the expected name and the names the file does contain.  With `shapes` (the same nesting, a shape
    tuple per name, ``None`` entries match any size) a variable of another shape raises the same way."""
    def have():
        return sorted(f"{k} {tuple(np.shape(npz[k]))}" for k in npz.files if not k.startswith("embedding/"))

    def take(n, shp):
        if isinstance(n, dict):
            return {k: take(v, shp[k] if shp is not None else None) for k, v in n.items()}
        if isinstance(n, list):
            return [take(v, shp[i] if shp is not None else None) for i, v in enumerate(n)]
        if n not in npz:
            raise KeyError(f"TF variable `{n}` not in the file; non-embedding variables present: {have()}")
        a = np.asarray(npz[n])
        if shp is not None and (a.ndim != len(shp) or any(e is not None and e != d for e, d in zip(shp, a.shape))):
            raise KeyError(f"TF variable `{n}` has shape {a.shape}, expected {tuple(shp)}; non-embedding variables "
                           f"present: {have()}")
        return a
    return take(names, shapes)


def _put_tf_names(out, names, values):
    """The inverse of :func:`resolve_tf_names`: ``out[name] = values`` as float32 for every name of the (possibly
    nested) table `names`, `values` nested the same way (dicts indexed by the table's keys)."""
    if isinstance(names, dict):
        for k in names:
            _put_tf_names(out, names[k], values[k])
    elif isinstance(names, list):
        for n, v in zip(names, values):
            _put_tf_names(out, n, v)
    else:
        out[names] = np.asarray(values, dtype=np.float32)
    return out


def autoint_tf_shapes(scheme, K, num_heads, head_dims):
    """Expected shapes for :func:`default_tf_names` ("AutoInt"): keras ``query/key/value [K, H, hd]``,
    ``attention_output [H, hd, K]``; legacy ``q, k [K, D]``, ``v [D, D]`` (applied to the projected keys),
    ``out [D, K]``; the head ``[F*K, 1]`` (F is not known here) and ``[1]``."""
    return {"autoint_mha": [_mha_tf_shapes(scheme, K, num_heads * hd, num_heads) for hd in head_dims],
            "out_kernel": (None, 1), "out_bias": (1,)}


def autoint_layers(mha, scheme):
    """Per-layer variables of either graph -> the engine's ``autoint_layers`` [{wq, wk, wv [K, D], wo [D, K]}],
    columns head-major (h * hd + j, the order ``_split_heads`` reshapes into).  keras: the [K, H, hd] / [H, hd, K]
    kernels flattened.  legacy: ``values = tf_dense(D)(keys)`` acts on the PROJECTED keys (attention.py:104-106),
    so V = (X Wk) Wv' and the effective value map is Wk Wv', multiplied in float64 and then cast."""
    _check_mha_scheme(scheme, "AutoInt")
    return [_mha_engine(lw, scheme) for lw in mha]


def autoint_weights(raw):
    """Engine weight dict for :class:`feat_models.AutoInt` from the raw variables of either graph: ``raw`` holds
    the embedding tables, ``autoint_scheme``, ``autoint_mha`` (per layer, as :func:`default_tf_names` names them),
    ``num_heads``, ``use_residual``, ``out_kernel`` and ``out_bias``; other entries pass through."""
    w = {k: v for k, v in raw.items() if k not in ("autoint_mha", "autoint_scheme")}
    w["autoint_layers"] = autoint_layers(raw["autoint_mha"], raw["autoint_scheme"])
    w["out_kernel"] = np.asarray(raw["out_kernel"], dtype=np.float32).reshape(-1)
    w["out_bias"] = np.float32(np.asarray(raw["out_bias"]).reshape(-1)[0])
    return w


def autoint_tf_variables(raw):
    """Raw AutoInt variables of either graph (the layout :func:`autoint_weights` takes, e.g.
    ``training.AutoIntTrainer.export_weights()``) -> ``{TF variable name: array}`` named by
    :func:`default_tf_names` for the raw dict's scheme: what ``save_tf_variables`` writes as
    ``<name>_tf_variables.npz``, and the inverse of ``load_reference_tf_model(..., "AutoInt")``."""
    names = default_tf_names("AutoInt", None, False, n_layers=len(raw["autoint_mha"]), scheme=raw["autoint_scheme"])
    out = to_tf_variables({k: raw[k] for k in EMBEDDING_SCOPE if k in raw})
    _put_tf_names(out, names["autoint_mha"], raw["autoint_mha"])
    out[names["out_kernel"]] = np.asarray(raw["out_kernel"], dtype=np.float32).reshape(-1, 1)
    out[names["out_bias"]] = np.asarray(raw["out_bias"], dtype=np.float32).reshape(1)
    return out


def transformer_tf_shapes(scheme, names, K, Kp, num_heads, T=None):
    """Expected shapes for the Transformer entries of `names` (:func:`default_tf_names`); D = Kp + K.  keras
    ``query/key/value [D, H, hd]``, ``attention_output [H, hd, D]``; legacy ``q, k, v, out [D, D]`` (v applied to the
    projected keys); FFN ``[D, 4D]``, ``[4D, D]``; positions ``[T, K]``; the MLP's first kernel ``[F*K + D, H1]``
    (F is not known here)."""
    D = Kp + K
    layer = dict(_mha_tf_shapes(scheme, D, D, num_heads), rms_att=(D,), rms_ffn=(D,), ffn1=(D, 4 * D), ffn2=(4 * D, D))
    out = {"tfm_layers": [layer] * len(names["tfm_layers"]), "rms_last": (D,), "rms_item": (Kp,), "out_kernel": (None, 1),
           "out_bias": (1,), "mlp": None}
    if "positional_encoding" in names:
        out["positional_encoding"] = (T, K)
    for k in ("ln_sparse", "ln_dense"):
        if k in names:
            out[k] = {"scale": (K,), "bias": (K,)}
    return out


def transformer_layers(layers, scheme):
    """Per-layer variables of either graph -> the engine's ``tfm_layers`` [{rms_att, wq, wk, wv, wo [D, D], rms_ffn,
    w1 [D, 4D], w2 [4D, D]}], columns head-major.  legacy: the value Dense acts on the PROJECTED keys
    (attention.py:104-106), so the effective value map Wk Wv' is multiplied in float64 and then cast."""
    _check_mha_scheme(scheme, "Transformer")
    f32 = lambda a: np.asarray(a, dtype=np.float32)      # noqa: E731
    return [dict(_mha_engine(lw, scheme), rms_att=f32(lw["rms_att"]).reshape(-1), rms_ffn=f32(lw["rms_ffn"]).reshape(-1),
                 w1=f32(lw["ffn1"]), w2=f32(lw["ffn2"])) for lw in layers]


def transformer_weights(raw):
    """Engine weight dict for :class:`feat_models.Transformer` from the raw variables of either graph: ``raw`` holds
    the embedding tables, ``tfm_scheme``, ``tfm_layers`` (per layer, as :func:`default_tf_names` names them),
    ``rms_last``, ``rms_item``, ``positional_encoding`` (trainable positions), ``ln_sparse`` / ``ln_dense``
    (elementwise mode), ``num_heads``, ``use_causal_mask``, ``feat_agg_mode``, ``mlp``, ``out_kernel`` and
    ``out_bias``; other entries pass through."""
    w = {k: v for k, v in raw.items() if k not in ("tfm_layers", "tfm_scheme")}
    w["tfm_layers"] = transformer_layers(raw["tfm_layers"], raw["tfm_scheme"])
    w["out_kernel"] = np.asarray(raw["out_kernel"], dtype=np.float32).reshape(-1)
    w["out_bias"] = np.float32(np.asarray(raw["out_bias"]).reshape(-1)[0])
    return w


def transformer_tf_variables(raw):
    """Raw Transformer variables of either graph (the layout :func:`transformer_weights` takes) -> ``{TF variable
    name: array}`` named by :func:`default_tf_names` for the raw dict's scheme and options: what ``save_tf_variables``
    writes as ``<name>_tf_variables.npz``, and the inverse of ``load_reference_tf_model(..., "Transformer", ...)``."""
    mlp = raw["mlp"]
    names = default_tf_names("Transformer", len(mlp["kernels"]), mlp.get("bn_in") is not None,
                             n_layers=len(raw["tfm_layers"]), scheme=raw["tfm_scheme"],
                             positional_embedding="trainable" if raw.get("positional_encoding") is not None else "sinusoidal",
                             feat_agg_mode=raw.get("feat_agg_mode", "concat"), item_sparse="ln_sparse" in raw,
                             item_dense="ln_dense" in raw)
    out = to_tf_variables({k: raw[k] for k in EMBEDDING_SCOPE if k in raw})
    _put_tf_names(out, {k: v for k, v in names.items() if k not in ("out_kernel", "out_bias")}, raw)
    out[names["out_kernel"]] = np.asarray(raw["out_kernel"], dtype=np.float32).reshape(-1, 1)
    out[names["out_bias"]] = np.asarray(raw["out_bias"], dtype=np.float32).reshape(1)
    return out


def _sim_names(scheme, n_hidden, use_bn):
    _check_mha_scheme(scheme, "SIM")
    head = _dense_name(2 if scheme == "keras" else 6)
    return {"seq_proj": "dense/kernel:0", "first_stage_mlp": _mlp_names("first_stage_mlp", n_hidden, use_bn),
            "first_stage_out_kernel": "dense_1/kernel:0", "first_stage_out_bias": "dense_1/bias:0",
            "sim_mha": _mha_tf_names(scheme, "", 0, 2), "mlp": _mlp_names("second_stage_mlp", n_hidden, use_bn),
            "out_kernel": f"{head}/kernel:0", "out_bias": f"{head}/bias:0"}


def sim_tf_shapes(scheme, K, num_heads):
    """Expected shapes for :func:`default_tf_names` ("SIM"): ``seq_proj [K', K]`` (K' not known here), the attention
    over width K (:func:`_mha_tf_shapes`), the heads ``[H_last, 1]`` and ``[1]``; the MLP stacks are not checked."""
    return {"seq_proj": (None, K), "first_stage_mlp": None, "first_stage_out_kernel": (None, 1),
            "first_stage_out_bias": (1,), "sim_mha": _mha_tf_shapes(scheme, K, K, num_heads), "mlp": None,
            "out_kernel": (None, 1), "out_bias": (1,)}


def sim_weights(raw):
    """Engine weight dict for :class:`feat_models.SIM` from the raw variables of either graph: ``raw`` holds the
    embedding tables, ``sim_scheme``, ``seq_proj``, ``sim_mha`` (as :func:`default_tf_names` names it), ``num_heads``,
    ``mlp``, ``out_kernel`` and ``out_bias``; the raw attention, the first-stage variables and other entries pass
    through (the engine ignores them), so :func:`sim_tf_variables` writes the dict back losslessly.  legacy: the value
    Dense acts on the PROJECTED keys, so the effective value map Wk Wv' is multiplied in float64 and then cast."""
    _check_mha_scheme(raw["sim_scheme"], "SIM")
    w = dict(raw)
    w["seq_proj"] = np.asarray(raw["seq_proj"], dtype=np.float32)
    w["sim_attention"] = _mha_engine(raw["sim_mha"], raw["sim_scheme"])
    w["out_kernel"] = np.asarray(raw["out_kernel"], dtype=np.float32).reshape(-1)
    w["out_bias"] = np.float32(np.asarray(raw["out_bias"]).reshape(-1)[0])
    return w


def sim_tf_variables(raw):
    """Raw SIM variables of either graph (the layout :func:`sim_weights` takes) -> ``{TF variable name: array}`` named
    by :func:`default_tf_names` for the raw dict's scheme: what ``save_tf_variables`` writes as
    ``<name>_tf_variables.npz``, and the inverse of ``load_reference_tf_model(..., "SIM", ...)``."""
    mlp = raw["mlp"]
    names = default_tf_names("SIM", len(mlp["kernels"]), mlp.get("bn_in") is not None, scheme=raw["sim_scheme"])
    out = to_tf_variables({k: raw[k] for k in EMBEDDING_SCOPE if k in raw})
    _put_tf_names(out, {k: v for k, v in names.items() if not k.endswith(("out_kernel", "out_bias"))}, raw)
    for k in ("first_stage_out_kernel", "out_kernel"):
        out[names[k]] = np.asarray(raw[k], dtype=np.float32).reshape(-1, 1)
    for k in ("first_stage_out_bias", "out_bias"):
        out[names[k]] = np.asarray(raw[k], dtype=np.float32).reshape(1)
    return out


# the embedding-scope tables of the DynEmbedBase models (YouTubeRetrieval, RNN4Rec, Caser, WaveNet)
DYN_EMBED_TABLES = {"user_embeds": "embedding/user_embeds_var:0", "seq_embeds": "embedding/seq_embeds_var:0",
                    "item_embeds": "embedding/item_embeds_var:0", "item_biases": "embedding/item_bias_var:0",
                    "sparse_embeds": "embedding/sparse_embeds_var:0", "dense_embeds": "embedding/dense_embeds_var:0"}


def _dyn_embed_tf_variables(w, keys):
    """``{TF variable name: float32 array}`` of the tables ``keys`` that ``w`` holds; ``item_biases`` written flat."""
    out = {}
    for k in keys:
        if w.get(k) is not None:
            a = np.asarray(w[k], dtype=np.float32)
            out[DYN_EMBED_TABLES[k]] = a.reshape(-1) if k == "item_biases" else a
    return out


def youtube_retrieval_tf_variables(w):
    """YouTubeRetrieval weights in the layout of ``feat_models.YouTubeRetrieval`` (e.g.
    ``training.YouTubeRetrievalTrainer.export_weights()``) -> ``{TF variable name: array}``: the ``embedding`` scope
    of ``youtube_retrieval.py:194-260`` (``seq_embeds_var`` [n_items, K], ``item_embeds_var`` [n_items, H],
    ``item_bias_var`` [n_items], ``sparse_embeds_var``, ``dense_embeds_var``) and the user tower's ``mlp`` dense_nn
    stack.  The inverse of ``load_reference_tf_model(..., "YouTubeRetrieval", ...)``."""
    out = _dyn_embed_tf_variables(w, ("seq_embeds", "item_embeds", "item_biases", "sparse_embeds", "dense_embeds"))
    mlp = w["mlp"]
    return _put_tf_names(out, _mlp_names("mlp", len(mlp["kernels"]), mlp.get("bn_in") is not None), mlp)


def _youtube_retrieval_weights(npz, n_hidden, use_bn, extra_names=None):
    """Engine weight dict of a saved YouTubeRetrieval: every name and shape checked (``KeyError`` naming the
    variable and listing what the file holds)."""
    seq = resolve_tf_names(npz, DYN_EMBED_TABLES["seq_embeds"])
    n_items, K = seq.shape if seq.ndim == 2 else (None, None)
    if n_items is None:
        raise KeyError(f"TF variable `{DYN_EMBED_TABLES['seq_embeds']}` has shape {seq.shape}, expected [n_items, K]")
    names = {"mlp": _mlp_names("mlp", n_hidden, use_bn)}
    names.update(extra_names or {})
    mlp = resolve_tf_names(npz, names)["mlp"]
    H = int(np.shape(mlp["kernels"][-1])[1]) if np.ndim(mlp["kernels"][-1]) == 2 else -1
    dims = [None] + [np.shape(k)[1] if np.ndim(k) == 2 else -1 for k in mlp["kernels"]]
    shapes = {"mlp": {"kernels": [(dims[i] if i else None, dims[i + 1]) for i in range(n_hidden)],
                      "biases": [(dims[i + 1],) for i in range(n_hidden)]}}
    if use_bn:
        din = np.shape(mlp["kernels"][0])[0]
        shapes["mlp"]["bn_in"] = {k: (din,) for k in ("gamma", "beta", "mean", "var")}
        shapes["mlp"]["bns"] = [{k: (dims[i + 1],) for k in ("gamma", "beta", "mean", "var")} for i in range(n_hidden - 1)]
    w = resolve_tf_names(npz, names, shapes)
    tables = {"seq_embeds": (n_items, K), "item_embeds": (n_items, H), "item_biases": (n_items,)}
    for k in ("sparse_embeds", "dense_embeds"):
        if DYN_EMBED_TABLES[k] in npz:
            tables[k] = (None, K)
    w.update(resolve_tf_names(npz, {k: DYN_EMBED_TABLES[k] for k in tables}, tables))
    if np.shape(mlp["kernels"][0])[0] % K:
        raise KeyError(f"TF variable `{names['mlp']['kernels'][0]}` has {np.shape(mlp['kernels'][0])[0]} input rows, "
                       f"not a multiple of K = {K}")
    return w


RNN_CELL_KINDS = {"gru_reset_after": 0, "gru_reset_before": 1, "lstm": 2}   # cell kinds of b200_rnn_encode
RNN_ACT_TANH, RNN_ACT_LN_TANH = 0, 1


def _rnn4rec_names(scheme, rnn_type, n_layers, use_layer_norm):
    if rnn_type not in ("gru", "lstm"):
        raise ValueError(f"`rnn_type` must be gru or lstm, not `{rnn_type}`")
    layers = []
    for i in range(n_layers):
        if scheme == "keras":
            sc = f"{rnn_type}{'' if i == 0 else f'_{i}'}/{rnn_type}_cell"
            lw = {k: f"{sc}/{k}:0" for k in ("kernel", "recurrent_kernel", "bias")}
            if use_layer_norm:
                ln = f"layer_normalization{'' if i == 0 else f'_{i}'}"
                lw.update(gamma=f"{ln}/gamma:0", beta=f"{ln}/beta:0")
        elif scheme == "legacy":
            sc = f"rnn/multi_rnn_cell/cell_{i}/{rnn_type}_cell"
            if rnn_type == "gru":
                lw = {f"{g}_{k}": f"{sc}/{g}/{k}:0" for g in ("gates", "candidate") for k in ("kernel", "bias")}
            else:
                lw = {k: f"{sc}/{k}:0" for k in ("kernel", "bias")}
        else:
            raise ValueError(f"unknown RNN4Rec naming scheme `{scheme}`")
        layers.append(lw)
    return {"rnn_layers": layers, "dense_kernel": "dense/kernel:0", "dense_bias": "dense/bias:0"}


def rnn4rec_tf_shapes(scheme, rnn_type, in_dim, hidden_units, use_layer_norm, K):
    """Expected shapes for :func:`default_tf_names` ("RNN4Rec"): keras GRU ``kernel [in, 3H]``, ``recurrent_kernel
    [H, 3H]``, ``bias [2, 3H]`` (reset_after: input row, recurrent row), keras LSTM ``[in, 4H]``, ``[H, 4H]``,
    ``[4H]``, LayerNorm ``[H]``; legacy GRU ``gates [in+H, 2H]`` + ``[2H]``, ``candidate [in+H, H]`` + ``[H]``,
    legacy LSTM ``[in+H, 4H]`` + ``[4H]``; the head ``[H_last, K]``, ``[K]``."""
    layers, d = [], int(in_dim)
    for H in hidden_units:
        H = int(H)
        if scheme == "keras":
            G = 3 if rnn_type == "gru" else 4
            lw = dict(kernel=(d, G * H), recurrent_kernel=(H, G * H), bias=(2, G * H) if rnn_type == "gru" else (G * H,))
            if use_layer_norm:
                lw.update(gamma=(H,), beta=(H,))
        elif rnn_type == "gru":
            lw = dict(gates_kernel=(d + H, 2 * H), gates_bias=(2 * H,), candidate_kernel=(d + H, H), candidate_bias=(H,))
        else:
            lw = dict(kernel=(d + H, 4 * H), bias=(4 * H,))
        layers.append(lw)
        d = H
    return {"rnn_layers": layers, "dense_kernel": (d, int(K)), "dense_bias": (int(K),)}


def rnn_layers(layers, scheme, rnn_type, in_dim, use_layer_norm):
    """Per-layer raw variables of either graph -> the engine's ``rnn_layers`` [{kind, act, W [in, G*H], U [H, G*H],
    bx [G*H], bh [G*H], gamma [H], beta [H]}] in the canonical layout of ``b200_rnn_encode``.  keras GRU: blocks
    z | r | h as stored, bias rows -> bx, bh.  keras LSTM: i | f | c | o as stored, the one bias -> bx.  legacy GRU:
    the ``[x, h]`` kernels split at row ``in``, gate blocks r | u reordered to u | r, then the candidate; biases -> bx.
    legacy LSTM: blocks i | j | f | o reordered to i | f | j | o, and ``forget_bias = 1.0`` (added at run time by
    ``LSTMCell``) folded into the f bias in float32."""
    f32 = lambda a: np.asarray(a, dtype=np.float32)      # noqa: E731
    out, d = [], int(in_dim)
    for lw in layers:
        if scheme == "keras":
            W, U = f32(lw["kernel"]), f32(lw["recurrent_kernel"])
            H = U.shape[0]
            if rnn_type == "gru":
                b = f32(lw["bias"]).reshape(2, 3 * H)
                kind, bx, bh = RNN_CELL_KINDS["gru_reset_after"], b[0], b[1]
            else:
                kind, bx, bh = RNN_CELL_KINDS["lstm"], f32(lw["bias"]).reshape(-1), np.zeros(4 * H, np.float32)
            act = RNN_ACT_LN_TANH if use_layer_norm else RNN_ACT_TANH
        elif scheme == "legacy":
            if rnn_type == "gru":
                gk, gb = f32(lw["gates_kernel"]), f32(lw["gates_bias"]).reshape(-1)
                ck, cb = f32(lw["candidate_kernel"]), f32(lw["candidate_bias"]).reshape(-1)
                H = ck.shape[1]
                perm = np.r_[H:2 * H, 0:H]
                W = np.concatenate([gk[:d, perm], ck[:d]], axis=1)
                U = np.concatenate([gk[d:, perm], ck[d:]], axis=1)
                kind, bx = RNN_CELL_KINDS["gru_reset_before"], np.concatenate([gb[perm], cb])
                bh = np.zeros(3 * H, np.float32)
            else:
                k, b = f32(lw["kernel"]), f32(lw["bias"]).reshape(-1)
                H = k.shape[1] // 4
                perm = np.r_[0:H, 2 * H:3 * H, H:2 * H, 3 * H:4 * H]
                W, U, bx = k[:d, perm], k[d:, perm], b[perm].copy()
                bx[H:2 * H] += np.float32(1.0)
                kind, bh = RNN_CELL_KINDS["lstm"], np.zeros(4 * H, np.float32)
            act = RNN_ACT_TANH
        else:
            raise ValueError(f"unknown RNN4Rec naming scheme `{scheme}`")
        ln = act == RNN_ACT_LN_TANH
        out.append(dict(kind=kind, act=act, W=np.ascontiguousarray(W), U=np.ascontiguousarray(U),
                        bx=np.ascontiguousarray(bx), bh=np.ascontiguousarray(bh),
                        gamma=f32(lw["gamma"]).reshape(-1) if ln else np.ones(H, np.float32),
                        beta=f32(lw["beta"]).reshape(-1) if ln else np.zeros(H, np.float32)))
        d = H
    return out


def rnn_raw_layers(layers, scheme, rnn_type, in_dim, forget_bias=1.0):
    """The inverse of :func:`rnn_layers`: canonical layers -> the per-layer raw variables of the graph `scheme`.  The
    gate reorderings are involutions and the ``[x, h]`` kernels are stacked back; the TF1 LSTM's f bias has
    ``forget_bias`` (1.0, what :func:`rnn_layers` folded in) subtracted in float32, so a raw -> canonical -> raw round
    trip is exact for every variable except that bias, which it returns as ``fl32(fl32(b + 1) - 1)``.
    ``forget_bias=0`` maps gradients, which the fold does not change."""
    f32 = lambda a: np.asarray(a, dtype=np.float32)      # noqa: E731
    out, d = [], int(in_dim)
    for lw in layers:
        W, U, bx, bh = f32(lw["W"]), f32(lw["U"]), f32(lw["bx"]).reshape(-1), f32(lw["bh"]).reshape(-1)
        H = U.shape[0]
        if scheme == "keras":
            raw = dict(kernel=W.copy(), recurrent_kernel=U.copy(),
                       bias=np.stack([bx, bh]) if rnn_type == "gru" else bx.copy())
            if int(lw["act"]) == RNN_ACT_LN_TANH:
                raw.update(gamma=f32(lw["gamma"]).copy(), beta=f32(lw["beta"]).copy())
        elif scheme == "legacy":
            if rnn_type == "gru":
                perm = np.r_[H:2 * H, 0:H]
                raw = dict(gates_kernel=np.concatenate([W[:, perm], U[:, perm]], axis=0), gates_bias=bx[perm],
                           candidate_kernel=np.concatenate([W[:, 2 * H:], U[:, 2 * H:]], axis=0),
                           candidate_bias=bx[2 * H:].copy())
            else:
                perm = np.r_[0:H, 2 * H:3 * H, H:2 * H, 3 * H:4 * H]
                b = bx[perm].copy()
                b[2 * H:3 * H] -= np.float32(forget_bias)
                raw = dict(kernel=np.concatenate([W, U], axis=0)[:, perm], bias=b)
        else:
            raise ValueError(f"unknown RNN4Rec naming scheme `{scheme}`")
        out.append({k: np.ascontiguousarray(v) for k, v in raw.items()})
        d = H
    return out


def rnn4rec_weights(raw):
    """Engine weight dict for :class:`feat_models.RNN4Rec` from the raw variables of either graph: ``raw`` holds
    ``seq_embeds`` [n_items+1, hidden_units[0]], ``item_embeds`` [n_items, K], ``item_biases`` [n_items],
    ``rnn_scheme``, ``rnn_type``, ``use_layer_norm``, ``rnn_layers`` (per layer, as :func:`default_tf_names` names
    them), ``dense_kernel`` [H_last, K] and ``dense_bias`` [K]."""
    w = _seq_model_tables(raw, ("seq_embeds", "item_embeds", "item_biases"))
    w["rnn_layers"] = rnn_layers(raw["rnn_layers"], raw["rnn_scheme"], raw["rnn_type"], w["seq_embeds"].shape[1],
                                 bool(raw.get("use_layer_norm", False)))
    return w


def rnn4rec_tf_variables(raw):
    """Raw RNN4Rec variables of either graph (the layout :func:`rnn4rec_weights` takes) -> ``{TF variable name:
    array}`` named by :func:`default_tf_names`: what ``save_tf_variables`` writes as ``<name>_tf_variables.npz``, and
    the inverse of ``load_reference_tf_model(..., "RNN4Rec", ...)``."""
    names = default_tf_names("RNN4Rec", None, False, n_layers=len(raw["rnn_layers"]), scheme=raw["rnn_scheme"],
                             rnn_type=raw["rnn_type"], use_layer_norm=bool(raw.get("use_layer_norm", False)))
    out = _dyn_embed_tf_variables(raw, ("seq_embeds", "item_embeds", "item_biases"))
    _put_tf_names(out, names["rnn_layers"], raw["rnn_layers"])
    out[names["dense_kernel"]] = np.asarray(raw["dense_kernel"], dtype=np.float32)
    out[names["dense_bias"]] = np.asarray(raw["dense_bias"], dtype=np.float32).reshape(-1)
    return out


def _rnn4rec_raw(npz, rnn_type, hidden_units, use_layer_norm, extra_names=None):
    """Raw RNN4Rec variables of a saved model, every name and shape checked; the scheme is read off the names."""
    scheme = "legacy" if any(k.startswith("rnn/multi_rnn_cell/") for k in npz.files) else "keras"
    hidden_units = [int(h) for h in hidden_units]
    names = default_tf_names("RNN4Rec", None, False, n_layers=len(hidden_units), scheme=scheme, rnn_type=rnn_type,
                             use_layer_norm=use_layer_norm)
    names.update(extra_names or {})
    item = resolve_tf_names(npz, DYN_EMBED_TABLES["item_embeds"])
    if item.ndim != 2:
        raise KeyError(f"TF variable `{DYN_EMBED_TABLES['item_embeds']}` has shape {item.shape}, expected [n_items, K]")
    n_items, K = item.shape
    tables = {"seq_embeds": (n_items + 1, hidden_units[0]), "item_embeds": (n_items, K), "item_biases": (n_items,)}
    raw = resolve_tf_names(npz, {k: DYN_EMBED_TABLES[k] for k in tables}, tables)
    raw.update(resolve_tf_names(npz, names, rnn4rec_tf_shapes(scheme, rnn_type, hidden_units[0], hidden_units,
                                                              use_layer_norm, K)))
    raw.update(rnn_scheme=scheme, rnn_type=rnn_type, use_layer_norm=bool(use_layer_norm and scheme == "keras"))
    return raw


# Caser / WaveNet (caser.py:162-221, wave_net.py:166-222): four embedding-scope tables, then auto-named Conv1D
# layers and the Dense head.  The names restate TensorFlow's naming rule and are unverified against a saved model.
CONV_TABLE_KEYS = ("user_embeds", "seq_embeds", "item_embeds", "item_biases")


def _conv_names(model_name, n_conv):
    """Caser: ``n_conv`` = T horizontal layers ``conv1d[_i]`` (i = 0..T-1, kernel size i+1) then the vertical
    ``conv1d_T``.  WaveNet: ``n_conv`` causal layers ``conv1d[_i]`` then the 1x1 layer ``conv1d_{n_conv}``."""
    conv = lambda i: {k: f"conv1d{'' if i == 0 else f'_{i}'}/{k}:0" for k in ("kernel", "bias")}   # noqa: E731
    last = "vertical" if model_name == "Caser" else "out_conv"
    return {"convs": [conv(i) for i in range(n_conv)], last: conv(n_conv), "dense_kernel": "dense/kernel:0",
            "dense_bias": "dense/bias:0"}


def conv_tf_shapes(model_name, n_users, n_items, K, T=None, nh=None, nv=None, F=None, n_conv=None):
    """Expected shapes of every Caser / WaveNet variable: the tables ``user_embeds [n_users+1, K]``, ``seq_embeds
    [n_items+1, K]``, ``item_embeds [n_items, 2K]``, ``item_biases [n_items]``; Caser ``W_h [h, K, nh]``, ``[nh]``
    (h = 1..T), ``Wv [1, T, nv]``, ``[nv]``, head ``[T*nh + K*nv, K]``; WaveNet ``[2, C_in, F]``, ``[F]`` per causal
    layer (C_in = K first, then F), ``[1, F, F]``, ``[F]``, head ``[F, K]``.  Keyed like :func:`_conv_names`."""
    out = {"user_embeds": (n_users + 1, K), "seq_embeds": (n_items + 1, K), "item_embeds": (n_items, 2 * K),
           "item_biases": (n_items,), "dense_bias": (K,)}
    if model_name == "Caser":
        out.update(convs=[{"kernel": (h, K, nh), "bias": (nh,)} for h in range(1, T + 1)],
                   vertical={"kernel": (1, T, nv), "bias": (nv,)}, dense_kernel=(T * nh + K * nv, K))
    else:
        out.update(convs=[{"kernel": (2, K if i == 0 else F, F), "bias": (F,)} for i in range(n_conv)],
                   out_conv={"kernel": (1, F, F), "bias": (F,)}, dense_kernel=(F, K))
    return out


def wavenet_dilations(n_blocks, n_layers_per_block, dilated=True):
    """Per-layer dilations of WaveNet's causal stack: ``2**i`` for layer i of each block (wave_net.py:199-208), or 1
    everywhere for a TF1-trained model, whose ``tf.layers.conv1d`` is built without ``dilation_rate``
    (layers/convolutional.py:19-27)."""
    return [2 ** i if dilated else 1 for _ in range(int(n_blocks)) for i in range(int(n_layers_per_block))]


def _seq_model_tables(raw, keys):
    """The tables ``keys`` (``item_biases`` flat) and the Dense head of a sequence model's raw variables, float32."""
    w = {k: np.asarray(raw[k], dtype=np.float32) for k in keys}
    w["item_biases"] = w["item_biases"].reshape(-1)
    w["dense_kernel"] = np.asarray(raw["dense_kernel"], dtype=np.float32)
    w["dense_bias"] = np.asarray(raw["dense_bias"], dtype=np.float32).reshape(-1)
    return w


def caser_weights(raw):
    """Engine weight dict of :class:`feat_models.Caser` from the raw variables (the four tables, ``convs`` = the T
    horizontal layers {kernel [h, K, nh], bias [nh]}, ``vertical`` {kernel [1, T, nv], bias [nv]}, the head):
    ``conv`` packs them as ``b200_caser_encode`` reads them, W_1 .. W_T, then b_h [T, nh], Wv [T, nv], bv [nv]."""
    f32 = lambda a: np.asarray(a, dtype=np.float32)      # noqa: E731
    convs, vert = raw["convs"], raw["vertical"]
    T, nh, nv = len(convs), int(np.shape(convs[0]["bias"])[-1]), int(np.shape(vert["bias"])[-1])
    w = _seq_model_tables(raw, CONV_TABLE_KEYS)
    w["conv"] = np.concatenate([f32(c["kernel"]).reshape(-1) for c in convs] +
                               [f32(c["bias"]).reshape(-1) for c in convs] +
                               [f32(vert["kernel"]).reshape(-1), f32(vert["bias"]).reshape(-1)])
    w.update(model="Caser", T=T, nh=nh, nv=nv)
    return w


def wavenet_weights(raw):
    """Engine weight dict of :class:`feat_models.WaveNet` from the raw variables (the four tables, ``convs`` = the
    causal layers {kernel [2, C_in, F], bias [F]}, ``out_conv`` {kernel [1, F, F], bias [F]}, ``dilations``, the
    head): ``conv`` packs them as ``b200_wavenet_encode`` reads them, per layer W then b, then W1, b1."""
    f32 = lambda a: np.asarray(a, dtype=np.float32).reshape(-1)      # noqa: E731
    parts = [f32(c[k]) for c in raw["convs"] + [raw["out_conv"]] for k in ("kernel", "bias")]
    w = _seq_model_tables(raw, CONV_TABLE_KEYS)
    w["conv"] = np.concatenate(parts)
    dil = [int(d) for d in raw["dilations"]]
    if len(dil) != len(raw["convs"]):
        raise ValueError(f"WaveNet: {len(dil)} dilations for {len(raw['convs'])} causal layers")
    w.update(model="WaveNet", F=int(np.shape(raw["out_conv"]["bias"])[-1]), dilations=dil)
    return w


def _conv_tf_variables(raw):
    """Raw Caser / WaveNet variables (what :func:`caser_weights` / :func:`wavenet_weights` take) -> ``{TF variable
    name: array}``: what ``save_tf_variables`` writes, and the inverse of ``load_reference_tf_model``."""
    model = "Caser" if "vertical" in raw else "WaveNet"
    names = _conv_names(model, len(raw["convs"]))
    return _put_tf_names(_dyn_embed_tf_variables(raw, CONV_TABLE_KEYS), names, raw)


# the dilations of WaveNet are not variables: the loader takes them as arguments
caser_tf_variables = wavenet_tf_variables = _conv_tf_variables


def _conv_raw(npz, model_name, n_filters=None, n_blocks=None, n_layers_per_block=None, dilated=True,
              extra_names=None):
    """Raw Caser / WaveNet variables of a saved model, every name and shape checked.  Caser reads T off the vertical
    kernel ``conv1d_{T}`` [1, T, nv]: the one layer whose index equals its kernel's T; nh and nv come off the first
    and the vertical bias.  WaveNet's graph (``n_filters``, ``n_blocks``, ``n_layers_per_block``, ``dilated``) is
    taken as arguments: the file does not tell the TF1 graph (dilation 1) from the TF2 one."""
    tab = resolve_tf_names(npz, {k: DYN_EMBED_TABLES[k] for k in ("user_embeds", "item_embeds")})
    if tab["user_embeds"].ndim != 2 or tab["item_embeds"].ndim != 2:
        raise KeyError(f"`{DYN_EMBED_TABLES['user_embeds']}` / `{DYN_EMBED_TABLES['item_embeds']}` must be 2-D")
    (nu1, K), n_items = tab["user_embeds"].shape, tab["item_embeds"].shape[0]
    if model_name == "Caser":
        T = None
        for n in npz.files:
            parts = n.split("/")
            if len(parts) == 2 and parts[1] == "kernel:0" and parts[0].startswith("conv1d_"):
                shp = np.shape(npz[n])
                if len(shp) == 3 and shp[0] == 1 and parts[0] == f"conv1d_{shp[1]}":
                    T = int(shp[1])
        if T is None:
            raise KeyError("Caser: no vertical kernel `conv1d_{T}/kernel:0` of shape [1, T, nv] in the file")
        names = _conv_names("Caser", T)
        nh = int(np.shape(resolve_tf_names(npz, names["convs"][0]["bias"]))[0])
        nv = int(np.shape(resolve_tf_names(npz, names["vertical"]["bias"]))[0])
        shapes = conv_tf_shapes("Caser", nu1 - 1, n_items, K, T=T, nh=nh, nv=nv)
    else:
        F, dil = int(n_filters), wavenet_dilations(n_blocks, n_layers_per_block, dilated)
        names = _conv_names("WaveNet", len(dil))
        shapes = conv_tf_shapes("WaveNet", nu1 - 1, n_items, K, F=F, n_conv=len(dil))
    names.update(extra_names or {})
    raw = resolve_tf_names(npz, {k: DYN_EMBED_TABLES[k] for k in CONV_TABLE_KEYS},
                           {k: shapes[k] for k in CONV_TABLE_KEYS})
    raw.update(resolve_tf_names(npz, names, {k: shapes[k] for k in names}))
    if model_name == "WaveNet":
        raw["dilations"] = dil
    return raw


def load_reference_tf_model(path, model_name, arch, n_hidden, use_bn, use_tf_attention=False, extra_names=None,
                            num_heads=None, att_embed_size=(8, 8, 8), use_residual=True, num_tfm_layers=1,
                            positional_embedding="trainable", use_causal_mask=False, feat_agg_mode="concat",
                            rnn_type="gru", hidden_units=(16,), use_layer_norm=False, n_filters=16, n_blocks=1,
                            n_layers_per_block=4, dilated=True):
    """Engine weight dict of a model saved by the reference (``save_tf_variables``,
    utils/save_load.py:70-98) WITHOUT a hand-written name map: the embedding-scope variables by their
    fixed names, the heads / MLPs / batch-norms through :func:`default_tf_names` (override single entries
    with `extra_names`).  AutoInt takes its own constructor arguments ``num_heads``, ``att_embed_size`` and
    ``use_residual``; its naming scheme (keras or legacy) is read off the names in the file, and every name
    and shape is checked.  Transformer likewise, with ``num_heads``, ``num_tfm_layers``, ``positional_embedding``,
    ``use_causal_mask`` and ``feat_agg_mode`` (``num_heads`` defaults to each model's own default: 2 for AutoInt, 1
    for Transformer).  YouTubeRetrieval (``n_hidden`` Dense layers in the user tower) returns the layout of
    ``feat_models.YouTubeRetrieval``, every name and shape checked.  RNN4Rec takes its constructor's ``rnn_type``,
    ``hidden_units`` and ``use_layer_norm`` (``n_hidden`` and ``use_bn`` are unused), reads the graph (keras or
    legacy) off the names, checks every name and shape and returns the layout of ``feat_models.RNN4Rec``.  Caser
    reads max_seq_len off the vertical kernel; WaveNet takes ``n_filters``, ``n_blocks``, ``n_layers_per_block`` and
    ``dilated`` (False for a TF1-trained model, whose causal layers all have dilation 1).  Both check every name and
    shape and return the layout of ``feat_models.Caser`` / ``feat_models.WaveNet``.  SIM takes ``num_heads`` (default 2),
    reads its attention graph (keras or legacy) off the names, checks every name and shape and returns the layout of
    ``feat_models.SIM``; the first-stage variables are read too and carried along."""
    from .feat_models import from_tf_variables

    npz = np.load(os.path.join(path, f"{model_name}_tf_variables.npz"))
    if arch == "YouTubeRetrieval":
        return _youtube_retrieval_weights(npz, n_hidden, use_bn, extra_names)
    if arch == "RNN4Rec":
        return rnn4rec_weights(_rnn4rec_raw(npz, rnn_type, hidden_units, bool(use_layer_norm), extra_names))
    if arch == "Caser":
        return caser_weights(_conv_raw(npz, "Caser", extra_names=extra_names))
    if arch == "WaveNet":
        return wavenet_weights(_conv_raw(npz, "WaveNet", n_filters, n_blocks, n_layers_per_block, dilated, extra_names))
    w = from_tf_variables(npz)
    if arch == "Transformer":
        scheme = "keras" if "transformer_layer1/multi_head_attention/query/kernel:0" in npz.files else "legacy"
        H = 1 if num_heads is None else int(num_heads)
        K = int(np.shape(npz[EMBEDDING_SCOPE["user_embeds"]])[1])
        # the elementwise layer norms exist for the item feature kinds the data has, which only the file tells
        item_sparse, item_dense = (f"elementwise_{k}_feats/layer_norm/scale:0" in npz.files for k in ("sparse", "dense"))
        names = default_tf_names(arch, n_hidden, use_bn, n_layers=int(num_tfm_layers), scheme=scheme,
                                 positional_embedding=positional_embedding, feat_agg_mode=feat_agg_mode,
                                 item_sparse=item_sparse, item_dense=item_dense)
        names.update(extra_names or {})
        D = int(np.shape(resolve_tf_names(npz, names["rms_last"]))[0])
        if D <= K or D % H:
            raise ValueError(f"Transformer: model width {D} (from `{names['rms_last']}`) must exceed K = {K} and be "
                             f"divisible by num_heads {H}")
        raw = resolve_tf_names(npz, names, transformer_tf_shapes(scheme, names, K, D - K, H))
        w.update(raw, tfm_scheme=scheme, num_heads=H, use_causal_mask=bool(use_causal_mask),
                 feat_agg_mode=feat_agg_mode)
        return transformer_weights(w)
    if num_heads is None:
        num_heads = 2
    if arch == "SIM":
        scheme = "keras" if "multi_head_attention/query/kernel:0" in npz.files else "legacy"
        names = default_tf_names(arch, n_hidden, use_bn, scheme=scheme)
        names.update(extra_names or {})
        K = int(np.shape(npz[EMBEDDING_SCOPE["user_embeds"]])[1])
        if K % int(num_heads):
            raise ValueError(f"SIM: embed size {K} must be divisible by num_heads {num_heads}")
        w.update(resolve_tf_names(npz, names, sim_tf_shapes(scheme, K, int(num_heads))), sim_scheme=scheme,
                 num_heads=int(num_heads))
        return sim_weights(w)
    if arch == "AutoInt":
        hds = autoint_head_dims(att_embed_size)
        scheme = "keras" if "multi_head_attention/query/kernel:0" in npz.files else "legacy"
        names = default_tf_names(arch, n_hidden, use_bn, n_layers=len(hds), scheme=scheme)
        names.update(extra_names or {})
        K = int(np.shape(npz[EMBEDDING_SCOPE["user_embeds"]])[1])
        raw = resolve_tf_names(npz, names, autoint_tf_shapes(scheme, K, int(num_heads), hds))
        if raw["out_kernel"].shape[0] % K or raw["out_kernel"].shape[0] < 2 * K:
            raise KeyError(f"TF variable `{names['out_kernel']}` has shape {raw['out_kernel'].shape}, expected "
                           f"[F*{K}, 1]")
        w.update(raw, autoint_scheme=scheme, num_heads=int(num_heads), use_residual=bool(use_residual))
        return autoint_weights(w)
    names = default_tf_names(arch, n_hidden, use_bn, use_tf_attention)
    names.update(extra_names or {})
    w.update(resolve_tf_names(npz, names))
    if use_tf_attention:
        w["use_tf_attention"] = True
    return w


def load_reference_wide_deep(path, model_name, n_hidden, use_bn):
    """Weight dict for :class:`feat_models.DeepFM` from a WideDeep model saved by the reference
    (``<model_name>_tf_variables.npz``; variables of ``libreco/algorithms/wide_deep.py:150-262``: ``embedding/
    {user,item,sparse,dense}_{wide,deep}_var``, ``wide_term``, the ``deep`` dense_nn stack, ``deep_term``) through
    :func:`feat_models.wide_deep_weights`."""
    from .feat_models import wide_deep_weights

    npz = np.load(os.path.join(path, f"{model_name}_tf_variables.npz"))

    def emb(name):
        key = f"embedding/{name}:0"
        return np.asarray(npz[key]) if key in npz else None

    rest = resolve_tf_names(npz, {"mlp": _mlp_names("deep", n_hidden, use_bn), "wide_kernel": "wide_term/kernel:0",
                                  "wide_bias": "wide_term/bias:0", "deep_kernel": "deep_term/kernel:0",
                                  "deep_bias": "deep_term/bias:0"})
    return wide_deep_weights(emb("user_wide_var"), emb("item_wide_var"), emb("sparse_wide_var"), emb("dense_wide_var"),
                             rest["wide_kernel"], rest["wide_bias"], emb("user_deep_var"), emb("item_deep_var"),
                             emb("sparse_deep_var"), emb("dense_deep_var"), rest["mlp"], rest["deep_kernel"],
                             rest["deep_bias"])

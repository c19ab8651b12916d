"""FM training step on the device (SURVEY.md §8f-1): the reference's graph in training mode
(``libreco/algorithms/fm.py:140-172``), mean sigmoid cross entropy (``tfops/loss.py:14-18``) and
``tf.train.AdamOptimizer`` grouped with the batch-norm update ops
(``libreco/training/tf_trainer.py:112-123``), one call per mini-batch:

    gather + FM term (b200_feat_forward)  ->  BN with batch statistics (b200_bn_train_forward)
    -> Dense(1, elu) head (b200_fm_head_forward) -> loss + d loss / d logit (b200_pointwise_loss)
    -> head backward (b200_fm_head_backward) -> scatter of the field gradients (b200_feat_backward)
    -> TF-Adam over every variable (b200_adam_dense)

Every variable, Adam slot and gradient buffer is a device tensor; nothing returns to the host
during a step (the loss stays a device scalar).  Embedding variables follow TensorFlow's
``_apply_sparse_shared`` semantics: m and v are decayed over the whole variable and the whole
variable moves, i.e. a dense Adam step with a zero-filled gradient.  torch: memory only.
"""
from __future__ import annotations

import ctypes
import functools

import numpy as np

from . import _lib
from .feat_models import (ACT_GELU, ACT_NONE, ACT_RELU, ACT_SWISH, FeatSpec, _dev, feat_backward, feat_forward, linear,
                          permute_mlp_input, tables_struct)
from .weights_io import _MHA_VARS, _check_mha_scheme, _mha_2d, _mha_tf_shapes

BN_EPS = 1e-3          # tf.layers.batch_normalization defaults
BN_MOMENTUM = 0.99
BETA1, BETA2 = 0.9, 0.999

_TABLES = ("user_embeds", "item_embeds", "sparse_embeds", "dense_embeds",
           "user_linear", "item_linear", "sparse_linear", "dense_linear")

_REG_VARS = _TABLES      # tf.get_variable(..., regularizer=self.reg): deepfm.py:186-259, two_tower.py:258-285, din.py, ...


def set_regularisation(tr, reg=None, lr_decay=False, decay_steps=0, decay_rate=0.96):
    """``reg`` (``tf.keras.regularizers.l2(reg)`` on the embedding / linear tables: the optimised loss gains
    ``reg * sum w^2``, the REPORTED loss stays the data loss) and ``lr_decay`` (``tf.train.exponential_decay``,
    staircase, ``decay_steps`` = batches per epoch in the reference) for any trainer of this module."""
    if reg is not None and not (isinstance(reg, float) and reg > 0.0):
        raise ValueError("reg must be float and positive...")
    tr.reg = float(reg) if reg else 0.0
    tr.decay_steps = int(decay_steps) if lr_decay else 0
    tr.decay_rate = float(decay_rate)
    return tr


def _weight_grad(dy, x):
    """dWt [dout, din] = dY^T X on the library's dense kernel.  The kernel tiles the OUTPUT rows over the SMs, so
    the product is taken in the orientation with more output rows (din > dout: (X^T dY)^T) — the reduction runs
    over the batch either way."""
    dyt, xt = dy.t().contiguous(), x.t().contiguous()
    if xt.shape[0] > dyt.shape[0]:
        return linear(xt, dyt, None, False, cache_split=False).t()
    return linear(dyt, xt, None, False, cache_split=False)


class _Trainer:
    """What every trainer of this module shares: the feature spec, device and embed size; the variables (cloned
    device copies of ``weights``), their gradient buffers and Adam slots; the tables struct the gather reads; the
    loss workspace; TF-Adam and ``step_graph``.  A subclass adds its own variables in ``_init_params``.

    ``linear_tables``: the model's linear (wide) tables are variables too (FM, DeepFM).  ``embed_table``: the
    variable whose width is the embed size K.  ``reg_vars``: the variables ``reg`` applies to."""

    linear_tables = False
    embed_table = "user_embeds"
    reg_vars = _REG_VARS

    def __init__(self, spec, weights, use_bn, lr, epsilon, device):
        import torch

        self._torch = torch
        K = int(weights[self.embed_table].shape[1])
        self.spec = spec if isinstance(spec, FeatSpec) else FeatSpec(spec, K, device)
        self.device, self.K = self.spec.device, K
        self.F = 2 + self.spec.n_sparse + self.spec.n_dense
        self.n_items = self.spec.n_items
        self.use_bn, self.lr, self.epsilon, self.t = bool(use_bn), float(lr), float(epsilon), 0
        self.moving = {}
        names = _TABLES if self.linear_tables else _TABLES[:4]
        self.params = {k: self._var(weights[k]) for k in names if weights.get(k) is not None}
        self._init_params(weights)
        p = self.params
        self.grads = {k: torch.zeros_like(v) for k, v in p.items()}
        self.m = {k: torch.zeros_like(v) for k, v in p.items()}
        self.v = {k: torch.zeros_like(v) for k, v in p.items()}
        self.tables = tables_struct(p)
        self._lws = torch.empty(int(_lib.lib.b200_loss_workspace_bytes()), dtype=torch.uint8, device=self.device)

    def _init_params(self, weights):
        raise NotImplementedError

    def _var(self, x, shape=None):
        """Trainable device copy of ``x`` (reshaped to ``shape`` first when given)."""
        if shape is not None:
            x = np.asarray(x).reshape(shape)
        return _dev(x, self.device, self._torch.float32).clone()

    def _export_tables(self):
        return {k: self.params[k].cpu().numpy() for k in _TABLES if k in self.params}

    def _loss(self, logit, labels_d):
        """Mean sigmoid cross entropy: (device loss, d loss / d logit)."""
        torch = self._torch
        R = int(logit.numel())
        loss = torch.empty((), dtype=torch.float32, device=self.device)
        dlogit = torch.empty(R, dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib.b200_pointwise_loss(_lib.ptr(logit), _lib.ptr(labels_d), R, 0, 0.25, 2.0, _lib.ptr(loss),
                                                _lib.ptr(dlogit), _lib.ptr(self._lws), self._lws.numel(),
                                                _lib.current_stream()))
        return loss, dlogit

    def _col_sum(self, X, out, wrow=None):
        X2 = X if X.dim() == 2 else X.view(-1, 1)
        _lib.check(_lib.lib.b200_col_reduce(_lib.ptr(X2), X2.stride(0), X2.shape[0], X2.shape[1], _lib.ptr(wrow), None, 0,
                                            _lib.ptr(out), _lib.current_stream()))

    def _axpy(self, y, x):
        """y += x (same shapes, contiguous) on the library's kernel."""
        _lib.check(_lib.lib.b200_axpy(_lib.ptr(y), _lib.ptr(x), 1.0, y.numel(), _lib.current_stream()))

    def _normalize(self, x):
        """(L2-normalised copy of the rows of x, x) with ``norm_embed``, else (x, None)."""
        if not self.norm_embed:
            return x, None
        y = x.clone()
        _lib.check(_lib.lib.b200_l2_normalize_rows(_lib.ptr(y), y.stride(0), y.shape[0], y.shape[1],
                                                   _lib.current_stream()))
        return y, x

    def _normalize_backward(self, dy, pre):
        """d loss / d x of ``_normalize`` (in place of dy) given its second result."""
        if pre is not None:
            _lib.check(_lib.lib.b200_l2_normalize_backward(_lib.ptr(pre), pre.stride(0), _lib.ptr(dy), dy.stride(0),
                                                           pre.shape[0], pre.shape[1], _lib.ptr(dy), dy.stride(0),
                                                           _lib.current_stream()))
        return dy

    # ---- one multi_head_attention layer (layers/attention.py:67-138; layout in weights_io) of ``self.scheme`` with
    # ``self.H`` heads: variables ``{prefix}{query, key, value, attention_output | output}`` held as 2-D views; the
    # model's attention core comes in as callables ----------------------------------------------------------------
    def _init_mha(self, prefix, lw, d_in, D, layer):
        """Adds one layer's variables from its raw ``lw`` of input width d_in and width D; ``ValueError`` if a shape
        differs."""
        want = _mha_tf_shapes(self.scheme, d_in, D, self.H)
        got = {n: tuple(np.shape(lw[n])) for n in want}
        if got != want:
            raise ValueError(f"{type(self).__name__} layer {layer}: attention shapes {got}, expected {want}")
        for n, shp in _mha_2d(self.scheme, d_in, D).items():
            self.params[prefix + n] = self._var(lw[n], shp)

    def _mha_forward(self, prefix, X, core, kv=None):
        """q = X Wq, k = S Wk, v = (k if legacy else S) Wv with S = ``kv`` (cross attention) or X, (o, lse) =
        core(q, k, v), then o Wo; returns (o Wo, cache)."""
        wq, wk, wv, wo = (self.params[prefix + n] for n in _MHA_VARS[self.scheme])
        src = X if kv is None else kv
        q = linear(X, wq.t().contiguous(), None, ACT_NONE, cache_split=False)
        k = linear(src, wk.t().contiguous(), None, ACT_NONE, cache_split=False)
        v = linear(k if self.scheme == "legacy" else src, wv.t().contiguous(), None, ACT_NONE, cache_split=False)
        o, lse = core(q, k, v)
        return (linear(o, wo.t().contiguous(), None, ACT_NONE, cache_split=False),
                dict(x=X, kv=kv, q=q, k=k, v=v, o=o, lse=lse))

    def _mha_backward(self, prefix, c, dY, core_backward):
        """Backward of ``_mha_forward`` given dY = d loss / d (o Wo): the four weight gradients ADDED into ``grads``;
        returns d loss / d X, or (d loss / d X, d loss / d kv) for cross attention.  ``core_backward(c, dO)`` returns
        (dq, dk, dv)."""
        p, g = self.params, self.grads
        nq, nk, nv, no = (prefix + n for n in _MHA_VARS[self.scheme])
        src = c["x"] if c["kv"] is None else c["kv"]
        g[no] += _weight_grad(dY, c["o"]).t()                     # dWo = O^T dY
        dO = linear(dY, p[no], None, ACT_NONE, cache_split=False)  # dO = dY Wo^T
        dq, dk, dv = core_backward(c, dO)
        if self.scheme == "legacy":                                # V = Kproj Wv': Wk gets the V path too
            g[nv] += _weight_grad(dv, c["k"]).t()                 # dWv' = Kproj^T dV
            self._axpy(dk, linear(dv, p[nv], None, ACT_NONE, cache_split=False))
        g[nq] += _weight_grad(dq, c["x"]).t()
        g[nk] += _weight_grad(dk, src).t()
        dX = linear(dq, p[nq], None, ACT_NONE, cache_split=False)
        dS = dX if c["kv"] is None else None
        if dS is None:
            dS = linear(dk, p[nk], None, ACT_NONE, cache_split=False)
        else:
            self._axpy(dS, linear(dk, p[nk], None, ACT_NONE, cache_split=False))
        if self.scheme == "keras":
            g[nv] += _weight_grad(dv, src).t()
            self._axpy(dS, linear(dv, p[nv], None, ACT_NONE, cache_split=False))
        return dX if c["kv"] is None else (dX, dS)

    def _export_mha(self, prefix, d_in, D):
        """One layer's variables in their raw shapes (the inverse of ``_init_mha``)."""
        return {n: self.params[prefix + n].cpu().numpy().reshape(shp)
                for n, shp in _mha_tf_shapes(self.scheme, d_in, D, self.H).items()}

    def _dense1_forward(self, h, prefix="out_"):
        """Logits of the Dense(1) head (variables ``{prefix}kernel`` [C], ``{prefix}bias`` [1]) on ``h`` [R, C]."""
        torch = self._torch
        p = self.params
        R = int(h.shape[0])
        logit = torch.empty(R, dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib.b200_concat_dense(_lib.ptr(h), h.stride(0), h.shape[1], None, 0, 0, None, 0, 0,
                                              _lib.ptr(p[prefix + "kernel"]), 0.0, R, _lib.ptr(logit),
                                              _lib.current_stream()))
        logit += p[prefix + "bias"]                 # device scalar add (the bias is a trainable variable)
        return logit

    def _dense1_backward(self, h, logit, labels_d, prefix="out_", dlogit=None):
        """Loss and the Dense(1) head's gradients (written into ``grads``); returns (loss, d loss / d h).  Given
        ``dlogit`` (d loss / d logit of a loss taken elsewhere) only the gradients are formed and the loss is None."""
        p, g = self.params, self.grads
        R = int(h.shape[0])
        loss = None
        if dlogit is None:
            loss, dlogit = self._loss(logit, labels_d)
        self._col_sum(h, g[prefix + "kernel"], dlogit)
        self._col_sum(dlogit, g[prefix + "bias"])
        # d h = dlogit (x) kernel: the Dense(1) transposed, on the library's dense kernel (din = 1)
        dh = linear(dlogit.view(R, 1), p[prefix + "kernel"].view(-1, 1), None, False, cache_split=False)
        return loss, dh

    def _items(self, items_d):
        """(rows of ``item_embeds`` [B, d] normalised with norm_embed, their pre-normalisation rows or None, biases
        [B] of ``item_biases``)."""
        torch = self._torch
        p, B = self.params, int(items_d.numel())
        d = int(p["item_embeds"].shape[1])
        I0 = torch.empty((B, d), dtype=torch.float32, device=self.device)
        b = torch.empty((B, 1), dtype=torch.float32, device=self.device)
        st = _lib.current_stream()
        _lib.check(_lib.lib.b200_gather_rows(_lib.ptr(p["item_embeds"]), d, d, _lib.ptr(items_d), B, _lib.ptr(I0), d,
                                             st))
        _lib.check(_lib.lib.b200_gather_rows(_lib.ptr(p["item_biases"]), 1, 1, _lib.ptr(items_d), B, _lib.ptr(b), 1,
                                             st))
        I, pre = self._normalize(I0)
        return I, pre, b.view(-1)

    def _score(self, u, I, b):
        """<u_r, I_r> + b_r per row."""
        torch = self._torch
        B = int(u.shape[0])
        rows = torch.arange(B, dtype=torch.int64, device=self.device)
        s = torch.empty(B, dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib.b200_gather_dot(_lib.ptr(u), u.stride(0), _lib.ptr(rows), _lib.ptr(I), I.stride(0),
                                            _lib.ptr(rows), B, int(u.shape[1]), 0, 0.0, 0.0, _lib.ptr(s),
                                            _lib.current_stream()))
        _lib.check(_lib.lib.b200_axpy(_lib.ptr(s), _lib.ptr(b), 1.0, B, _lib.current_stream()))
        return s

    def _device_counters(self):
        """The Adam step counter and step size live on the device (allocated outside any graph capture)."""
        if getattr(self, "_step_dev", None) is None:
            torch = self._torch
            self._step_dev = torch.full((1,), int(self.t), dtype=torch.int64, device=self.device)
            self._lr_t = torch.zeros(1, dtype=torch.float32, device=self.device)

    def _adam_update(self):
        """TF-Adam over every variable with the step counter and the bias-corrected step size ON THE DEVICE
        (``b200_adam_begin_step`` / ``b200_adam_dense_dev``): the same launches work eagerly and inside a captured
        CUDA graph."""
        self._device_counters()
        lib, st = _lib.lib, _lib.current_stream()
        reg = float(getattr(self, "reg", 0.0) or 0.0)
        if reg > 0.0:             # L2 on the embedding / linear tables only (the variables built with regularizer=reg)
            for k in self.reg_vars:
                if k in self.params:
                    _lib.check(lib.b200_axpy(_lib.ptr(self.grads[k]), _lib.ptr(self.params[k]), 2.0 * reg,
                                             self.params[k].numel(), st))
        decay_steps = int(getattr(self, "decay_steps", 0) or 0)
        _lib.check(lib.b200_adam_begin_step(_lib.ptr(self._step_dev), self.lr, BETA1, BETA2,
                                            float(getattr(self, "decay_rate", 0.96)), decay_steps, _lib.ptr(self._lr_t),
                                            st))
        for k, v in self.params.items():
            _lib.check(lib.b200_adam_dense_dev(_lib.ptr(v), _lib.ptr(self.m[k]), _lib.ptr(self.v[k]),
                                               _lib.ptr(self.grads[k]), v.numel(), _lib.ptr(self._lr_t), BETA1, BETA2,
                                               self.epsilon, st))
        self.t += 1

    def step_graph(self, *inputs):
        """``step`` captured ONCE per input shape into a CUDA graph and replayed — a step is ~100 small launches
        (gather, BN, dense layers, reductions, one Adam launch per variable), launch-bound when issued one by one
        from Python.  Inputs are copied into static buffers; the returned loss is a static device scalar, valid
        until the next replay.  Semantics are those of ``step``."""
        torch = self._torch
        graphs = self.__dict__.setdefault("_graphs", {})
        key = tuple(None if x is None else (tuple(x.shape), x.dtype) for x in inputs)
        ent = graphs.get(key)
        if ent is None:
            self._device_counters()
            static = [None if x is None else x.detach().clone() for x in inputs]
            graph = torch.cuda.CUDAGraph()
            launches0 = int(_lib.lib.b200_launch_count())
            with torch.cuda.graph(graph):
                loss = self.step(*static)          # recorded, not executed (the host counter `t` advances here)
            ent = graphs[key] = (graph, static, loss, int(_lib.lib.b200_launch_count()) - launches0)
        else:
            for s_, x in zip(ent[1], inputs):
                if s_ is not None:
                    s_.copy_(x, non_blocking=True)
            self.t += 1
        ent[0].replay()
        self.graph_launches_per_step = ent[3]      # this library's kernels inside one replay
        return ent[2]


class FMTrainer(_Trainer):
    """Owns the FM variables of ``fm.py`` (scope "embedding" tables + the two Dense(1) heads + BN),
    their Adam slots and gradient buffers.  ``weights`` uses the inference layout of
    ``feat_models.FM`` / ``oracle.tf_models.make_fm_weights``."""

    linear_tables = True

    def __init__(self, spec, weights, use_bn=True, lr=1e-3, epsilon=1e-5, device=None):
        super().__init__(spec, weights, use_bn, lr, epsilon, device)
        self._buf = {}

    def _init_params(self, weights):
        p, K = self.params, self.K
        p["lin_kernel"] = self._var(weights["lin_kernel"], -1)
        p["lin_bias"] = self._var(weights["lin_bias"], 1)
        p["pw_kernel"] = self._var(weights["pw_kernel"], -1)
        p["pw_bias"] = self._var(weights["pw_bias"], 1)
        if self.use_bn:
            bn = weights.get("fm_bn")
            one, zero = np.ones(K, np.float32), np.zeros(K, np.float32)
            p["bn_gamma"] = self._var(bn["gamma"] if bn else one)
            p["bn_beta"] = self._var(bn["beta"] if bn else zero)
            self.moving_mean = self._var(bn["mean"] if bn else zero)
            self.moving_var = self._var(bn["var"] if bn else one)

    def _buffers(self, R):
        torch = self._torch
        if self._buf.get("R") != R:
            K, dev, f32 = self.K, self.device, torch.float32
            nb = int(_lib.lib.b200_fm_head_backward_workspace_bytes(R, K))
            self._buf = dict(
                R=R, S=torch.empty((R, K), dtype=f32, device=dev), Q=torch.empty((R, K), dtype=f32, device=dev),
                pw=torch.empty((R, K), dtype=f32, device=dev), y=torch.empty((R, K), dtype=f32, device=dev),
                dpw=torch.empty((R, K), dtype=f32, device=dev), lin=torch.empty(R, dtype=f32, device=dev),
                z=torch.empty(R, dtype=f32, device=dev), logit=torch.empty(R, dtype=f32, device=dev),
                dlogit=torch.empty(R, dtype=f32, device=dev), loss=torch.empty((), dtype=f32, device=dev),
                mean=torch.empty(K, dtype=f32, device=dev), var=torch.empty(K, dtype=f32, device=dev),
                ws=torch.empty(nb, dtype=torch.uint8, device=dev), lws=self._lws)
        return self._buf

    def forward(self, users_d, items_d):
        """Training-mode logits of the batch (batch statistics in the BN); fills the step buffers."""
        lib, st, p, K = _lib.lib, _lib.current_stream(), self.params, self.K
        R = int(users_d.numel())
        b = self._buffers(R)
        feat_forward(self.spec.layout, self.tables, users_d, items_d, R, pw=b["pw"], lin=b["lin"],
                     lin_kernel=p["lin_kernel"], ssum=b["S"], sqsum=b["Q"])
        y = b["pw"]
        if self.use_bn:
            _lib.check(lib.b200_bn_train_forward(
                _lib.ptr(b["pw"]), K, R, K, _lib.ptr(p["bn_gamma"]), _lib.ptr(p["bn_beta"]), BN_EPS, BN_MOMENTUM,
                _lib.ptr(b["y"]), K, _lib.ptr(b["mean"]), _lib.ptr(b["var"]), _lib.ptr(self.moving_mean),
                _lib.ptr(self.moving_var), st))
            y = b["y"]
        _lib.check(lib.b200_fm_head_forward(_lib.ptr(y), K, R, K, _lib.ptr(p["pw_kernel"]), _lib.ptr(p["pw_bias"]),
                                            _lib.ptr(b["lin"]), _lib.ptr(p["lin_bias"]), _lib.ptr(b["z"]),
                                            _lib.ptr(b["logit"]), st))
        return b["logit"]

    def step(self, users_d, items_d, labels_d):
        """One optimisation step on (users, items, labels) device tensors; returns the device loss."""
        torch = self._torch
        lib, st, p, g, K = _lib.lib, _lib.current_stream(), self.params, self.grads, self.K
        users_d = users_d.to(torch.int64).contiguous()
        items_d = items_d.to(torch.int64).contiguous()
        labels_d = labels_d.to(torch.float32).contiguous()
        R = int(users_d.numel())
        self.forward(users_d, items_d)
        b = self._buf
        _lib.check(lib.b200_pointwise_loss(_lib.ptr(b["logit"]), _lib.ptr(labels_d), R, 0, 0.25, 2.0, _lib.ptr(b["loss"]),
                                           _lib.ptr(b["dlogit"]), _lib.ptr(b["lws"]), b["lws"].numel(), st))
        bn = self.use_bn
        _lib.check(lib.b200_fm_head_backward(
            _lib.ptr(b["dlogit"]), _lib.ptr(b["z"]), _lib.ptr(b["pw"]), K, R, K,
            _lib.ptr(b["mean"]) if bn else None, _lib.ptr(b["var"]) if bn else None,
            _lib.ptr(p["bn_gamma"]) if bn else None, _lib.ptr(p["bn_beta"]) if bn else None, BN_EPS,
            _lib.ptr(p["pw_kernel"]), _lib.ptr(b["dpw"]), K, _lib.ptr(g["pw_kernel"]), _lib.ptr(g["pw_bias"]),
            _lib.ptr(g["bn_gamma"]) if bn else None, _lib.ptr(g["bn_beta"]) if bn else None,
            _lib.ptr(g["lin_bias"]), _lib.ptr(b["ws"]), b["ws"].numel(), st))
        feat_backward(self.spec.layout, self.tables, users_d, items_d, R, g, dpw=b["dpw"], S=b["S"],
                      dlogit=b["dlogit"], lin_kernel=p["lin_kernel"])
        self._adam_update()
        return b["loss"]

    def export_weights(self):
        """Inference weight dict (feat_models.FM layout) with the BN moving statistics."""
        p = self.params
        w = self._export_tables()
        w.update(lin_kernel=p["lin_kernel"].cpu().numpy(), lin_bias=np.float32(p["lin_bias"].cpu().numpy()[0]),
                 pw_kernel=p["pw_kernel"].cpu().numpy(), pw_bias=np.float32(p["pw_bias"].cpu().numpy()[0]))
        if self.use_bn:
            w["fm_bn"] = dict(gamma=p["bn_gamma"].cpu().numpy(), beta=p["bn_beta"].cpu().numpy(),
                              mean=self.moving_mean.cpu().numpy(), var=self.moving_var.cpu().numpy())
        return w


class _StackTrainer(_Trainer):
    """Shared pieces of the trainers built on ``dense_nn`` stacks (``libreco/layers/dense.py:12-49``, training mode):
    parameters ``{prefix}Wt{i}`` [dout, din], ``{prefix}b{i}``, ``{prefix}bn{j}_gamma|beta`` (+ moving statistics
    ``moving[f"{prefix}bn{j}"]``), forward / backward of one stack on the library kernels."""

    def _init_stack(self, prefix, mlp):
        """Adds one stack's variables (trainable layout = transposed kernel [dout, din], what the GEMM reads);
        returns its number of Dense layers."""
        p = self.params
        n = len(mlp["kernels"])
        for i in range(n):
            p[f"{prefix}Wt{i}"] = self._var(np.ascontiguousarray(np.asarray(mlp["kernels"][i]).T))
            p[f"{prefix}b{i}"] = self._var(mlp["biases"][i])
        if self.use_bn:
            for j, bn in enumerate([mlp.get("bn_in")] + list(mlp.get("bns") or [])):
                p[f"{prefix}bn{j}_gamma"] = self._var(bn["gamma"])
                p[f"{prefix}bn{j}_beta"] = self._var(bn["beta"])
                self.moving[f"{prefix}bn{j}"] = (self._var(bn["mean"]), self._var(bn["var"]))
        return n

    def _bn_forward(self, x, name):
        torch = self._torch
        p = self.params
        R, C = x.shape
        y = torch.empty_like(x)
        mean = torch.empty(C, dtype=torch.float32, device=self.device)
        var = torch.empty(C, dtype=torch.float32, device=self.device)
        mm, mv = self.moving[name]
        _lib.check(_lib.lib.b200_bn_train_forward(
            _lib.ptr(x), x.stride(0), R, C, _lib.ptr(p[f"{name}_gamma"]), _lib.ptr(p[f"{name}_beta"]), BN_EPS,
            BN_MOMENTUM, _lib.ptr(y), y.stride(0), _lib.ptr(mean), _lib.ptr(var), _lib.ptr(mm), _lib.ptr(mv),
            _lib.current_stream()))
        return y, (mean, var)

    def _bn_backward(self, dy, x, stats, name, relu_mask):
        torch = self._torch
        p, g = self.params, self.grads
        R, C = x.shape
        dx = torch.empty_like(x)
        ws = torch.empty(C * 2, dtype=torch.float64, device=self.device)
        _lib.check(_lib.lib.b200_bn_train_backward(
            _lib.ptr(dy), dy.stride(0), _lib.ptr(x), x.stride(0), R, C, _lib.ptr(stats[0]), _lib.ptr(stats[1]),
            _lib.ptr(p[f"{name}_gamma"]), BN_EPS, 1 if relu_mask else 0, _lib.ptr(dx), dx.stride(0),
            _lib.ptr(g[f"{name}_gamma"]), _lib.ptr(g[f"{name}_beta"]), _lib.ptr(ws), ws.numel() * 8,
            _lib.current_stream()))
        return dx

    def _stack_forward(self, prefix, n_layers, x, act=ACT_RELU):
        """BN(input) -> [Dense -> act -> BN] x (L-1) -> Dense with batch statistics; returns (out, cache).  ``act``:
        relu (fused into the dense kernel) or swish (``dense_nn(..., activation=swish)``; its pre-activation is kept
        for the backward)."""
        p = self.params
        c = dict(concat=x, bn_stats={}, dense_in=[], act_out=[], pre_act=[])
        a = x
        if self.use_bn:
            a, c["bn_stats"][0] = self._bn_forward(a, f"{prefix}bn0")
        for i in range(n_layers):
            last = i == n_layers - 1
            c["dense_in"].append(a)
            fused = last or act == ACT_RELU
            a = linear(a, p[f"{prefix}Wt{i}"], p[f"{prefix}b{i}"], ACT_RELU if not last and fused else ACT_NONE,
                       cache_split=False)                                    # weights change every step
            if not last:
                if not fused:
                    c["pre_act"].append(a)
                    a = self._activation(a, act)
                c["act_out"].append(a)
                if self.use_bn:
                    a, c["bn_stats"][i + 1] = self._bn_forward(a, f"{prefix}bn{i + 1}")
        return a, c

    def _activation(self, z, act):
        y = self._torch.empty_like(z)
        _lib.check(_lib.lib.b200_activation_forward(_lib.ptr(z), z.numel(), act, _lib.ptr(y), _lib.current_stream()))
        return y

    def _stack_backward(self, prefix, n_layers, c, da, act=ACT_RELU):
        """Gradients of the stack's variables ADDED into ``self.grads``; returns d loss / d input.  ``act`` as in
        ``_stack_forward``: a relu output masks the BN backward (or b200_relu_backward), a swish block runs the BN
        backward unmasked and then b200_activation_backward from the saved pre-activation."""
        torch = self._torch
        lib, st, p, g = _lib.lib, _lib.current_stream(), self.params, self.grads
        da = da.contiguous()
        for i in range(n_layers - 1, -1, -1):
            if i != n_layers - 1:
                a_out = c["act_out"][i]
                relu = act == ACT_RELU
                if self.use_bn:
                    da = self._bn_backward(da, a_out, c["bn_stats"][i + 1], f"{prefix}bn{i + 1}", relu)
                elif relu:
                    dh = torch.empty_like(da)
                    _lib.check(lib.b200_relu_backward(_lib.ptr(da), _lib.ptr(a_out), da.numel(), _lib.ptr(dh), st))
                    da = dh
                if not relu:
                    z = c["pre_act"][i]
                    dz = torch.empty_like(da)
                    _lib.check(lib.b200_activation_backward(_lib.ptr(da), _lib.ptr(z), da.numel(), act, _lib.ptr(dz),
                                                            st))
                    da = dz
            x = c["dense_in"][i]
            da = da.contiguous()
            # dWt [dout, din] = dY^T X ; db = column sums of dY ; dX = dY Wt
            g[f"{prefix}Wt{i}"] += _weight_grad(da, x)
            self._col_sum(da, g[f"{prefix}b{i}"])
            da = linear(da, p[f"{prefix}Wt{i}"].t().contiguous(), None, False, cache_split=False)
        return self._bn_backward(da, c["concat"], c["bn_stats"][0], f"{prefix}bn0", False) if self.use_bn else da

    def _export_stack(self, prefix, n):
        p = self.params
        mlp = dict(kernels=[p[f"{prefix}Wt{i}"].t().contiguous().cpu().numpy() for i in range(n)],
                   biases=[p[f"{prefix}b{i}"].cpu().numpy() for i in range(n)])
        if self.use_bn:
            def bn(j):
                mm, mv = self.moving[f"{prefix}bn{j}"]
                return dict(gamma=p[f"{prefix}bn{j}_gamma"].cpu().numpy(), beta=p[f"{prefix}bn{j}_beta"].cpu().numpy(),
                            mean=mm.cpu().numpy(), var=mv.cpu().numpy())
            mlp["bn_in"] = bn(0)
            mlp["bns"] = [bn(i + 1) for i in range(n - 1)]
        return mlp


class DeepFMTrainer(_StackTrainer):
    """DeepFM training step on the device: ``libreco/algorithms/deepfm.py:143-175`` with
    ``dense_nn`` in training mode (``libreco/layers/dense.py:12-49``: BN(input) -> [Dense -> ReLU ->
    BN] x (L-1) -> Dense, no dropout = the reference's default), mean sigmoid CE, TF-Adam.

    The Dense layers run on the library's own GEMM kernels (``feat_models.linear``: wgmma 3xTF32 or
    exact-fma SIMT) — forward ``Y = X Wt^T + b``, backward ``dX = dY Wt`` and ``dWt = dY^T X`` are the
    same kernel on transposed operands.  ``weights`` uses the inference layout of
    ``feat_models.DeepFM`` / ``oracle.tf_models.make_deepfm_weights``."""

    linear_tables = True

    def __init__(self, spec, weights, use_bn=True, lr=1e-3, epsilon=1e-5, device=None):
        super().__init__(spec, weights, use_bn, lr, epsilon, device)

    def _init_params(self, weights):
        p = self.params
        for k in ("lin_kernel", "out_kernel"):
            p[k] = self._var(weights[k], -1)
        for k in ("lin_bias", "out_bias"):
            p[k] = self._var(weights[k], 1)
        self.n_layers = self._init_stack("", weights["mlp"])
        self.H = int(p[f"Wt{self.n_layers - 1}"].shape[0])

    def forward(self, users_d, items_d):
        torch = self._torch
        p, K = self.params, self.K
        R = int(users_d.numel())
        f32, dev = torch.float32, self.device
        concat = torch.empty((R, self.F * K), dtype=f32, device=dev)
        pw, lin = torch.empty((R, K), dtype=f32, device=dev), torch.empty(R, dtype=f32, device=dev)
        S, Q = torch.empty((R, K), dtype=f32, device=dev), torch.empty((R, K), dtype=f32, device=dev)
        feat_forward(self.spec.layout, self.tables, users_d, items_d, R, concat=concat, pw=pw, lin=lin,
                     lin_kernel=p["lin_kernel"], ssum=S, sqsum=Q)
        a, c = self._stack_forward("", self.n_layers, concat)
        logit = torch.empty(R, dtype=f32, device=dev)
        _lib.check(_lib.lib.b200_deepfm_head_forward(
            _lib.ptr(lin), _lib.ptr(p["lin_bias"]), _lib.ptr(pw), K, K, _lib.ptr(a), a.stride(0), self.H,
            _lib.ptr(p["out_kernel"]), _lib.ptr(p["out_bias"]), R, _lib.ptr(logit), _lib.current_stream()))
        c.update(R=R, users=users_d, items=items_d, pw=pw, lin=lin, S=S, deep=a, logit=logit)
        self._cache = c
        return logit

    def backward(self, labels_d):
        """Loss + every gradient buffer filled (before the optimiser); returns the device loss."""
        torch = self._torch
        p, g, K, H = self.params, self.grads, self.K, self.H
        c = self._cache
        R, f32, dev = c["R"], torch.float32, self.device
        loss, dlogit = self._loss(c["logit"], labels_d)
        dlin = torch.empty(R, dtype=f32, device=dev)
        dpw = torch.empty((R, K), dtype=f32, device=dev)
        da = torch.empty((R, H), dtype=f32, device=dev)
        _lib.check(_lib.lib.b200_deepfm_head_backward(_lib.ptr(dlogit), _lib.ptr(p["out_kernel"]), K, H, R,
                                                      _lib.ptr(dlin), _lib.ptr(dpw), K, _lib.ptr(da), H,
                                                      _lib.current_stream()))
        # out_kernel = [w_lin | w_pw (K) | w_deep (H)]: weighted column sums with the row weights dlogit
        gk = g["out_kernel"]
        lin_full = c["lin"] + p["lin_bias"]                      # elementwise add of a device scalar (plumbing)
        self._col_sum(lin_full.view(R, 1), gk[0:1], dlogit)
        self._col_sum(c["pw"], gk[1:1 + K], dlogit)
        self._col_sum(c["deep"], gk[1 + K:], dlogit)
        self._col_sum(dlogit.view(R, 1), g["out_bias"])
        self._col_sum(dlin.view(R, 1), g["lin_bias"])
        dconcat = self._stack_backward("", self.n_layers, c, da)
        feat_backward(self.spec.layout, self.tables, c["users"], c["items"], R, g, dpw=dpw, S=c["S"], dconcat=dconcat,
                      dlogit=dlin, lin_kernel=p["lin_kernel"])
        return loss

    def step(self, users_d, items_d, labels_d):
        torch = self._torch
        users_d = users_d.to(torch.int64).contiguous()
        items_d = items_d.to(torch.int64).contiguous()
        labels_d = labels_d.to(torch.float32).contiguous()
        self.forward(users_d, items_d)
        loss = self.backward(labels_d)
        self._adam_update()
        self._cache = None
        return loss

    def export_weights(self):
        p = self.params
        w = self._export_tables()
        w.update(lin_kernel=p["lin_kernel"].cpu().numpy(), lin_bias=np.float32(p["lin_bias"].cpu().numpy()[0]),
                 out_kernel=p["out_kernel"].cpu().numpy(), out_bias=np.float32(p["out_bias"].cpu().numpy()[0]))
        w["mlp"] = self._export_stack("", self.n_layers)
        return w


class TwoTowerTrainer(_StackTrainer):
    """TwoTower training step on the device, in-batch softmax loss (the reference's default):
    ``libreco/algorithms/two_tower.py:306-346,400-410`` (both towers, ``dense_nn`` in training mode, optional
    ``tf.linalg.l2_normalize``), ``tfops/loss.py:71-75`` + ``two_tower.py:458-479`` (``U V^T / temperature -
    log Q``, optional accidental-hit mask, mean sparse softmax CE with the diagonal as labels), TF-Adam.

        per tower: K1 gather (b200_feat_forward, tower layout) -> BN/Dense/ReLU stack (b200_bn_train_forward,
        b200_linear_*) -> b200_l2_normalize_rows;  S = U V^T (b200_linear_*) -> b200_softmax_inbatch_loss
        (S becomes dS) -> dU = dS V, dV = dS^T U -> b200_l2_normalize_backward -> stack backward ->
        b200_feat_backward (scatter into the SHARED sparse / dense tables) -> b200_adam_dense

    ``weights``: layout of ``feat_models.TwoTower`` / ``synthetic.make_two_tower_weights``.  ``temperature``
    must be positive (the learned-temperature variant, ``temperature <= 0``, is not built)."""

    def __init__(self, spec, weights, use_bn=True, norm_embed=False, temperature=1.0, remove_accidental_hits=False,
                 lr=1e-3, epsilon=1e-5, device=None):
        if temperature <= 0:
            raise ValueError("learned temperature (temperature <= 0) is not supported")
        self.norm_embed = bool(norm_embed)
        self.temperature, self.remove_hits = float(temperature), bool(remove_accidental_hits)
        super().__init__(spec, weights, use_bn, lr, epsilon, device)

    def _init_params(self, weights):
        self.n_layers = {which: self._init_stack(f"{which}_", weights[f"{which}_tower"]) for which in ("user", "item")}

    # ---- one tower ----------------------------------------------------------------------------------
    def tower_forward(self, which, ids_d):
        torch = self._torch
        n = int(ids_d.numel())
        L, pos = self.spec.side(which)
        x = torch.empty((n, len(pos) * self.K), dtype=torch.float32, device=self.device)
        feat_forward(L, self.tables, ids_d, ids_d, n, concat=x)
        a, c = self._stack_forward(f"{which}_", self.n_layers[which], x)
        c["ids"] = ids_d
        c["out"], c["pre_norm"] = self._normalize(a)
        return c

    def tower_backward(self, which, c, da):
        n = int(c["ids"].numel())
        da = self._normalize_backward(da.contiguous(), c["pre_norm"])
        dconcat = self._stack_backward(f"{which}_", self.n_layers[which], c, da)
        feat_backward(self.spec.side(which)[0], self.tables, c["ids"], c["ids"], n, self.grads, dconcat=dconcat)

    # ---- loss / step --------------------------------------------------------------------------------
    def forward_backward(self, users_d, items_d, correction_d=None):
        """Loss (device scalar) with every gradient buffer filled.  ``correction_d``: item_corrections[items]
        of the batch (``two_tower.py:425-435``, ``tf_feed_dicts.py:121-122``) or None (use_correction=False)."""
        torch = self._torch
        cu = self.tower_forward("user", users_d)
        ci = self.tower_forward("item", items_d)
        U, V = cu["out"], ci["out"]
        B = int(U.shape[0])
        S = linear(U, V, None, False, cache_split=False)          # [B, B] = U V^T
        loss = torch.empty((), dtype=torch.float32, device=self.device)
        corr = correction_d.to(torch.float32).contiguous() if correction_d is not None else None
        _lib.check(_lib.lib.b200_softmax_inbatch_loss(_lib.ptr(S), S.stride(0), B, self.temperature, _lib.ptr(corr),
                                                      _lib.ptr(items_d) if self.remove_hits else None, 1, _lib.ptr(loss),
                                                      _lib.ptr(self._lws), self._lws.numel(), _lib.current_stream()))
        dU = linear(S, V.t().contiguous(), None, False, cache_split=False)
        dV = linear(S.t().contiguous(), U.t().contiguous(), None, False, cache_split=False)
        self.tower_backward("user", cu, dU)
        self.tower_backward("item", ci, dV)
        self._last = (U, V)
        return loss

    def step(self, users_d, items_d, correction_d=None):
        torch = self._torch
        users_d = users_d.to(torch.int64).contiguous()
        items_d = items_d.to(torch.int64).contiguous()
        loss = self.forward_backward(users_d, items_d, correction_d)
        self._adam_update()
        self._last = None
        return loss

    def export_weights(self):
        w = self._export_tables()
        for which in ("user", "item"):
            w[f"{which}_tower"] = self._export_stack(f"{which}_", self.n_layers[which])
        w["user_dense_cols"] = list(self.spec.user_dense_cols)
        w["item_dense_cols"] = list(self.spec.item_dense_cols)
        return w


class _SeqTrainer(_StackTrainer):
    """YouTubeRanking and DIN: the F field blocks and a sequence block -> one ``dense_nn`` stack -> Dense(1), mean
    sigmoid CE, TF-Adam.  The batch carries one behaviour sequence per ROW (``seqs`` [R, T] padded with ``n_items``,
    ``lens`` [R]; ``libreco/batch/sequence.py:75-91``).  A subclass fills the sequence block of the stack input
    (``forward``) and sends its gradient back (``backward``).  ``mlp_act``: the activation of the ``dense_nn``
    stack.  The item feature table G (``combine_seq_features``, concat mode) of the models that attend over item
    features is built by ``_build_G`` and its gradient folded back by ``_fold_dG``."""

    mlp_act = ACT_RELU

    def __init__(self, spec, weights, use_bn=True, lr=1e-3, epsilon=1e-5, device=None):
        super().__init__(spec, weights, use_bn, lr, epsilon, device)

    def _init_params(self, weights):
        self.n_layers = self._init_stack("", weights["mlp"])
        self.params["out_kernel"] = self._var(weights["out_kernel"], -1)
        self.params["out_bias"] = self._var(weights["out_bias"], 1)

    def _init_item_table(self):
        """Columns of G: the item embedding, then one block per item sparse field (index columns of the spec) and
        per item dense field (value x that field's embedding)."""
        torch = self._torch
        sp = self.spec
        self._is = [sp.is_[:, j].to(torch.int64).contiguous() for j in range(sp.is_.shape[1])] if sp.is_ is not None else []
        self._id = [sp.id_[:, j].contiguous() for j in range(sp.id_.shape[1])] if sp.id_ is not None else []
        self._id_cols = list(sp.item_dense_cols)
        self.Kp = self.K * (1 + len(self._is) + len(self._id))

    def _build_G(self):
        torch = self._torch
        p, K, st = self.params, self.K, _lib.current_stream()
        n = self.n_items + 1
        G = torch.empty((n, self.Kp), dtype=torch.float32, device=self.device)
        G[:, :K].copy_(p["item_embeds"][:n])
        off = K
        for idx in self._is:
            blk = G[:, off:off + K]
            _lib.check(_lib.lib.b200_gather_rows(_lib.ptr(p["sparse_embeds"]), K, K, _lib.ptr(idx), n, _lib.ptr(blk),
                                                 G.stride(0), st))
            off += K
        for vals, col in zip(self._id, self._id_cols):
            G[:, off:off + K] = vals[:, None] * p["dense_embeds"][col][None, :]
            off += K
        return G

    def _fold_dG(self, dG):
        """dG [n_items+1, K'] back into the tables G was built from: the item-embedding block added, sparse blocks
        through b200_scatter_add_rows, dense blocks through b200_col_reduce."""
        lib, st, g, K = _lib.lib, _lib.current_stream(), self.grads, self.K
        n = self.n_items + 1
        g["item_embeds"][:n] += dG[:, :K]
        off = K
        for idx in self._is:
            blk = dG[:, off:off + K]
            _lib.check(lib.b200_scatter_add_rows(_lib.ptr(g["sparse_embeds"]), K, K, _lib.ptr(idx), n, _lib.ptr(blk),
                                                 dG.stride(0), st))
            off += K
        for vals, col in zip(self._id, self._id_cols):
            blk = dG[:, off:off + K]
            _lib.check(lib.b200_col_reduce(_lib.ptr(blk), dG.stride(0), n, K, _lib.ptr(vals), None, 0,
                                           _lib.ptr(g["dense_embeds"][col]), st))
            off += K

    def _head_forward(self, x, **cache):
        """Stack + Dense(1) on the filled input ``x``; caches what the backward needs and returns the logits."""
        R = int(x.shape[0])
        h, c = self._stack_forward("", self.n_layers, x, self.mlp_act)
        logit = self._dense1_forward(h)
        c.update(R=R, h=h, logit=logit, **cache)
        self._cache = c
        return logit

    def _head_backward(self, labels_d):
        """Loss, the gradients of the head, the stack and the field tables; returns (loss, d loss / d input)."""
        g, c = self.grads, self._cache
        R = c["R"]
        loss, da = self._dense1_backward(c["h"], c["logit"], labels_d)
        dx = self._stack_backward("", self.n_layers, c, da, self.mlp_act)
        feat_backward(self.spec.layout, self.tables, c["users"], c["items"], R, g, dconcat=dx)
        return loss, dx

    def step(self, users_d, items_d, seqs_d, lens_d, labels_d):
        torch = self._torch
        self.forward(users_d.to(torch.int64).contiguous(), items_d.to(torch.int64).contiguous(),
                     seqs_d.to(torch.int32).contiguous(), lens_d.to(torch.int32).contiguous())
        loss = self.backward(labels_d.to(torch.float32).contiguous())
        self._adam_update()
        self._cache = None
        return loss

    def export_weights(self):
        p = self.params
        w = self._export_tables()
        w["mlp"] = self._export_stack("", self.n_layers)
        w["out_kernel"] = p["out_kernel"].cpu().numpy()
        w["out_bias"] = np.float32(p["out_bias"].cpu().numpy()[0])
        return w


class YouTubeRankingTrainer(_SeqTrainer):
    """YouTubeRanking training step on the device: ``libreco/algorithms/youtube_ranking.py:167-218`` in training
    mode (concat(user, item, pooled behaviour sequence, sparse, dense) -> ``dense_nn`` -> Dense(1)), mean sigmoid
    CE, TF-Adam.

        K1 gather (b200_feat_forward) + b200_seq_pool -> stack forward -> b200_concat_dense -> b200_pointwise_loss
        -> stack backward -> b200_feat_backward (field gradients) + b200_seq_pool_backward (sequence gradient into
        the item-embedding table) -> b200_adam_dense

    Internally the pooled block sits AFTER the F field blocks (the inference engine's layout); the first kernel and
    the input batch-norm are permuted on the way in and out (``feat_models.permute_mlp_input``)."""

    def _init_params(self, weights):
        K, F = self.K, self.F
        self.perm = np.concatenate([np.arange(0, 2 * K), np.arange(3 * K, (F + 1) * K), np.arange(2 * K, 3 * K)])
        super()._init_params(dict(weights, mlp=permute_mlp_input(weights["mlp"], self.perm)))

    def forward(self, users_d, items_d, seqs_d, lens_d):
        torch = self._torch
        K, F = self.K, self.F
        R = int(users_d.numel())
        x = torch.empty((R, (F + 1) * K), dtype=torch.float32, device=self.device)
        feat_forward(self.spec.layout, self.tables, users_d, items_d, R, concat=x)
        rows = torch.arange(R, dtype=torch.int64, device=self.device)
        pooled = x[:, F * K:]
        E = self.params["item_embeds"]
        _lib.check(_lib.lib.b200_seq_pool(_lib.ptr(E), E.stride(0), K, self.n_items, _lib.ptr(seqs_d), seqs_d.stride(0),
                                          _lib.ptr(lens_d), seqs_d.shape[1], _lib.ptr(rows), R, 0, 0, _lib.ptr(pooled),
                                          pooled.stride(0), _lib.current_stream()))
        return self._head_forward(x, users=users_d, items=items_d, seqs=seqs_d, lens=lens_d, rows=rows)

    def backward(self, labels_d):
        K, F = self.K, self.F
        c = self._cache
        loss, dx = self._head_backward(labels_d)
        dpool = dx[:, F * K:]
        ge = self.grads["item_embeds"]
        _lib.check(_lib.lib.b200_seq_pool_backward(_lib.ptr(dpool), dpool.stride(0), K, self.n_items,
                                                   _lib.ptr(c["seqs"]), c["seqs"].stride(0), _lib.ptr(c["lens"]),
                                                   c["seqs"].shape[1], _lib.ptr(c["rows"]), c["R"], _lib.ptr(ge),
                                                   ge.stride(0), _lib.current_stream()))
        return loss

    def export_weights(self):
        w = super().export_weights()
        inv = np.argsort(self.perm)
        w["mlp"]["kernels"][0] = w["mlp"]["kernels"][0][inv]
        if self.use_bn:
            w["mlp"]["bn_in"] = {k: v[inv] for k, v in w["mlp"]["bn_in"].items()}
        return w


class DINTrainer(_SeqTrainer):
    """DIN training step on the device: ``libreco/algorithms/din.py:165-250`` in training mode (paper attention,
    ``libreco/layers/attention.py:28-64``; concat(user, item, sparse, dense, attention output) -> ``dense_nn`` ->
    Dense(1)), mean sigmoid CE, TF-Adam.  One behaviour sequence per ROW (``lens`` [R] >= 1, T <= 64).

        item feature table G = [item emb | its sparse embs | value x dense embs] rebuilt from the CURRENT tables
        (b200_gather_rows per item sparse field) -> K1 gather + b200_din_attention -> stack forward ->
        b200_concat_dense -> b200_pointwise_loss -> stack backward -> b200_feat_backward (field gradients) +
        b200_din_attention_backward (dG + attention weight gradients) -> dG folded back into the tables
        (item-embedding block added, sparse blocks through b200_scatter_add_rows, dense blocks through
        b200_col_reduce) -> b200_adam_dense_dev
    """

    def _init_params(self, weights):
        super()._init_params(weights)
        p = self.params
        att = weights["attention"]
        p["att_k1"] = self._var(att["k1"])
        p["att_b1"] = self._var(att["b1"])
        p["att_k2"] = self._var(att["k2"], -1)
        p["att_b2"] = self._var(att["b2"], 1)
        self._b2_host = float(np.asarray(att["b2"]).reshape(-1)[0])      # Dense(1) bias enters the kernels by value
        self._init_item_table()

    def forward(self, users_d, items_d, seqs_d, lens_d):
        torch = self._torch
        p, K, F, Kp = self.params, self.K, self.F, self.Kp
        R = int(users_d.numel())
        T = int(seqs_d.shape[1])
        G = self._build_G()
        x = torch.empty((R, F * K + Kp), dtype=torch.float32, device=self.device)
        feat_forward(self.spec.layout, self.tables, users_d, items_d, R, concat=x)
        rows = torch.arange(R, dtype=torch.int64, device=self.device)
        att_out = x[:, F * K:]
        # the Dense(1) bias shifts every logit of a row alike: the softmax ignores it, its gradient is exactly 0 and
        # TF-Adam never moves it — the initial value is passed by value, no device read
        b2 = self._b2_host
        _lib.check(_lib.lib.b200_din_attention(
            _lib.ptr(G), G.stride(0), Kp, _lib.ptr(items_d), _lib.ptr(seqs_d), seqs_d.stride(0), _lib.ptr(lens_d), T,
            _lib.ptr(rows), R, 0, 0, _lib.ptr(p["att_k1"]), _lib.ptr(p["att_b1"]), _lib.ptr(p["att_k2"]), b2,
            _lib.ptr(att_out), att_out.stride(0), _lib.current_stream()))
        return self._head_forward(x, T=T, users=users_d, items=items_d, seqs=seqs_d, lens=lens_d, rows=rows, G=G, b2=b2)

    def backward(self, labels_d):
        torch = self._torch
        lib, st, p, g, K, F, Kp = _lib.lib, _lib.current_stream(), self.params, self.grads, self.K, self.F, self.Kp
        c = self._cache
        R = c["R"]
        loss, dx = self._head_backward(labels_d)
        # ---- attention backward: gradient of the item feature table + the attention weights
        G = c["G"]
        n = self.n_items + 1
        dG = torch.zeros((n, Kp), dtype=torch.float32, device=self.device)
        datt = dx[:, F * K:]
        _lib.check(lib.b200_din_attention_backward(
            _lib.ptr(G), G.stride(0), Kp, _lib.ptr(c["items"]), _lib.ptr(c["seqs"]), c["seqs"].stride(0),
            _lib.ptr(c["lens"]), c["T"], _lib.ptr(c["rows"]), R, _lib.ptr(p["att_k1"]), _lib.ptr(p["att_b1"]),
            _lib.ptr(p["att_k2"]), c["b2"], _lib.ptr(datt), datt.stride(0), _lib.ptr(dG), dG.stride(0),
            _lib.ptr(g["att_k1"]), _lib.ptr(g["att_b1"]), _lib.ptr(g["att_k2"]), _lib.ptr(g["att_b2"]), st))
        self._fold_dG(dG)
        return loss

    def export_weights(self):
        p = self.params
        w = super().export_weights()
        w["attention"] = dict(k1=p["att_k1"].cpu().numpy(), b1=p["att_b1"].cpu().numpy(), k2=p["att_k2"].cpu().numpy(),
                              b2=np.float32(p["att_b2"].cpu().numpy()[0]))
        return w


class TransformerTrainer(_SeqTrainer):
    """Transformer training step on the device: ``libreco/algorithms/transformer.py:203-339`` in training mode (no
    dropout), mean sigmoid CE, TF-Adam.  One behaviour sequence per ROW (``seqs`` [R, T], ``lens`` [R], clamped to
    [1, T] as the training collator gives them).

        G (the item feature table, concat mode, from the CURRENT tables) -> X = [G[seq_t] || pos_t] over R*T rows
        (b200_gather_rows) -> per layer: b200_rms_norm_forward -> Q / K / V projections (b200_linear_*) ->
        b200_transformer_attention_forward (masked) -> output projection + residual -> rms -> W1 ->
        b200_activation_forward (gelu) -> W2 + residual -> rms_last -> target attention of [rms_item(G[item]) || 1]
        (b200_transformer_target_attention) -> K1 gather + swish ``dense_nn`` -> Dense(1) -> b200_pointwise_loss
        -> the reverse (b200_transformer_target_attention_backward, b200_rms_norm_backward + b200_col_reduce for
        the scales, b200_transformer_attention_backward, b200_activation_backward, the dense kernels for every
        projection) -> dX[:, :K'] and dq[:K'] scattered into dG (b200_scatter_add_rows), the trainable positions'
        gradient a column reduction -> dG folded into the tables as DIN does -> b200_feat_backward ->
        b200_adam_dense_dev

    ``weights``: the RAW variables of either graph, as ``synthetic.make_transformer_weights`` makes them (the
    tables, ``tfm_scheme``, ``tfm_layers``, ``rms_last``, ``rms_item``, ``positional_encoding`` when the positions
    are trainable — absent, the sinusoidal table is a constant —, ``num_heads``, ``use_causal_mask``, ``mlp``,
    ``out_kernel``, ``out_bias``).  keras ``query`` / ``key`` / ``value`` [D, H, hd] and ``attention_output``
    [H, hd, D] are held as [D, D]; legacy ``value`` acts on the PROJECTED keys, so Wk is trained through both of its
    paths.  ``export_weights`` returns the same raw layout.  ``reg`` applies to the embedding tables only.

    Raises ``ValueError`` before anything is launched for shapes outside the kernels' envelope (T <= 64,
    D = K' + K <= 128, 1..4 layers, heads dividing D), ``feat_agg_mode="elementwise"`` (its layer-norm backward is
    not built) and multi-sparse fields with a combiner other than "normal" (the pooling backward is not built)."""

    mlp_act = ACT_SWISH

    def __init__(self, spec, weights, use_bn=True, lr=1e-3, epsilon=1e-5, device=None):
        from .feat_models import _spec_get

        g = _spec_get(spec) if not isinstance(spec, FeatSpec) else (lambda k, d=None: d)
        if weights.get("feat_agg_mode", "concat") != "concat":
            raise ValueError("TransformerTrainer: only feat_agg_mode \"concat\" trains; the layer-norm backward of "
                             "\"elementwise\" is not built")
        if g("multi_sparse_combine_info") is not None and weights.get("multi_sparse_combiner", "sqrtn") != "normal":
            raise ValueError("TransformerTrainer: multi-sparse fields need the combiner \"normal\"; the pooling "
                             "backward is not built")
        self._combiner = weights.get("multi_sparse_combiner")
        super().__init__(spec, weights, use_bn, lr, epsilon, device)
        self._sin = {}

    def _init_params(self, weights):
        from .feat_models import TRANSFORMER_MAX_D, TRANSFORMER_MAX_LAYERS, TRANSFORMER_MAX_T

        super()._init_params(weights)
        self._init_item_table()
        p, K, F, Kp = self.params, self.K, self.F, self.Kp
        D = self.D = Kp + K
        H = self.H = int(weights["num_heads"])
        self.scheme = weights["tfm_scheme"]
        _check_mha_scheme(self.scheme, "TransformerTrainer")
        layers = list(weights["tfm_layers"])
        if D > TRANSFORMER_MAX_D or not 1 <= len(layers) <= TRANSFORMER_MAX_LAYERS or H < 1 or D % H:
            raise ValueError(f"TransformerTrainer: width D = {D} (item features {Kp} + positions {K}), {len(layers)} "
                             f"layers, {H} heads outside D <= {TRANSFORMER_MAX_D}, 1..{TRANSFORMER_MAX_LAYERS} layers, "
                             f"heads dividing D")
        want = dict(rms_att=(D,), rms_ffn=(D,), ffn1=(D, 4 * D), ffn2=(4 * D, D))
        for l, lw in enumerate(layers):
            self._init_mha(f"tfm{l}_", lw, D, D, l)
            got = {n: tuple(np.shape(lw[n])) for n in want}
            if got != want:
                raise ValueError(f"TransformerTrainer layer {l}: shapes {got}, expected {want}")
            for n in want:
                p[f"tfm{l}_{n}"] = self._var(lw[n], want[n])
        self.n_tfm = len(layers)
        for n, shp in (("rms_last", D), ("rms_item", Kp)):
            if np.size(weights[n]) != shp:
                raise ValueError(f"TransformerTrainer: {n} has {np.size(weights[n])} entries, expected {shp}")
            p[n] = self._var(weights[n], -1)
        pos = weights.get("positional_encoding")
        self.T_pos = None
        if pos is not None:
            T = np.shape(pos)[0]
            if np.ndim(pos) != 2 or np.shape(pos)[1] != K or not 1 <= T <= TRANSFORMER_MAX_T:
                raise ValueError(f"TransformerTrainer: positional table of shape {np.shape(pos)}, expected (T, {K}) "
                                 f"with T <= {TRANSFORMER_MAX_T}")
            p["positional_encoding"] = self._var(pos)
            self.T_pos = T
        n_in = np.shape(weights["mlp"]["kernels"][0])[0]
        if n_in != F * K + D:
            raise ValueError(f"TransformerTrainer: the first MLP layer takes {n_in} inputs, expected F*K + D = "
                             f"{F}*{K} + {D}")
        self.causal = bool(weights.get("use_causal_mask", False))

    def _positions(self, T):
        """The positional table [T, K] of this batch: the trainable variable, or the constant sinusoidal table
        (uploaded once per T, outside any graph capture)."""
        from .feat_models import TRANSFORMER_MAX_T, sinusoidal_positions

        if not 1 <= T <= TRANSFORMER_MAX_T:
            raise ValueError(f"TransformerTrainer: sequence length {T} outside 1..{TRANSFORMER_MAX_T}")
        if self.T_pos is not None:
            if T != self.T_pos:
                raise ValueError(f"TransformerTrainer: sequences of length {T}, the positional table has {self.T_pos} "
                                 f"rows")
            return self.params["positional_encoding"]
        if T not in self._sin:
            self._sin[T] = _dev(sinusoidal_positions(T, self.K), self.device, self._torch.float32)
        return self._sin[T]

    def _rms(self, x, name, out=None):
        """(rms_norm(x) with the scale variable ``name``, rstd [rows]); written into ``out`` when given."""
        torch = self._torch
        R, D = x.shape
        y = out if out is not None else torch.empty((R, D), dtype=torch.float32, device=self.device)
        rstd = torch.empty(R, dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib.b200_rms_norm_forward(_lib.ptr(x), x.stride(0), R, D, _lib.ptr(self.params[name]),
                                                  _lib.ptr(y), y.stride(0), _lib.ptr(rstd), _lib.current_stream()))
        return y, rstd

    def _rms_backward(self, dy, x, rstd, name):
        """d input of ``_rms``; the scale's gradient sum_r rstd dy x is ADDED into ``grads[name]``."""
        lib, st = _lib.lib, _lib.current_stream()
        R, D = x.shape
        dx = self._torch.empty((R, D), dtype=self._torch.float32, device=self.device)
        _lib.check(lib.b200_rms_norm_backward(_lib.ptr(dy), dy.stride(0), _lib.ptr(x), x.stride(0), _lib.ptr(rstd), R, D,
                                              _lib.ptr(self.params[name]), _lib.ptr(dx), dx.stride(0), st))
        _lib.check(lib.b200_col_reduce(_lib.ptr(dy), dy.stride(0), R, D, _lib.ptr(rstd), _lib.ptr(x), x.stride(0),
                                       _lib.ptr(self.grads[name]), st))
        return dx

    def forward(self, users_d, items_d, seqs_d, lens_d):
        """Training-mode logits of the batch (batch statistics in the BN); caches what the backward needs."""
        torch = self._torch
        lib, st, p = _lib.lib, _lib.current_stream(), self.params
        K, F, Kp, D, H = self.K, self.F, self.Kp, self.D, self.H
        R, T = int(seqs_d.shape[0]), int(seqs_d.shape[1])
        pos = self._positions(T)
        hd = D // H
        scale = float(np.float32(1.0 / np.sqrt(hd)))
        f32, dev = torch.float32, self.device
        lens = lens_d.clamp(1, T).to(torch.int32).contiguous()
        G = self._build_G()
        RT = R * T
        seq_idx = seqs_d.reshape(-1).to(torch.int64)
        X = torch.empty((RT, D), dtype=f32, device=dev)
        _lib.check(lib.b200_gather_rows(_lib.ptr(G), G.stride(0), Kp, _lib.ptr(seq_idx), RT, _lib.ptr(X), D, st))
        X.view(R, T, D)[:, :, Kp:] = pos                       # broadcast copy of the positions (plumbing)

        def core(q, k, v):
            o = torch.empty((RT, D), dtype=f32, device=dev)
            lse = torch.empty(R * H * T, dtype=f32, device=dev)
            _lib.check(lib.b200_transformer_attention_forward(
                _lib.ptr(q), q.stride(0), _lib.ptr(k), k.stride(0), _lib.ptr(v), v.stride(0), _lib.ptr(lens), R, T, H,
                hd, int(self.causal), scale, _lib.ptr(o), o.stride(0), _lib.ptr(lse), st))
            return o, lse

        layers = []
        for l in range(self.n_tfm):
            h1, r1 = self._rms(X, f"tfm{l}_rms_att")
            a, mha = self._mha_forward(f"tfm{l}_", h1, core)
            self._axpy(a, X)
            h2, r2 = self._rms(a, f"tfm{l}_rms_ffn")
            z = linear(h2, p[f"tfm{l}_ffn1"].t().contiguous(), None, ACT_NONE, cache_split=False)
            gz = self._activation(z, ACT_GELU)
            y = linear(gz, p[f"tfm{l}_ffn2"].t().contiguous(), None, ACT_NONE, cache_split=False)
            self._axpy(y, a)
            layers.append(dict(x=X, r1=r1, mha=mha, a=a, h2=h2, r2=r2, z=z, gz=gz))
            X = y
        S, rl = self._rms(X, "rms_last")
        # the target query [rms_item(G[item]) || 1..1]
        Gi = torch.empty((R, Kp), dtype=f32, device=dev)
        _lib.check(lib.b200_gather_rows(_lib.ptr(G), G.stride(0), Kp, _lib.ptr(items_d), R, _lib.ptr(Gi), Kp, st))
        Q = torch.empty((R, D), dtype=f32, device=dev)
        Q[:, Kp:] = 1.0
        _, ri = self._rms(Gi, "rms_item", out=Q[:, :Kp])
        x = torch.empty((R, F * K + D), dtype=f32, device=dev)
        feat_forward(self.spec.layout, self.tables, users_d, items_d, R, concat=x)
        su = x[:, F * K:]
        rows = torch.arange(R, dtype=torch.int64, device=dev)
        slots = rows.to(torch.int32)
        _lib.check(lib.b200_transformer_target_attention(_lib.ptr(Q), Q.stride(0), _lib.ptr(S), T, D, _lib.ptr(lens),
                                                         _lib.ptr(slots), _lib.ptr(rows), R, 0, 0, _lib.ptr(su),
                                                         su.stride(0), st))
        return self._head_forward(x, users=users_d, items=items_d, T=T, lens=lens, seq_idx=seq_idx, layers=layers,
                                  XL=X, S=S, rl=rl, Gi=Gi, ri=ri, Q=Q)

    def backward(self, labels_d):
        """Loss + every gradient buffer filled (before the optimiser); returns the device loss."""
        torch = self._torch
        lib, st, p, g = _lib.lib, _lib.current_stream(), self.params, self.grads
        K, F, Kp, D, H = self.K, self.F, self.Kp, self.D, self.H
        c = self._cache
        R, T = c["R"], c["T"]
        RT, hd = R * T, D // H
        scale = float(np.float32(1.0 / np.sqrt(hd)))
        f32, dev = torch.float32, self.device
        loss, dx = self._head_backward(labels_d)
        dsu = dx[:, F * K:]
        dq = torch.empty((R, D), dtype=f32, device=dev)
        dX = torch.empty((RT, D), dtype=f32, device=dev)
        _lib.check(lib.b200_transformer_target_attention_backward(
            _lib.ptr(c["Q"]), c["Q"].stride(0), _lib.ptr(c["S"]), T, D, _lib.ptr(c["lens"]), _lib.ptr(dsu),
            dsu.stride(0), R, _lib.ptr(dq), dq.stride(0), _lib.ptr(dX), st))
        n = self.n_items + 1
        dG = torch.zeros((n, Kp), dtype=f32, device=dev)
        dGi = self._rms_backward(dq[:, :Kp], c["Gi"], c["ri"], "rms_item")      # the ones padding is a constant
        _lib.check(lib.b200_scatter_add_rows(_lib.ptr(dG), Kp, Kp, _lib.ptr(c["items"]), R, _lib.ptr(dGi), Kp, st))
        dX = self._rms_backward(dX, c["XL"], c["rl"], "rms_last")

        def core_backward(m, dO):
            dqh, dk, dv = (torch.empty((RT, D), dtype=f32, device=dev) for _ in range(3))
            _lib.check(lib.b200_transformer_attention_backward(
                _lib.ptr(m["q"]), m["q"].stride(0), _lib.ptr(m["k"]), m["k"].stride(0), _lib.ptr(m["v"]),
                m["v"].stride(0), _lib.ptr(m["o"]), m["o"].stride(0), _lib.ptr(m["lse"]), _lib.ptr(dO), dO.stride(0),
                _lib.ptr(c["lens"]), R, T, H, hd, int(self.causal), scale, _lib.ptr(dqh), _lib.ptr(dk), _lib.ptr(dv), D,
                st))
            return dqh, dk, dv

        for l in range(self.n_tfm - 1, -1, -1):
            a_ = c["layers"][l]
            n1, n2 = f"tfm{l}_ffn1", f"tfm{l}_ffn2"
            # y = a + gelu(rms_ffn(a) W1) W2
            g[n2] += _weight_grad(dX, a_["gz"]).t()
            dgz = linear(dX, p[n2], None, ACT_NONE, cache_split=False)
            dz = torch.empty_like(dgz)
            _lib.check(lib.b200_activation_backward(_lib.ptr(dgz), _lib.ptr(a_["z"]), dz.numel(), ACT_GELU, _lib.ptr(dz),
                                                    st))
            g[n1] += _weight_grad(dz, a_["h2"]).t()
            dh2 = linear(dz, p[n1], None, ACT_NONE, cache_split=False)
            da = self._rms_backward(dh2, a_["a"], a_["r2"], f"tfm{l}_rms_ffn")
            self._axpy(da, dX)
            # a = x + MHA(rms_att(x))
            dh1 = self._mha_backward(f"tfm{l}_", a_["mha"], da, core_backward)
            dXn = self._rms_backward(dh1, a_["x"], a_["r1"], f"tfm{l}_rms_att")
            self._axpy(dXn, da)
            dX = dXn
        # X = [G[seq_t] || pos_t]: the item block into dG, the positions' gradient a column reduction over the rows
        _lib.check(lib.b200_scatter_add_rows(_lib.ptr(dG), Kp, Kp, _lib.ptr(c["seq_idx"]), RT, _lib.ptr(dX), D, st))
        if self.T_pos is not None:
            dpos = torch.zeros(T * D, dtype=f32, device=dev)
            _lib.check(lib.b200_col_reduce(_lib.ptr(dX), T * D, R, T * D, None, None, 0, _lib.ptr(dpos), st))
            g["positional_encoding"] += dpos.view(T, D)[:, Kp:]
        self._fold_dG(dG)
        return loss

    def step_graph(self, users_d, items_d, seqs_d, lens_d, labels_d):
        self._positions(int(seqs_d.shape[1]))       # the sinusoidal table is uploaded before any capture
        return super().step_graph(users_d, items_d, seqs_d, lens_d, labels_d)

    def export_weights(self):
        """The raw variables in the scheme they came in (``weights_io.transformer_weights`` makes the inference
        dict, ``weights_io.transformer_tf_variables`` the reference's variable names)."""
        p, D, H = self.params, self.D, self.H
        w = super().export_weights()
        layers = [dict(self._export_mha(f"tfm{l}_", D, D), **{n: p[f"tfm{l}_{n}"].cpu().numpy()
                                                              for n in ("rms_att", "rms_ffn", "ffn1", "ffn2")})
                  for l in range(self.n_tfm)]
        w.update(tfm_scheme=self.scheme, tfm_layers=layers, rms_last=p["rms_last"].cpu().numpy(),
                 rms_item=p["rms_item"].cpu().numpy(), num_heads=H, use_causal_mask=self.causal,
                 feat_agg_mode="concat", out_kernel=w["out_kernel"].reshape(-1, 1),
                 out_bias=np.asarray(w["out_bias"], dtype=np.float32).reshape(1))
        if self.T_pos is not None:
            w["positional_encoding"] = p["positional_encoding"].cpu().numpy()
        if self._combiner is not None:
            w["multi_sparse_combiner"] = self._combiner
        return w


class AutoIntTrainer(_Trainer):
    """AutoInt training step on the device: ``libreco/algorithms/autoint.py:146-168`` in training mode (the fields
    [user, item, sparse.., dense..] stacked into X [F, K], L layers of ``multi_head_attention(X, X)``
    (``libreco/layers/attention.py:67-125``, optionally ``X + mha(X)``), Flatten, Dense(1)), mean sigmoid CE,
    TF-Adam.  The graph has no BN and no dropout; ``reg`` applies to the embedding tables only.

        K1 gather (b200_feat_forward, X as [R*F, K]) -> per layer: Q, K, V projections over R*F rows
        (b200_linear_*) -> b200_autoint_attention_forward -> output projection (b200_linear_*) -> residual add
        (b200_axpy) -> b200_concat_dense -> b200_pointwise_loss -> the reverse, with
        b200_autoint_attention_backward for the attention core and the dense kernels for every projection's input
        and weight gradient -> b200_feat_backward (scatter into the tables) -> b200_adam_dense_dev

    ``weights``: the RAW variables of either graph, as ``synthetic.make_autoint_weights`` makes them (the tables,
    ``autoint_scheme``, ``autoint_mha``, ``num_heads``, ``use_residual``, ``out_kernel``, ``out_bias``).  Each
    scheme trains its own variables: keras ``query`` / ``key`` / ``value`` [K, H, hd] (held as [K, D]) and
    ``attention_output`` [H, hd, K] (held as [D, K]); legacy ``query`` / ``key`` [K, D], ``value`` [D, D]
    applied to the projected keys (V = (X Wk) Wv', so Wk is trained through both of its paths) and ``output``
    [D, K].  ``export_weights`` returns the same raw layout and scheme.

    Multi-sparse fields must use the combiner "normal" (every member its own field): the pooling backward is not
    built.  Shapes outside the attention kernels' envelope (F <= 130, K <= 64, H * hd <= 64, 1..4 layers) raise
    ``ValueError`` before anything is launched."""

    def __init__(self, spec, weights, lr=1e-3, epsilon=1e-5, device=None):
        from .feat_models import _spec_get

        g = _spec_get(spec) if not isinstance(spec, FeatSpec) else (lambda k, d=None: d)
        if g("multi_sparse_combine_info") is not None and weights.get("multi_sparse_combiner", "sqrtn") != "normal":
            raise ValueError("AutoIntTrainer: multi-sparse fields need the combiner \"normal\"; the pooling backward "
                             "is not built")
        super().__init__(spec, weights, False, lr, epsilon, device)

    def _init_params(self, weights):
        from .feat_models import AUTOINT_MAX_D, AUTOINT_MAX_F, AUTOINT_MAX_K, AUTOINT_MAX_LAYERS

        p, K, F = self.params, self.K, self.F
        self.scheme = weights["autoint_scheme"]
        H = self.H = int(weights["num_heads"])
        self.use_residual = bool(weights.get("use_residual", True))
        self._combiner = weights.get("multi_sparse_combiner")
        mha = list(weights["autoint_mha"])
        _check_mha_scheme(self.scheme, "AutoIntTrainer")
        if K > AUTOINT_MAX_K or F > AUTOINT_MAX_F or not 1 <= len(mha) <= AUTOINT_MAX_LAYERS or H < 1:
            raise ValueError(f"AutoIntTrainer: K {K}, F {F}, {len(mha)} layers, {H} heads outside K <= "
                             f"{AUTOINT_MAX_K}, F <= {AUTOINT_MAX_F}, 1..{AUTOINT_MAX_LAYERS} layers, heads >= 1")
        self.head_dims = []
        for l, lw in enumerate(mha):
            D = int(np.prod(np.shape(lw["query"])[1:]))
            if D % H or not 1 <= D <= AUTOINT_MAX_D:
                raise ValueError(f"AutoIntTrainer layer {l}: width {D} with {H} heads, expected a multiple of the "
                                 f"heads <= {AUTOINT_MAX_D}")
            self._init_mha(f"mha{l}_", lw, K, D, l)
            self.head_dims.append(D // H)
        if np.size(weights["out_kernel"]) != F * K:
            raise ValueError(f"AutoIntTrainer: out_kernel has {np.size(weights['out_kernel'])} entries, expected "
                             f"F*K = {F}*{K}")
        p["out_kernel"] = self._var(weights["out_kernel"], -1)
        p["out_bias"] = self._var(weights["out_bias"], 1)

    def forward(self, users_d, items_d):
        """Training-mode logits of the batch; caches what the backward needs."""
        torch = self._torch
        K, F, H = self.K, self.F, self.H
        R = int(users_d.numel())
        f32, dev = torch.float32, self.device
        x = torch.empty((R, F * K), dtype=f32, device=dev)
        feat_forward(self.spec.layout, self.tables, users_d, items_d, R, concat=x)
        X = x.view(R * F, K)

        def core(q, k, v, hd):
            o = torch.empty((R * F, H * hd), dtype=f32, device=dev)
            lse = torch.empty(R * H * F, dtype=f32, device=dev)
            _lib.check(_lib.lib.b200_autoint_attention_forward(
                _lib.ptr(q), q.stride(0), _lib.ptr(k), k.stride(0), _lib.ptr(v), v.stride(0), R, F, H, hd,
                float(1.0 / np.sqrt(hd)), _lib.ptr(o), o.stride(0), _lib.ptr(lse), _lib.current_stream()))
            return o, lse

        layers = []
        for l, hd in enumerate(self.head_dims):
            y, a = self._mha_forward(f"mha{l}_", X, functools.partial(core, hd=hd))
            if self.use_residual:
                self._axpy(y, X)
            layers.append(a)
            X = y
        h = X.view(R, F * K)
        logit = self._dense1_forward(h)
        self._cache = dict(R=R, users=users_d, items=items_d, layers=layers, h=h, logit=logit)
        return logit

    def backward(self, labels_d):
        """Loss + every gradient buffer filled (before the optimiser); returns the device loss."""
        torch = self._torch
        K, F, H = self.K, self.F, self.H
        c = self._cache
        R = c["R"]
        loss, dh = self._dense1_backward(c["h"], c["logit"], labels_d)

        def core_backward(a, dO, hd):
            D = H * hd
            dq, dk, dv = (torch.empty((R * F, D), dtype=torch.float32, device=self.device) for _ in range(3))
            _lib.check(_lib.lib.b200_autoint_attention_backward(
                _lib.ptr(a["q"]), a["q"].stride(0), _lib.ptr(a["k"]), a["k"].stride(0), _lib.ptr(a["v"]),
                a["v"].stride(0), _lib.ptr(a["o"]), a["o"].stride(0), _lib.ptr(a["lse"]), _lib.ptr(dO), dO.stride(0),
                R, F, H, hd, float(1.0 / np.sqrt(hd)), _lib.ptr(dq), _lib.ptr(dk), _lib.ptr(dv), D,
                _lib.current_stream()))
            return dq, dk, dv

        dX = dh.view(R * F, K)
        for l in range(len(self.head_dims) - 1, -1, -1):
            dXn = self._mha_backward(f"mha{l}_", c["layers"][l], dX,
                                     functools.partial(core_backward, hd=self.head_dims[l]))
            if self.use_residual:
                self._axpy(dXn, dX)
            dX = dXn
        feat_backward(self.spec.layout, self.tables, c["users"], c["items"], R, self.grads, dconcat=dX.view(R, F * K))
        return loss

    def step(self, users_d, items_d, labels_d):
        """One optimisation step on (users, items, labels) device tensors; returns the device loss."""
        torch = self._torch
        self.forward(users_d.to(torch.int64).contiguous(), items_d.to(torch.int64).contiguous())
        loss = self.backward(labels_d.to(torch.float32).contiguous())
        self._adam_update()
        self._cache = None
        return loss

    def export_weights(self):
        """The raw variables in the scheme they came in (``weights_io.autoint_weights`` makes the inference dict)."""
        p, H = self.params, self.H
        w = self._export_tables()
        mha = [self._export_mha(f"mha{l}_", self.K, H * hd) for l, hd in enumerate(self.head_dims)]
        w.update(autoint_scheme=self.scheme, autoint_mha=mha, num_heads=H, use_residual=self.use_residual,
                 out_kernel=p["out_kernel"].cpu().numpy().reshape(-1, 1), out_bias=p["out_bias"].cpu().numpy().reshape(1))
        if self._combiner is not None:
            w["multi_sparse_combiner"] = self._combiner
        return w


UNIQUE_MAX_SAMPLED = 65536      # B200_UNIQUE_MAX_SAMPLED: the candidate sampler's envelope
RETRIEVAL_LOSSES = {"sampled_softmax": 0, "nce": 1}


class YouTubeRetrievalTrainer(_StackTrainer):
    """YouTubeRetrieval training step on the device: ``libreco/algorithms/youtube_retrieval.py:169-260`` in training
    mode (user vector = ``dense_nn(concat(sqrtn-pooled history over seq_embeds_var, user sparse embeddings, user dense
    value x embedding))``) and ``YoutubeRetrievalTrainer._build_train_ops`` (``libreco/training/tf_trainer.py:162-245``):
    S = ``num_sampled_per_batch`` (or ``batch_size``) distinct candidates from TensorFlow's unique uniform /
    log-uniform sampler, ``tf.nn.sampled_softmax_loss`` or ``tf.nn.nce_loss`` over ``item_embeds_var`` /
    ``item_bias_var`` with accidental hits removed and log Q subtracted, mean over the batch, optional L2 ``reg``
    on all five tables, TF-Adam.

        b200_unique_candidates (ids [S] + num_tries, both on the device; the draw stream is keyed by the device
        Adam step) -> b200_seq_pool + K1 over the user-side fields (no id field) -> stack forward ->
        [b200_l2_normalize_rows] -> b200_gather_rows (sampled and label rows) -> logits U W_s^T (b200_linear_*) and
        true logits (b200_gather_dot) -> b200_sampled_class_loss (logits become d loss / d logits) ->
        dU = dL W_s + dtrue W_label, dW_s = dL^T U (b200_linear_*) -> [b200_l2_normalize_backward] ->
        b200_scatter_add_rows (sampled rows, label rows, biases; labels repeat) + b200_col_reduce (sampled-bias
        column sums) -> stack backward -> b200_seq_pool_backward + b200_feat_backward -> b200_adam_dense_dev

    ``weights``: the layout of ``feat_models.YouTubeRetrieval`` (``seq_embeds`` [n_items, K], ``item_embeds``
    [n_items, H], ``item_biases`` [n_items], ``sparse_embeds``, ``dense_embeds``, ``mlp`` ending in H units).  A
    batch is (users, label items, one history per row ``seqs`` [B, T] padded with ``n_items``, ``lens`` [B]); a row
    at position 0 of its user's history has ``lens`` 1 and the pad id (``b200_interacted_seqs``), which pools to
    the zero vector of the reference's empty history and sends no gradient.  With ``norm_embed`` the user vectors
    and the gathered item rows are L2-normalised (only gathered rows get gradients, so this is the reference's
    normalisation of the whole table).  Raises ``ValueError`` before any launch for an unknown ``loss_type``, S
    outside 1..min(n_items, 65536), or multi-sparse fields with a combiner other than "normal"."""

    embed_table = "seq_embeds"
    reg_vars = _REG_VARS + ("seq_embeds", "item_biases")

    def __init__(self, spec, weights, loss_type="sampled_softmax", batch_size=256, num_sampled_per_batch=None,
                 sampler="uniform", norm_embed=False, use_bn=True, lr=1e-3, epsilon=1e-5, seed=42, device=None):
        from .feat_models import _spec_get

        if loss_type not in RETRIEVAL_LOSSES:
            raise ValueError(f"YouTubeRetrievalTrainer: loss_type must be one of {sorted(RETRIEVAL_LOSSES)}, "
                             f"got `{loss_type}`")
        g = _spec_get(spec) if not isinstance(spec, FeatSpec) else (lambda k, d=None: d)
        if g("multi_sparse_combine_info") is not None and weights.get("multi_sparse_combiner", "sqrtn") != "normal":
            raise ValueError("YouTubeRetrievalTrainer: multi-sparse fields need the combiner \"normal\"; the pooling "
                             "backward is not built")
        n_items = int(spec.n_items if isinstance(spec, FeatSpec) else g("n_items"))
        S = int(num_sampled_per_batch) if num_sampled_per_batch and num_sampled_per_batch > 0 else int(batch_size)
        if not 1 <= S <= min(n_items, UNIQUE_MAX_SAMPLED):
            raise ValueError(f"YouTubeRetrievalTrainer: num_sampled {S} outside 1..min(n_items = {n_items}, "
                             f"{UNIQUE_MAX_SAMPLED})")
        for k, rows in (("seq_embeds", n_items), ("item_embeds", n_items), ("item_biases", n_items)):
            if np.shape(weights[k])[0] != rows:
                raise ValueError(f"YouTubeRetrievalTrainer: {k} has {np.shape(weights[k])[0]} rows, expected n_items = "
                                 f"{n_items} (no OOV row)")
        self.loss_type, self.loss_kind = loss_type, RETRIEVAL_LOSSES[loss_type]
        self.sampler, self.sampler_kind = sampler, 0 if sampler == "uniform" else 1     # anything else: TF's default
        self.S, self.seed, self.norm_embed = S, int(seed), bool(norm_embed)
        self._combiner = weights.get("multi_sparse_combiner")
        super().__init__(spec, weights, use_bn, lr, epsilon, device)
        torch = self._torch
        self._device_counters()
        self.sampled = torch.empty(S, dtype=torch.int64, device=self.device)
        self.num_tries = torch.empty(1, dtype=torch.int64, device=self.device)
        self._owner = torch.full((self.n_items,), -1, dtype=torch.int32, device=self.device)     # 0xFF bytes: all free

    def _init_params(self, weights):
        p = self.params
        p["seq_embeds"] = self._var(weights["seq_embeds"])
        p["item_biases"] = self._var(weights["item_biases"], -1)
        self.n_layers = self._init_stack("", weights["mlp"])
        self.H = int(p[f"Wt{self.n_layers - 1}"].shape[0])
        if tuple(p["item_embeds"].shape) != (self.n_items, self.H):
            raise ValueError(f"YouTubeRetrievalTrainer: item_embeds {tuple(p['item_embeds'].shape)}, expected "
                             f"(n_items, last hidden units) = ({self.n_items}, {self.H})")

    def sample(self):
        """This step's candidates: device ids [S] (distinct, in draw order) and the device ``num_tries``, drawn from
        (seed, the device Adam step)."""
        _lib.check(_lib.lib.b200_unique_candidates(
            self.sampler_kind, self.n_items, self.S, self.seed, _lib.ptr(self._step_dev), _lib.ptr(self._owner),
            self._owner.numel() * 4, _lib.ptr(self.sampled), _lib.ptr(self.num_tries), _lib.current_stream()))
        return self.sampled, self.num_tries

    def user_forward(self, users_d, seqs_d, lens_d):
        """User vectors [B, H] of the batch (training-mode BN) before any normalisation; returns (U, cache)."""
        torch = self._torch
        K = self.K
        B = int(users_d.numel())
        L, pos = self.spec.side("user", with_id=False)
        x = torch.empty((B, (1 + len(pos)) * K), dtype=torch.float32, device=self.device)
        rows = torch.arange(B, dtype=torch.int64, device=self.device)
        E = self.params["seq_embeds"]
        _lib.check(_lib.lib.b200_seq_pool(_lib.ptr(E), E.stride(0), K, self.n_items, _lib.ptr(seqs_d), seqs_d.stride(0),
                                          _lib.ptr(lens_d), seqs_d.shape[1], _lib.ptr(rows), B, 0, 0, _lib.ptr(x),
                                          x.stride(0), _lib.current_stream()))
        if pos:
            feat_forward(L, self.tables, users_d, users_d, B, concat=x[:, K:])
        U, c = self._stack_forward("", self.n_layers, x)
        c.update(users=users_d, seqs=seqs_d, lens=lens_d, rows=rows, fields=bool(pos))
        return U, c

    def forward_backward(self, users_d, items_d, seqs_d, lens_d):
        """Loss (device scalar) with every gradient buffer filled; the candidates stay in ``sampled`` /
        ``num_tries``."""
        torch = self._torch
        lib, st, p, g, K, H, S = _lib.lib, _lib.current_stream(), self.params, self.grads, self.K, self.H, self.S
        f32, dev = torch.float32, self.device
        B = int(users_d.numel())
        ids, tries = self.sample()
        U0, c = self.user_forward(users_d, seqs_d, lens_d)
        W = p["item_embeds"]
        Ws0 = torch.empty((S, H), dtype=f32, device=dev)
        Wl0 = torch.empty((B, H), dtype=f32, device=dev)
        _lib.check(lib.b200_gather_rows(_lib.ptr(W), W.stride(0), H, _lib.ptr(ids), S, _lib.ptr(Ws0), H, st))
        _lib.check(lib.b200_gather_rows(_lib.ptr(W), W.stride(0), H, _lib.ptr(items_d), B, _lib.ptr(Wl0), H, st))
        U, U_pre = self._normalize(U0)
        Ws, Ws_pre = self._normalize(Ws0)
        Wl, Wl_pre = self._normalize(Wl0)
        rows = c["rows"]
        logits = linear(U, Ws, None, False, cache_split=False)                  # [B, S] = U W_s^T
        true = torch.empty(B, dtype=f32, device=dev)
        _lib.check(lib.b200_gather_dot(_lib.ptr(U), U.stride(0), _lib.ptr(rows), _lib.ptr(Wl), Wl.stride(0),
                                       _lib.ptr(rows), B, H, 0, 0.0, 0.0, _lib.ptr(true), st))
        loss = torch.empty((), dtype=f32, device=dev)
        dtrue = torch.empty(B, dtype=f32, device=dev)
        ws = torch.empty(int(lib.b200_sampled_class_loss_workspace_bytes(B, S)), dtype=torch.uint8, device=dev)
        _lib.check(lib.b200_sampled_class_loss(
            self.loss_kind, _lib.ptr(logits), logits.stride(0), B, S, _lib.ptr(true), _lib.ptr(items_d), _lib.ptr(ids),
            _lib.ptr(p["item_biases"]), self.sampler_kind, self.n_items, _lib.ptr(tries), _lib.ptr(loss),
            _lib.ptr(dtrue), _lib.ptr(ws), ws.numel(), st))
        dL = logits                                                              # now d loss / d logits
        # dU = dL W_s + dtrue (x) W_label ; dW_s = dL^T U ; dW_label = dtrue (x) U  (row scalings: elementwise)
        dU = linear(dL, Ws.t().contiguous(), None, False, cache_split=False)
        _lib.check(lib.b200_axpy(_lib.ptr(dU), _lib.ptr(dtrue[:, None] * Wl), 1.0, dU.numel(), st))
        dWs = _weight_grad(dL, U).contiguous()
        dWl = dtrue[:, None] * U
        dU = self._normalize_backward(dU, U_pre)
        dWs = self._normalize_backward(dWs, Ws_pre)
        dWl = self._normalize_backward(dWl, Wl_pre)
        gW, gb = g["item_embeds"], g["item_biases"]
        _lib.check(lib.b200_scatter_add_rows(_lib.ptr(gW), gW.stride(0), H, _lib.ptr(ids), S, _lib.ptr(dWs), H, st))
        _lib.check(lib.b200_scatter_add_rows(_lib.ptr(gW), gW.stride(0), H, _lib.ptr(items_d), B, _lib.ptr(dWl), H, st))
        db = torch.zeros(S, dtype=f32, device=dev)
        self._col_sum(dL, db)
        _lib.check(lib.b200_scatter_add_rows(_lib.ptr(gb), 1, 1, _lib.ptr(ids), S, _lib.ptr(db), 1, st))
        _lib.check(lib.b200_scatter_add_rows(_lib.ptr(gb), 1, 1, _lib.ptr(items_d), B, _lib.ptr(dtrue), 1, st))
        # user tower
        dx = self._stack_backward("", self.n_layers, c, dU)
        ge = g["seq_embeds"]
        _lib.check(lib.b200_seq_pool_backward(_lib.ptr(dx), dx.stride(0), K, self.n_items, _lib.ptr(seqs_d),
                                              seqs_d.stride(0), _lib.ptr(lens_d), seqs_d.shape[1], _lib.ptr(rows), B,
                                              _lib.ptr(ge), ge.stride(0), st))
        if c["fields"]:
            feat_backward(self.spec.side("user", with_id=False)[0], self.tables, users_d, users_d, B, g,
                          dconcat=dx[:, K:])
        return loss

    def step(self, users_d, items_d, seqs_d, lens_d):
        """One optimisation step on (users, label items, histories [B, T], lengths [B]) device tensors; returns the
        device loss."""
        torch = self._torch
        loss = self.forward_backward(users_d.to(torch.int64).contiguous(), items_d.to(torch.int64).contiguous(),
                                     seqs_d.to(torch.int32).contiguous(), lens_d.to(torch.int32).contiguous())
        self._adam_update()
        return loss

    def export_weights(self):
        """The inference layout of ``feat_models.YouTubeRetrieval``."""
        p = self.params
        w = {k: v for k, v in self._export_tables().items() if k != "user_embeds"}
        w.update(seq_embeds=p["seq_embeds"].cpu().numpy(), item_biases=p["item_biases"].cpu().numpy(),
                 mlp=self._export_stack("", self.n_layers))
        if self._combiner is not None:
            w["multi_sparse_combiner"] = self._combiner
        return w


RNN4REC_LOSSES = {"cross_entropy": 0, "focal": 1, "bpr": 2}


class RNN4RecTrainer(_Trainer):
    """RNN4Rec training step on the device: ``libreco/algorithms/rnn4rec.py:151-237`` in training mode (no dropout)
    with ``layers/recurrent.py:4-63``, the losses of ``tfops/loss.py:4-25`` and TF-Adam
    (``training/tf_trainer.py:103-124``).  The user vector of a row is ``Dense(embed_size)(rnn(seq_embeds[seq]))``
    over the row's own sequence:

        b200_gather_rows (the layer-0 input rows) -> b200_rnn_train_forward (the stacked cells, saving per step)
        -> b200_linear_f32 (the head) -> [b200_l2_normalize_rows] -> scores <u, i> + b_i (b200_gather_dot)
        -> b200_pointwise_loss / b200_pairwise_loss -> head and item gradients (b200_scatter_add_rows)
        -> per layer, top down: b200_rnn_backward (dGx, dGh), then dW = X^T dGx, dU = H_prev^T dGh, dX = dGx W^T
        on the dense kernels and the bias / gamma / beta sums on b200_col_reduce -> b200_scatter_add_rows of dX_0
        into seq_embeds -> b200_adam_dense_dev

    ``weights``: the raw variables of either TensorFlow graph (``synthetic.make_rnn4rec_weights``,
    ``weights_io._rnn4rec_raw``).  The Adam variables are the TF variables' elements in the kernel's canonical order
    (gate reordering and the split of the TF1 ``[x, h]`` kernels are permutations): W, U and the bias of every layer,
    bh only for the Keras GRU, gamma / beta only with layer norm, the head, and the three tables.  The TF1 LSTM's
    ``forget_bias = 1.0`` stays folded into the trained f bias; :meth:`export_weights` subtracts it again.

    A pointwise step is ``step(users, items, seqs, lens, labels)`` (``cross_entropy``, ``focal``); a ``bpr`` step is
    ``step(users, items_pos, seqs, lens, items_neg)``: row r scores its sequence against items_pos[r] and
    items_neg[r].  ``seqs`` [B, T] holds item ids padded with the pad row ``n_items`` and ``lens`` [B] the valid
    prefix of each row (a row at history position 0 has len 1 and the pad id).  ``users`` is not read (the model has
    no user table).  With ``norm_embed`` users and items are L2-normalised; the BPR branch, as the reference's
    (``rnn4rec.py:189-195``), scores the normalised items against the UN-normalised user vectors.  ``ValueError``
    before any launch for shapes outside the envelope of ``b200_rnn_encode``, an unknown ``loss_type``,
    ``rnn_type`` or scheme, the rating task, a ``seq_embeds`` row count other than ``n_items + 1`` and a batch whose
    saved state does not fit in the free device memory."""

    embed_table = "item_embeds"
    reg_vars = ("seq_embeds", "item_embeds", "item_biases")

    def __init__(self, spec, weights, loss_type="cross_entropy", norm_embed=False, task="ranking", lr=1e-3,
                 epsilon=1e-5, device=None):
        from .feat_models import RNN_MAX_DIM, RNN_MAX_LAYERS, RNN_MAX_T, _spec_get   # noqa: F401
        from .weights_io import rnn4rec_weights

        if task != "ranking":
            raise ValueError(f"RNN4RecTrainer: task `{task}` is not supported (ranking only)")
        if loss_type not in RNN4REC_LOSSES:
            raise ValueError(f"RNN4RecTrainer: loss_type must be one of {sorted(RNN4REC_LOSSES)}, got `{loss_type}`")
        if weights.get("rnn_scheme") not in ("keras", "legacy"):
            raise ValueError(f"RNN4RecTrainer: unknown rnn_scheme `{weights.get('rnn_scheme')}`")
        if weights.get("rnn_type") not in ("gru", "lstm"):
            raise ValueError(f"RNN4RecTrainer: rnn_type must be gru or lstm, not `{weights.get('rnn_type')}`")
        n_items = int(spec.n_items if isinstance(spec, FeatSpec) else _spec_get(spec)("n_items"))
        if np.shape(weights["seq_embeds"])[0] != n_items + 1:
            raise ValueError(f"RNN4RecTrainer: seq_embeds has {np.shape(weights['seq_embeds'])[0]} rows, expected "
                             f"n_items + 1 = {n_items + 1}")
        self.scheme, self.rnn_type = weights["rnn_scheme"], weights["rnn_type"]
        self.use_layer_norm = bool(weights.get("use_layer_norm", False)) and self.scheme == "keras"
        canon = rnn4rec_weights(weights)
        self.in_dim = int(canon["seq_embeds"].shape[1])
        self.hidden = [int(lw["U"].shape[0]) for lw in canon["rnn_layers"]]
        if not 1 <= len(self.hidden) <= RNN_MAX_LAYERS:
            raise ValueError(f"RNN4RecTrainer: {len(self.hidden)} recurrent layers, supported 1 to {RNN_MAX_LAYERS}")
        if max([self.in_dim] + self.hidden) > RNN_MAX_DIM:
            raise ValueError(f"RNN4RecTrainer: input width {self.in_dim} / hidden sizes {self.hidden} exceed "
                             f"{RNN_MAX_DIM}")
        self.loss_type, self.norm_embed = loss_type, bool(norm_embed)
        self._canon = canon
        super().__init__(spec, canon, False, lr, epsilon, device)
        self._canon = None

    def _init_params(self, weights):
        import ctypes

        torch = self._torch
        p = self.params
        layers = weights["rnn_layers"]
        self.kinds = [int(lw["kind"]) for lw in layers]
        self.acts = [int(lw["act"]) for lw in layers]
        self._kinds = (ctypes.c_int32 * len(layers))(*self.kinds)
        self._hid = (ctypes.c_int32 * len(layers))(*self.hidden)
        self._acts = (ctypes.c_int32 * len(layers))(*self.acts)
        packed, self._offs, d = [], [], self.in_dim
        for lw, H in zip(layers, self.hidden):
            flat = np.concatenate([np.asarray(lw[k], np.float32).reshape(-1)
                                   for k in ("W", "U", "bx", "bh", "gamma", "beta")])
            if flat.size != int(_lib.lib.b200_rnn_layer_floats(int(lw["kind"]), d, H)):
                raise ValueError(f"RNN4RecTrainer: layer of kind {lw['kind']} with input {d} and hidden {H} has "
                                 f"{flat.size} packed floats")
            self._offs.append(sum(a.size for a in packed))
            packed.append(flat)
            d = H
        # the packed weights the kernels read; the variables are views into it
        self.rnn_w = _dev(np.concatenate(packed), self.device, torch.float32).clone()
        d = self.in_dim
        for l, (H, kind) in enumerate(zip(self.hidden, self.kinds)):
            GH = (4 if kind == 2 else 3) * H
            o = self._offs[l]
            views = dict(W=(o, (d, GH)), U=(o + d * GH, (H, GH)), bx=(o + (d + H) * GH, (GH,)),
                         bh=(o + (d + H + 1) * GH, (GH,)), gamma=(o + (d + H + 2) * GH, (H,)),
                         beta=(o + (d + H + 2) * GH + H, (H,)))
            names = ["W", "U", "bx"] + (["bh"] if kind == 0 else []) + (["gamma", "beta"] if self.acts[l] else [])
            for k in names:
                off, shape = views[k]
                p[f"rnn{l}_{k}"] = self.rnn_w[off:off + int(np.prod(shape))].view(shape)
            d = H
        p["seq_embeds"] = self._var(weights["seq_embeds"])
        p["item_biases"] = self._var(weights["item_biases"], -1)
        p["dense_Wt"] = self._var(np.asarray(weights["dense_kernel"]).T.copy())       # [K, H_last]
        p["dense_b"] = self._var(weights["dense_bias"], -1)

    # -- memory ------------------------------------------------------------------------------------------------------
    def saved_bytes_per_row(self, T):
        """Device bytes one batch row keeps for the backward at sequence length T: the saved tensors of every layer
        (h_{t-1}, y_t, the gates, the cell block, and x^ + rstd with layer norm), the layer-0 input rows, and the
        largest layer's transient gradients (dGx, dGh, dX, dLN, dLN x^)."""
        per_t, trans, d = self.in_dim, 0, self.in_dim
        for l, (H, kind) in enumerate(zip(self.hidden, self.kinds)):
            GH = (4 if kind == 2 else 3) * H
            per_t += 3 * H + GH + (H + 1 if self.acts[l] else 0)
            trans = max(trans, GH * (2 if kind == 0 else 1) + d + (2 * H if self.acts[l] else 0))
            d = H
        return 4 * T * (per_t + trans)

    def _check_batch(self, B, T):
        from .feat_models import RNN_MAX_T

        torch = self._torch
        if not 1 <= T <= RNN_MAX_T:
            raise ValueError(f"RNN4RecTrainer: sequence length {T} outside [1, {RNN_MAX_T}]")
        need = B * self.saved_bytes_per_row(T)
        free = torch.cuda.mem_get_info(self.device)[0] + torch.cuda.memory_reserved(self.device) - \
            torch.cuda.memory_allocated(self.device)
        if need > free:
            raise ValueError(f"RNN4RecTrainer: a batch of {B} rows x T = {T} keeps {need} B for the backward, "
                             f"{free} B are free")

    # -- forward -----------------------------------------------------------------------------------------------------
    def encode(self, seqs_d, lens_d):
        """[B, H_last] encoder outputs of the rows ``seqs_d`` [B, T] / ``lens_d`` [B] with the saved state; returns
        (h, cache)."""
        torch = self._torch
        f32, dev = torch.float32, self.device
        B, T = int(seqs_d.shape[0]), int(seqs_d.shape[1])
        rows = torch.arange(B, dtype=torch.int64, device=dev)
        idx = seqs_d.reshape(-1).to(torch.int64)
        E = self.params["seq_embeds"]
        X0 = torch.empty((B * T, self.in_dim), dtype=f32, device=dev)
        _lib.check(_lib.lib.b200_gather_rows(_lib.ptr(E), E.stride(0), self.in_dim, _lib.ptr(idx), B * T,
                                             _lib.ptr(X0), X0.stride(0), _lib.current_stream()))
        saved, ptrs = [], []
        for l, (H, kind) in enumerate(zip(self.hidden, self.kinds)):
            GH = (4 if kind == 2 else 3) * H
            sv = [torch.empty((B * T, H), dtype=f32, device=dev), torch.empty((B * T, H), dtype=f32, device=dev),
                  torch.empty((B * T, GH), dtype=f32, device=dev), torch.empty((B * T, H), dtype=f32, device=dev)]
            sv += ([torch.empty((B * T, H), dtype=f32, device=dev), torch.empty(B * T, dtype=f32, device=dev)]
                   if self.acts[l] else [None, None])
            saved.append(sv)
            ptrs += [t.data_ptr() if t is not None else None for t in sv]
        table = (_ctypes_ptr_array(len(ptrs)))(*ptrs)
        h = torch.empty((B, self.hidden[-1]), dtype=f32, device=dev)
        _lib.check(_lib.lib.b200_rnn_train_forward(
            _lib.ptr(rows), B, _lib.ptr(lens_d), _lib.ptr(seqs_d), seqs_d.stride(0), T, _lib.ptr(E), E.stride(0),
            self.in_dim, len(self.hidden), self._kinds, self._hid, self._acts, _lib.ptr(self.rnn_w), _lib.ptr(h),
            h.stride(0), table, _lib.current_stream()))
        return h, dict(rows=rows, idx=idx, X0=X0, saved=saved, B=B, T=T, lens=lens_d)

    def user_vectors(self, seqs_d, lens_d):
        """The head over the encoder output (before any normalisation): [B, K] and the cache."""
        h, c = self.encode(seqs_d, lens_d)
        p = self.params
        u = linear(h, p["dense_Wt"], p["dense_b"], ACT_NONE, impl="f32")
        c["h"] = h
        return u, c

    # -- one step ----------------------------------------------------------------------------------------------------
    def forward_backward(self, items_d, seqs_d, lens_d, labels_or_neg):
        """Loss (device scalar) with every gradient buffer filled."""
        torch = self._torch
        lib, st, p, g, K = _lib.lib, _lib.current_stream(), self.params, self.grads, self.K
        f32, dev = torch.float32, self.device
        B = int(seqs_d.shape[0])
        u0, c = self.user_vectors(seqs_d, lens_d)
        loss = torch.empty((), dtype=f32, device=dev)
        gI, gb = g["item_embeds"], g["item_biases"]
        if self.loss_type == "bpr":
            neg_d = labels_or_neg
            Ip, Ip_pre, bp = self._items(items_d)
            In, In_pre, bn = self._items(neg_d)
            pos, neg = self._score(u0, Ip, bp), self._score(u0, In, bn)
            dpos = torch.empty(B, dtype=f32, device=dev)
            dneg = torch.empty(B, dtype=f32, device=dev)
            _lib.check(lib.b200_pairwise_loss(_lib.ptr(pos), B, _lib.ptr(neg), B, 0, 0.0, 0.25, 2.0, 1, _lib.ptr(loss),
                                              _lib.ptr(dpos), _lib.ptr(dneg), _lib.ptr(self._lws), self._lws.numel(),
                                              st))
            du = dpos[:, None] * Ip + dneg[:, None] * In           # the user side is not normalised (see above)
            dIp = self._normalize_backward(dpos[:, None] * u0, Ip_pre)
            dIn = self._normalize_backward(dneg[:, None] * u0, In_pre)
            for ids, dI, db in ((items_d, dIp, dpos), (neg_d, dIn, dneg)):
                _lib.check(lib.b200_scatter_add_rows(_lib.ptr(gI), K, K, _lib.ptr(ids), B, _lib.ptr(dI), K, st))
                _lib.check(lib.b200_scatter_add_rows(_lib.ptr(gb), 1, 1, _lib.ptr(ids), B, _lib.ptr(db), 1, st))
        else:
            u, u_pre = self._normalize(u0)
            I, I_pre, b = self._items(items_d)
            logit = self._score(u, I, b)
            dlogit = torch.empty(B, dtype=f32, device=dev)
            _lib.check(lib.b200_pointwise_loss(_lib.ptr(logit), _lib.ptr(labels_or_neg), B,
                                               RNN4REC_LOSSES[self.loss_type], 0.25, 2.0, _lib.ptr(loss),
                                               _lib.ptr(dlogit), _lib.ptr(self._lws), self._lws.numel(), st))
            du = self._normalize_backward(dlogit[:, None] * I, u_pre)
            dI = self._normalize_backward(dlogit[:, None] * u, I_pre)
            _lib.check(lib.b200_scatter_add_rows(_lib.ptr(gI), K, K, _lib.ptr(items_d), B, _lib.ptr(dI), K, st))
            _lib.check(lib.b200_scatter_add_rows(_lib.ptr(gb), 1, 1, _lib.ptr(items_d), B, _lib.ptr(dlogit), 1, st))
        du = du.contiguous()
        # the Dense head
        h = c["h"]
        g["dense_Wt"].copy_(_weight_grad(du, h))
        self._col_sum(du, g["dense_b"])
        dh = linear(du, p["dense_Wt"].t().contiguous(), None, False, cache_split=False)
        self.rnn_backward(c, dout=dh)
        return loss

    def rnn_backward(self, c, dout):
        """Backward of :meth:`encode` given d loss / d h [B, H_last]: every recurrent variable's gradient and the
        seq_embeds rows'."""
        torch = self._torch
        lib, st, g = _lib.lib, _lib.current_stream(), self.grads
        f32, dev = torch.float32, self.device
        B, T = c["B"], c["T"]
        S = B * T
        dy = None
        for l in range(len(self.hidden) - 1, -1, -1):
            H, kind, act = self.hidden[l], self.kinds[l], self.acts[l]
            GH = (4 if kind == 2 else 3) * H
            d = self.in_dim if l == 0 else self.hidden[l - 1]
            sv = c["saved"][l]
            dgx = torch.empty((S, GH), dtype=f32, device=dev)
            dgh = torch.empty((S, GH), dtype=f32, device=dev) if kind == 0 else None
            dln = torch.empty((S, H), dtype=f32, device=dev) if act else None
            dlnx = torch.empty((S, H), dtype=f32, device=dev) if act else None
            table = (_ctypes_ptr_array(6))(*[t.data_ptr() if t is not None else None for t in sv])
            lw = self.rnn_w[self._offs[l]:]
            _lib.check(lib.b200_rnn_backward(
                _lib.ptr(c["rows"]), B, _lib.ptr(c["lens"]), T, kind, d, H, act, _lib.ptr(lw),
                _lib.ptr(dout) if dy is None else None, dout.stride(0) if dy is None else 0, _lib.ptr(dy), table,
                _lib.ptr(dgx), _lib.ptr(dgh), _lib.ptr(dln), _lib.ptr(dlnx), st))
            X = c["X0"] if l == 0 else c["saved"][l - 1][1]
            pre = f"rnn{l}_"
            g[pre + "W"].copy_(_weight_grad(dgx, X).t())
            hp = sv[0]
            if kind == 1:        # TF1 GRU: the candidate block of U acts on r o h_{t-1}
                g[pre + "U"][:, :2 * H].copy_(_weight_grad(dgx[:, :2 * H].contiguous(), hp).t())
                g[pre + "U"][:, 2 * H:].copy_(_weight_grad(dgx[:, 2 * H:].contiguous(), sv[3]).t())
            else:
                g[pre + "U"].copy_(_weight_grad(dgx if dgh is None else dgh, hp).t())
            self._col_sum(dgx, g[pre + "bx"])
            if kind == 0:
                self._col_sum(dgh, g[pre + "bh"])
            if act:
                self._col_sum(dlnx, g[pre + "gamma"])
                self._col_sum(dln, g[pre + "beta"])
            W = self.params[pre + "W"]
            dy = linear(dgx, W, None, False, cache_split=False)          # dX = dGx W^T [S, d]
        ge = g["seq_embeds"]
        _lib.check(lib.b200_scatter_add_rows(_lib.ptr(ge), ge.stride(0), self.in_dim, _lib.ptr(c["idx"]), S,
                                             _lib.ptr(dy), dy.stride(0), st))

    def step(self, users_d, items_d, seqs_d, lens_d, labels_or_neg):
        """One optimisation step; returns the device loss.  Pointwise losses: ``step(users, items, seqs, lens,
        labels)``; bpr: ``step(users, items_pos, seqs, lens, items_neg)``."""
        torch = self._torch
        seqs_d = seqs_d.to(torch.int32).contiguous()
        self._check_batch(int(seqs_d.shape[0]), int(seqs_d.shape[1]))
        x = labels_or_neg.to(torch.int64 if self.loss_type == "bpr" else torch.float32).contiguous()
        loss = self.forward_backward(items_d.to(torch.int64).contiguous(), seqs_d, lens_d.to(torch.int32).contiguous(),
                                     x)
        self._adam_update()
        return loss

    def canonical_layers(self):
        """The trained layers in the canonical layout of ``weights_io.rnn_layers``."""
        out, d = [], self.in_dim
        w = self.rnn_w.cpu().numpy()
        for l, (H, kind) in enumerate(zip(self.hidden, self.kinds)):
            GH = (4 if kind == 2 else 3) * H
            o = self._offs[l]
            seg = lambda a, n: w[o + a:o + a + n]        # noqa: E731
            out.append(dict(kind=kind, act=self.acts[l], W=seg(0, d * GH).reshape(d, GH).copy(),
                            U=seg(d * GH, H * GH).reshape(H, GH).copy(), bx=seg((d + H) * GH, GH).copy(),
                            bh=seg((d + H + 1) * GH, GH).copy(), gamma=seg((d + H + 2) * GH, H).copy(),
                            beta=seg((d + H + 2) * GH + H, H).copy()))
            d = H
        return out

    def export_weights(self):
        """The raw variables of the trainer's scheme (``rnn4rec_weights``, ``rnn4rec_tf_variables`` and
        ``feat_models.RNN4Rec`` take them as they stand)."""
        from .weights_io import rnn_raw_layers

        p = self.params
        return dict(rnn_scheme=self.scheme, rnn_type=self.rnn_type, use_layer_norm=self.use_layer_norm,
                    seq_embeds=p["seq_embeds"].cpu().numpy(), item_embeds=p["item_embeds"].cpu().numpy(),
                    item_biases=p["item_biases"].cpu().numpy(),
                    rnn_layers=rnn_raw_layers(self.canonical_layers(), self.scheme, self.rnn_type, self.in_dim),
                    dense_kernel=p["dense_Wt"].cpu().numpy().T.copy(), dense_bias=p["dense_b"].cpu().numpy())

CONV_LOSSES = {"cross_entropy": 0, "focal": 1}


class _ConvSeqTrainer(_Trainer):
    """What the Caser and WaveNet training steps share (``caser.py:135-221``, ``wave_net.py:139-222`` in training
    mode, the losses of ``tfops/loss.py:4-25``, TF-Adam of ``training/tf_trainer.py:103-124``).  The user vector of
    a row is ``[user_embeds[u] | head(encoder(seq_embeds[seq]))]`` (2K wide), scored against ``item_embeds`` (2K)
    plus ``item_biases``:

        b200_gather_rows (user rows, the T input rows) -> b200_{caser,wavenet}_train_forward (saving the max-pool
        argmax, and WaveNet's layer outputs) -> the Dense head on b200_linear_f32 -> [b200_l2_normalize_rows]
        -> <u, i> + b_i (b200_gather_dot) -> b200_pointwise_loss -> [normalisation backward] -> b200_scatter_add_rows
        of the item, bias and user-row gradients -> head backward -> encoder backward -> b200_scatter_add_rows of dX
        into seq_embeds -> b200_adam_dense_dev

    ``weights``: the raw variables (``synthetic.make_caser_weights`` / ``make_wavenet_weights``,
    ``weights_io._conv_raw``) or the packed dict of ``weights_io.caser_weights`` / ``wavenet_weights``.  The Adam
    variables are the four tables, the head and every TF convolution variable, the last as views into the packed
    buffer ``conv_w`` that the kernels read (the packed layout is TensorFlow's, element for element); their gradients
    are views into ``conv_g``.  ``step(users, items, seqs, lens, labels)``: ``seqs`` [B, T] holds item ids padded with
    the pad row ``n_items``, which is trained like any other row (neither graph masks by length, so ``lens`` is
    accepted and not read).  ``users`` must lie in ``[0, n_users]``: they index ``user_embeds`` unchecked (a check
    would synchronise the host every step and break graph capture).  ``ValueError`` before any launch for ``bpr``
    (neither graph defines it), an unknown loss, the rating task, a ``seq_embeds`` row count other than
    ``n_items + 1``, shapes outside the envelope of the encoders and a batch whose saved state does not fit in the
    free device memory."""

    embed_table = "seq_embeds"
    reg_vars = ("user_embeds", "seq_embeds", "item_embeds")   # item_bias_var has no regularizer (caser.py:171-175)
    NAME = ""
    HEAD_ACT = ACT_NONE

    def __init__(self, spec, weights, loss_type="cross_entropy", norm_embed=False, task="ranking", lr=1e-3,
                 epsilon=1e-5, device=None):
        from .feat_models import CONV_MAX_K, _spec_get

        name = type(self).__name__
        if task != "ranking":
            raise ValueError(f"{name}: task `{task}` is not supported (ranking only)")
        if loss_type not in CONV_LOSSES:
            raise ValueError(f"{name}: loss_type must be one of {sorted(CONV_LOSSES)}, got `{loss_type}` (the graph "
                             "defines no bpr loss)")
        w = weights if "conv" in weights else self._pack(weights)
        g = None if isinstance(spec, FeatSpec) else _spec_get(spec)
        n_users = int(spec.n_users if g is None else g("n_users"))
        n_items = int(spec.n_items if g is None else g("n_items"))
        K = int(np.shape(w["seq_embeds"])[1])
        if not 1 <= K <= CONV_MAX_K:
            raise ValueError(f"{name}: embed_size {K} outside [1, {CONV_MAX_K}]")
        if np.shape(w["seq_embeds"])[0] != n_items + 1:
            raise ValueError(f"{name}: seq_embeds has {np.shape(w['seq_embeds'])[0]} rows, expected n_items + 1 = "
                             f"{n_items + 1}")
        shapes = {"user_embeds": (n_users + 1, K), "item_embeds": (n_items, 2 * K), "item_biases": (n_items,),
                  "dense_bias": (K,)}
        for k, shp in shapes.items():
            if tuple(np.shape(w[k])) != shp:
                raise ValueError(f"{name}: `{k}` has shape {np.shape(w[k])}, expected {shp}")
        self._check_encoder(w, K)
        self.loss_type, self.norm_embed = loss_type, bool(norm_embed)
        super().__init__(spec, w, False, lr, epsilon, device)
        torch = self._torch
        self.conv_g = torch.zeros_like(self.conv_w)
        for k, (off, shape) in self._views.items():
            self.grads[k] = self.conv_g[off:off + int(np.prod(shape))].view(shape)

    def _init_params(self, weights):
        p = self.params
        p["seq_embeds"] = self._var(weights["seq_embeds"])
        p["item_biases"] = self._var(weights["item_biases"], -1)
        p["dense_Wt"] = self._var(np.asarray(weights["dense_kernel"]).T.copy())      # [K, D]
        p["dense_b"] = self._var(weights["dense_bias"], -1)
        self.conv_w = self._var(weights["conv"], -1)
        self._views = self._conv_views()
        for k, (off, shape) in self._views.items():
            p[k] = self.conv_w[off:off + int(np.prod(shape))].view(shape)

    # -- memory ------------------------------------------------------------------------------------------------------
    def _check_batch(self, B, T):
        from .feat_models import CONV_MAX_T

        torch = self._torch
        name = type(self).__name__
        if not 1 <= T <= CONV_MAX_T:
            raise ValueError(f"{name}: sequence length {T} outside [1, {CONV_MAX_T}]")
        self._check_T(T)
        need = B * self.saved_bytes_per_row(T)
        free = torch.cuda.mem_get_info(self.device)[0] + torch.cuda.memory_reserved(self.device) - \
            torch.cuda.memory_allocated(self.device)
        if need > free:
            raise ValueError(f"{name}: a batch of {B} rows x T = {T} keeps {need} B for the backward, {free} B are "
                             "free")

    def _check_T(self, T):
        pass

    # -- forward -----------------------------------------------------------------------------------------------------
    def user_vectors(self, users_d, seqs_d):
        """``[user_embeds[users] | head(encoder(seqs))]`` [B, 2K] before any normalisation, and the cache of the
        backward."""
        torch = self._torch
        f32, dev, K = torch.float32, self.device, self.K
        B, T = int(seqs_d.shape[0]), int(seqs_d.shape[1])
        p, st = self.params, _lib.current_stream()
        users_d = users_d.to(torch.int64).contiguous()
        seqs_d = seqs_d.to(torch.int32).contiguous()
        rows = torch.arange(B, dtype=torch.int64, device=dev)
        idx = seqs_d.reshape(-1).to(torch.int64)
        E = p["seq_embeds"]
        X0 = torch.empty((B * T, K), dtype=f32, device=dev)
        _lib.check(_lib.lib.b200_gather_rows(_lib.ptr(E), E.stride(0), K, _lib.ptr(idx), B * T, _lib.ptr(X0), K, st))
        c = dict(users=users_d, rows=rows, idx=idx, X0=X0, seqs=seqs_d, B=B, T=T)
        feat = self._encode(c)
        u = torch.empty((B, 2 * K), dtype=f32, device=dev)
        U = p["user_embeds"]
        _lib.check(_lib.lib.b200_gather_rows(_lib.ptr(U), U.stride(0), K, _lib.ptr(users_d), B, _lib.ptr(u), u.stride(0),
                                             st))
        head = linear(feat, p["dense_Wt"], p["dense_b"], self.HEAD_ACT, impl="f32")
        u[:, K:] = head
        c.update(feat=feat, head=head)
        return u, c

    # -- one step ----------------------------------------------------------------------------------------------------
    def forward_backward(self, users_d, items_d, seqs_d, lens_d, labels_d):
        """Loss (device scalar) with every gradient buffer filled (``lens_d`` is not read)."""
        torch = self._torch
        lib, st, p, g, K = _lib.lib, _lib.current_stream(), self.params, self.grads, self.K
        B = int(seqs_d.shape[0])
        u0, c = self.user_vectors(users_d, seqs_d)
        u, u_pre = self._normalize(u0)
        I, I_pre, b = self._items(items_d)
        logit = self._score(u, I, b)
        loss = torch.empty((), dtype=torch.float32, device=self.device)
        dlogit = torch.empty(B, dtype=torch.float32, device=self.device)
        _lib.check(lib.b200_pointwise_loss(_lib.ptr(logit), _lib.ptr(labels_d), B, CONV_LOSSES[self.loss_type], 0.25,
                                           2.0, _lib.ptr(loss), _lib.ptr(dlogit), _lib.ptr(self._lws),
                                           self._lws.numel(), st))
        du = self._normalize_backward(dlogit[:, None] * I, u_pre).contiguous()
        dI = self._normalize_backward(dlogit[:, None] * u, I_pre).contiguous()
        gI, gb, gU = g["item_embeds"], g["item_biases"], g["user_embeds"]
        _lib.check(lib.b200_scatter_add_rows(_lib.ptr(gI), 2 * K, 2 * K, _lib.ptr(items_d), B, _lib.ptr(dI), 2 * K,
                                             st))
        _lib.check(lib.b200_scatter_add_rows(_lib.ptr(gb), 1, 1, _lib.ptr(items_d), B, _lib.ptr(dlogit), 1, st))
        _lib.check(lib.b200_scatter_add_rows(_lib.ptr(gU), K, K, _lib.ptr(c["users"]), B, _lib.ptr(du), 2 * K, st))
        # the Dense head; ReLU's mask is the same read from its output
        dh = du[:, K:].contiguous()
        if self.HEAD_ACT == ACT_RELU:
            _lib.check(lib.b200_activation_backward(_lib.ptr(dh), _lib.ptr(c["head"]), dh.numel(), ACT_RELU,
                                                    _lib.ptr(dh), st))
        g["dense_Wt"].copy_(_weight_grad(dh, c["feat"]))
        self._col_sum(dh, g["dense_b"])
        dF = linear(dh, p["dense_Wt"].t().contiguous(), None, False, cache_split=False)
        dX = self._encoder_backward(c, dF)
        ge = g["seq_embeds"]
        _lib.check(lib.b200_scatter_add_rows(_lib.ptr(ge), ge.stride(0), K, _lib.ptr(c["idx"]), B * c["T"],
                                             _lib.ptr(dX), dX.stride(0), st))
        return loss

    def step(self, users_d, items_d, seqs_d, lens_d, labels_d):
        """One optimisation step; returns the device loss."""
        torch = self._torch
        seqs_d = seqs_d.to(torch.int32).contiguous()
        self._check_batch(int(seqs_d.shape[0]), int(seqs_d.shape[1]))
        loss = self.forward_backward(users_d.to(torch.int64).contiguous(), items_d.to(torch.int64).contiguous(),
                                     seqs_d, lens_d, labels_d.to(torch.float32).contiguous())
        self._adam_update()
        return loss

    def _export_common(self):
        p = self.params
        out = {k: p[k].cpu().numpy() for k in ("user_embeds", "seq_embeds", "item_embeds", "item_biases")}
        out.update(dense_kernel=p["dense_Wt"].cpu().numpy().T.copy(), dense_bias=p["dense_b"].cpu().numpy())
        return out


class CaserTrainer(_ConvSeqTrainer):
    """Caser's training step (``caser.py:135-221``): ``b200_caser_train_forward`` saves each horizontal column's
    max-pool argmax; ``b200_caser_backward`` routes the head's gradient through it (and through the vertical
    columns' ReLU) into dX and every convolution variable.  The head is ``Dense(K, relu)``.  See
    :class:`_ConvSeqTrainer`; the sequence length is the weights' T."""

    HEAD_ACT = ACT_RELU

    @staticmethod
    def _pack(raw):
        from .weights_io import caser_weights

        return caser_weights(raw)

    def _check_encoder(self, w, K):
        from .feat_models import CONV_MAX_FILTERS, CONV_MAX_T

        self.T, self.nh, self.nv = int(w["T"]), int(w["nh"]), int(w["nv"])
        if not 1 <= self.T <= CONV_MAX_T:
            raise ValueError(f"CaserTrainer: max_seq_len {self.T} outside [1, {CONV_MAX_T}]")
        if not (1 <= self.nh <= CONV_MAX_FILTERS and 1 <= self.nv <= CONV_MAX_FILTERS):
            raise ValueError(f"CaserTrainer: nh_filters {self.nh} / nv_filters {self.nv} outside "
                             f"[1, {CONV_MAX_FILTERS}]")
        self.D = self.T * self.nh + K * self.nv
        if np.size(w["conv"]) != int(_lib.lib.b200_caser_weight_floats(self.T, K, self.nh, self.nv)):
            raise ValueError(f"CaserTrainer: {np.size(w['conv'])} packed convolution floats do not match T {self.T}, "
                             f"K {K}, nh {self.nh}, nv {self.nv}")
        if tuple(np.shape(w["dense_kernel"])) != (self.D, K):
            raise ValueError(f"CaserTrainer: `dense_kernel` has shape {np.shape(w['dense_kernel'])}, expected "
                             f"({self.D}, {K})")

    def _check_T(self, T):
        if T != self.T:
            raise ValueError(f"CaserTrainer: sequences of length {T}, the model has {self.T} horizontal convolutions")

    def _conv_views(self):
        """{variable: (offset, TF shape)} in the packed layout: W_1 .. W_T, the T biases, Wv, bv."""
        T, K, nh, nv = self.T, self.K, self.nh, self.nv
        out, off = {}, 0
        for h in range(1, T + 1):
            out[f"conv{h - 1}_kernel"] = (off, (h, K, nh))
            off += h * K * nh
        for h in range(1, T + 1):
            out[f"conv{h - 1}_bias"] = (off, (nh,))
            off += nh
        out["vertical_kernel"] = (off, (1, T, nv))
        out["vertical_bias"] = (off + T * nv, (nv,))
        return out

    def saved_bytes_per_row(self, T):
        """Device bytes one batch row keeps for the backward: the input rows and dX (T x K each), the features and
        dF (D each), the argmax (T nh), the user vector and its gradient (2K each), the head (K), and the row's
        share of the weight-gradient partials."""
        ws = int(_lib.lib.b200_caser_backward_workspace_floats(256, T, self.K, self.nh, self.nv))
        return 4 * (2 * T * self.K + 2 * self.D + T * self.nh + 5 * self.K) + -(-4 * ws // 256)

    def _encode(self, c):
        torch = self._torch
        B, T = c["B"], c["T"]
        E = self.params["seq_embeds"]
        feat = torch.empty((B, self.D), dtype=torch.float32, device=self.device)
        arg = torch.empty((B, T * self.nh), dtype=torch.int32, device=self.device)
        _lib.check(_lib.lib.b200_caser_train_forward(
            _lib.ptr(c["rows"]), B, _lib.ptr(c["seqs"]), c["seqs"].stride(0), T, _lib.ptr(E), E.stride(0), self.K,
            self.nh, self.nv, _lib.ptr(self.conv_w), _lib.ptr(feat), feat.stride(0), _lib.ptr(arg),
            _lib.current_stream()))
        c["arg"] = arg
        return feat

    def _encoder_backward(self, c, dF):
        torch = self._torch
        B, T, K = c["B"], c["T"], self.K
        n_ws = int(_lib.lib.b200_caser_backward_workspace_floats(B, T, K, self.nh, self.nv))
        ws = torch.empty(max(n_ws, 1), dtype=torch.float32, device=self.device)
        dX = torch.empty((B * T, K), dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib.b200_caser_backward(
            B, T, K, self.nh, self.nv, _lib.ptr(dF), dF.stride(0), _lib.ptr(c["feat"]), c["feat"].stride(0),
            _lib.ptr(c["arg"]), _lib.ptr(c["X0"]), K, _lib.ptr(self.conv_w), _lib.ptr(dX), K, _lib.ptr(self.conv_g),
            _lib.ptr(ws), n_ws, _lib.current_stream()))
        return dX

    def export_weights(self):
        """The raw variables (``caser_weights``, ``caser_tf_variables`` and ``feat_models.Caser`` take them)."""
        out = self._export_common()
        v = {k: self.params[k].cpu().numpy() for k in self._views}
        out["convs"] = [dict(kernel=v[f"conv{i}_kernel"], bias=v[f"conv{i}_bias"]) for i in range(self.T)]
        out["vertical"] = dict(kernel=v["vertical_kernel"], bias=v["vertical_bias"])
        return out


class WaveNetTrainer(_ConvSeqTrainer):
    """WaveNet's training step (``wave_net.py:139-222``): ``b200_wavenet_train_forward`` saves every causal layer's
    output and the 1x1 layer's argmax over t.  The backward runs on the dense kernels plus three position kernels:
    ``b200_wavenet_pool_backward`` puts the gradient at each argmax; then the 1x1 layer's products; then, per causal
    layer from the top, the ReLU mask (``b200_activation_backward`` on the saved output), the kernel gradient
    ``[x_{t-d} | x_t]^T dpre`` over ``b200_wavenet_layer_inputs``, and ``dx`` from ``dpre [W0; W1]^T`` shifted by
    ``b200_wavenet_layer_dx``.  The head is ``Dense(K)``.  The dilations come from the weights (1 everywhere for a
    TF1-trained graph).  See :class:`_ConvSeqTrainer`."""

    @staticmethod
    def _pack(raw):
        from .weights_io import wavenet_weights

        return wavenet_weights(raw)

    def _check_encoder(self, w, K):
        from .feat_models import CONV_MAX_F, CONV_MAX_LAYERS

        self.n_filters, self.dilations = int(w["F"]), [int(d) for d in w["dilations"]]
        if not 1 <= self.n_filters <= CONV_MAX_F:
            raise ValueError(f"WaveNetTrainer: n_filters {self.n_filters} outside [1, {CONV_MAX_F}]")
        if not 1 <= len(self.dilations) <= CONV_MAX_LAYERS or min(self.dilations) < 1:
            raise ValueError(f"WaveNetTrainer: dilations {self.dilations}: 1 to {CONV_MAX_LAYERS} causal layers, each "
                             "dilation >= 1")
        if np.size(w["conv"]) != int(_lib.lib.b200_wavenet_weight_floats(K, self.n_filters, len(self.dilations))):
            raise ValueError(f"WaveNetTrainer: {np.size(w['conv'])} packed convolution floats do not match K {K}, "
                             f"F {self.n_filters}, {len(self.dilations)} causal layers")
        if tuple(np.shape(w["dense_kernel"])) != (self.n_filters, K):
            raise ValueError(f"WaveNetTrainer: `dense_kernel` has shape {np.shape(w['dense_kernel'])}, expected "
                             f"({self.n_filters}, {K})")
        self.D = self.n_filters
        self._dil = (ctypes.c_int32 * len(self.dilations))(*self.dilations)

    def _conv_views(self):
        """{variable: (offset, TF shape)} in the packed layout: per causal layer kernel [2, C, F], bias; then the 1x1
        layer's kernel [1, F, F], bias."""
        K, F = self.K, self.n_filters
        out, off = {}, 0
        for l in range(len(self.dilations)):
            C = K if l == 0 else F
            out[f"conv{l}_kernel"] = (off, (2, C, F))
            out[f"conv{l}_bias"] = (off + 2 * C * F, (F,))
            off += 2 * C * F + F
        out["out_conv_kernel"] = (off, (1, F, F))
        out["out_conv_bias"] = (off + F * F, (F,))
        return out

    def saved_bytes_per_row(self, T):
        """Device bytes one batch row keeps for the backward: the input rows (T x K), every causal layer's output
        (L x T x F), the argmax, features, user vector and head (F + F + 4K + K), dZ / dy (T x F each) and the
        largest layer's transients (dpre, [x_{t-d} | x_t], the [2C] product, dx)."""
        K, F, L = self.K, self.n_filters, len(self.dilations)
        C = max(K, F)
        return 4 * (T * K + L * T * F + 2 * F + 5 * K + 2 * T * F + T * (F + 5 * C))

    def _encode(self, c):
        torch = self._torch
        B, T, F = c["B"], c["T"], self.n_filters
        E = self.params["seq_embeds"]
        feat = torch.empty((B, F), dtype=torch.float32, device=self.device)
        ys = torch.empty((len(self.dilations), B * T, F), dtype=torch.float32, device=self.device)
        arg = torch.empty((B, F), dtype=torch.int32, device=self.device)
        _lib.check(_lib.lib.b200_wavenet_train_forward(
            _lib.ptr(c["rows"]), B, _lib.ptr(c["seqs"]), c["seqs"].stride(0), T, _lib.ptr(E), E.stride(0), self.K,
            len(self.dilations), F, self._dil, _lib.ptr(self.conv_w), _lib.ptr(feat), feat.stride(0), _lib.ptr(ys),
            _lib.ptr(arg), _lib.current_stream()))
        c.update(arg=arg, ys=ys)
        return feat

    def _encoder_backward(self, c, dF):
        torch = self._torch
        lib, st, p, g = _lib.lib, _lib.current_stream(), self.params, self.grads
        B, T, F, K = c["B"], c["T"], self.n_filters, self.K
        S, L = B * T, len(self.dilations)
        f32, dev = torch.float32, self.device
        dZ = torch.empty((S, F), dtype=f32, device=dev)
        _lib.check(lib.b200_wavenet_pool_backward(B, T, F, _lib.ptr(dF), dF.stride(0), _lib.ptr(c["arg"]),
                                                  _lib.ptr(dZ), st))
        ys = c["ys"]
        g["out_conv_kernel"][0].copy_(_weight_grad(dZ, ys[L - 1]).t())       # W1[c, f] += y[t, c] dZ[t, f]
        self._col_sum(dZ, g["out_conv_bias"])
        dy = linear(dZ, p["out_conv_kernel"][0], None, False, cache_split=False)    # dZ W1^T
        for l in range(L - 1, -1, -1):
            C, d = (K if l == 0 else F), self.dilations[l]
            dpre = torch.empty((S, F), dtype=f32, device=dev)
            _lib.check(lib.b200_activation_backward(_lib.ptr(dy), _lib.ptr(ys[l]), S * F, ACT_RELU, _lib.ptr(dpre),
                                                    st))
            x = c["X0"] if l == 0 else ys[l - 1]
            xin = torch.empty((S, 2 * C), dtype=f32, device=dev)
            _lib.check(lib.b200_wavenet_layer_inputs(_lib.ptr(x), x.stride(0), B, T, C, d, _lib.ptr(xin), st))
            g[f"conv{l}_kernel"].view(2 * C, F).copy_(_weight_grad(dpre, xin).t())
            self._col_sum(dpre, g[f"conv{l}_bias"])
            P = linear(dpre, p[f"conv{l}_kernel"].view(2 * C, F), None, False, cache_split=False)   # [S, 2C]
            dy = torch.empty((S, C), dtype=f32, device=dev)
            _lib.check(lib.b200_wavenet_layer_dx(_lib.ptr(P), B, T, C, d, _lib.ptr(dy), C, st))
        return dy

    def export_weights(self):
        """The raw variables (``wavenet_weights``, ``wavenet_tf_variables`` and ``feat_models.WaveNet`` take them)."""
        out = self._export_common()
        v = {k: self.params[k].cpu().numpy() for k in self._views}
        out["convs"] = [dict(kernel=v[f"conv{i}_kernel"], bias=v[f"conv{i}_bias"]) for i in range(len(self.dilations))]
        out["out_conv"] = dict(kernel=v["out_conv_kernel"], bias=v["out_conv_bias"])
        out["dilations"] = list(self.dilations)
        return out


def _ctypes_ptr_array(n):
    import ctypes

    return ctypes.c_void_p * n


SIM_LOSSES = {"cross_entropy": 0, "focal": 1}


class SIMTrainer(_SeqTrainer):
    """SIM training step on the device: ``libreco/algorithms/sim.py:193-304`` in training mode (no dropout), mean
    sigmoid cross entropy or focal loss on ``alpha * z1 + beta * z2``, TF-Adam.  Every row carries its own dual
    sequences (``collate.DeviceDualSequenceBuilder``): ``long_seqs`` [R, L], ``short_seqs`` [R, S] and their lengths,
    clamped to [1, L] / [1, S] as the collator gives them.

        G (the item feature table, concat mode, from the CURRENT tables) -> Gp = G Wp (b200_linear_f32, the bits the
        inference engine selects from) -> q = Gp[item] (b200_gather_rows)
        first stage: b200_sim_gsu_forward also sums pooled = sum_{t < long_len} Gp[long_t] -> dense_nn "fs_" on
            [q, pooled] -> Dense(1) = z1
        second stage: the GSU selection (b200_sim_gsu_forward) -> Gp of the selected rows -> multi_head_attention
            of q over them (projections on the dense kernels, b200_sim_esu_forward) -> short attention
            (b200_transformer_target_attention) -> K1 gather -> dense_nn on [fields.., long_out, short_out] ->
            Dense(1) = z2
        -> b200_pointwise_loss -> the reverse (b200_sim_esu_backward, b200_transformer_target_attention_backward,
        the dense kernels) -> dGp: query and short-key rows through b200_scatter_add_rows, the selected and pooled
        rows through b200_sim_long_backward -> dWp = G^T dGp, dG = dGp Wp^T folded into the tables ->
        b200_feat_backward -> b200_adam_dense_dev

    ``weights``: the RAW variables of either attention graph, as ``synthetic.make_sim_weights`` and
    ``weights_io.load_reference_tf_model(..., "SIM", ...)`` give them.  The second stage's first kernel is held with
    the sequence block after the field blocks (the inference engine's layout) and permuted back on export.
    ``export_weights`` returns the same raw layout (``weights_io.sim_weights`` makes the serving dict,
    ``weights_io.sim_tf_variables`` the reference's variable names).  ``reg`` applies to the embedding tables only.

    Raises ``ValueError`` before anything is launched for alpha or beta outside [0, 1], an unknown ``loss_type``, the
    rating task, shapes outside the kernels' envelope (K <= 64 with heads dividing K, L <= 256, S <= 64,
    search_topk <= min(32, L)), multi-sparse fields with a combiner other than "normal" (the pooling backward is not
    built) and first layers whose width disagrees with the fields."""

    def __init__(self, spec, weights, search_topk=10, alpha=1.0, beta=1.0, loss_type="cross_entropy", use_bn=True,
                 lr=1e-3, epsilon=1e-5, device=None, task="ranking"):
        from .feat_models import _spec_get

        if not (0.0 <= float(alpha) <= 1.0 and 0.0 <= float(beta) <= 1.0):
            raise ValueError(f"SIMTrainer: alpha {alpha} and beta {beta} must lie in [0, 1]")
        if task != "ranking":
            raise ValueError(f"SIMTrainer: task {task!r} is not supported, SIM trains the ranking task only")
        if loss_type not in SIM_LOSSES:
            raise ValueError(f"SIMTrainer: unsupported loss_type {loss_type!r}, expected one of {sorted(SIM_LOSSES)}")
        g = _spec_get(spec) if not isinstance(spec, FeatSpec) else (lambda k, d=None: d)
        if g("multi_sparse_combine_info") is not None and weights.get("multi_sparse_combiner", "sqrtn") != "normal":
            raise ValueError("SIMTrainer: multi-sparse fields need the combiner \"normal\"; the pooling backward is "
                             "not built")
        self._combiner = weights.get("multi_sparse_combiner")
        self.alpha, self.beta, self.loss_type = float(alpha), float(beta), loss_type
        self.topk = int(search_topk)
        super().__init__(spec, weights, use_bn, lr, epsilon, device)

    def _init_params(self, weights):
        from .feat_models import SIM_MAX_K, SIM_MAX_TOPK

        K, F = self.K, self.F
        H = self.H = int(weights["num_heads"])
        self.scheme = weights["sim_scheme"]
        _check_mha_scheme(self.scheme, "SIMTrainer")
        if K > SIM_MAX_K or H < 1 or K % H:
            raise ValueError(f"SIMTrainer: embed size {K} with {H} heads outside K <= {SIM_MAX_K}, heads dividing K")
        if not 1 <= self.topk <= SIM_MAX_TOPK:
            raise ValueError(f"SIMTrainer: search_topk {self.topk} outside [1, {SIM_MAX_TOPK}]")
        for name, want in (("mlp", (F + 2) * K), ("first_stage_mlp", 2 * K)):
            n_in = np.shape(weights[name]["kernels"][0])[0]
            if n_in != want:
                raise ValueError(f"SIMTrainer: the first layer of {name} takes {n_in} inputs, expected {want} "
                                 f"(F = {F}, K = {K})")
        # reference order [long, short, user, item, sparse.., dense..] -> ours [user, item, sparse.., dense.., long, short]
        self.perm = np.concatenate([np.arange(2 * K, (F + 2) * K), np.arange(0, 2 * K)])
        super()._init_params(dict(weights, mlp=permute_mlp_input(weights["mlp"], self.perm)))
        p = self.params
        self.n_fs = self._init_stack("fs_", weights["first_stage_mlp"])
        p["first_stage_out_kernel"] = self._var(weights["first_stage_out_kernel"], -1)
        p["first_stage_out_bias"] = self._var(weights["first_stage_out_bias"], 1)
        self._init_item_table()
        if np.shape(weights["seq_proj"]) != (self.Kp, K):
            raise ValueError(f"SIMTrainer: seq_proj has shape {np.shape(weights['seq_proj'])}, expected "
                             f"({self.Kp}, {K})")
        p["seq_projT"] = self._var(np.ascontiguousarray(np.asarray(weights["seq_proj"]).T))
        self._init_mha("sim_", weights["sim_mha"], K, K, 0)

    def _check_batch(self, L, S):
        from .feat_models import SIM_MAX_L, SIM_MAX_S

        if not 1 <= L <= SIM_MAX_L or not 1 <= S <= SIM_MAX_S or self.topk > L:
            raise ValueError(f"SIMTrainer: long length {L}, short length {S}, search_topk {self.topk} outside "
                             f"L <= {SIM_MAX_L}, S <= {SIM_MAX_S}, search_topk <= L")

    def forward(self, users_d, items_d, long_seqs, long_lens, short_seqs, short_lens):
        """Training-mode logits alpha z1 + beta z2 of the batch (batch statistics in the BN); caches what the backward
        needs."""
        torch = self._torch
        lib, st, p = _lib.lib, _lib.current_stream(), self.params
        K, F, H, k = self.K, self.F, self.H, self.topk
        R, L, S = int(users_d.numel()), int(long_seqs.shape[1]), int(short_seqs.shape[1])
        f32, dev = torch.float32, self.device
        G = self._build_G()
        Gp = linear(G, p["seq_projT"], None, ACT_NONE, impl="f32")
        q = torch.empty((R, K), dtype=f32, device=dev)
        _lib.check(lib.b200_gather_rows(_lib.ptr(Gp), Gp.stride(0), K, _lib.ptr(items_d), R, _lib.ptr(q), K, st))
        # first-stage input [q || pooled]; the GSU kernel writes the pooled block
        xf = torch.empty((R, 2 * K), dtype=f32, device=dev)
        xf[:, :K] = q
        sel = torch.empty((R, k), dtype=torch.int32, device=dev)
        pooled = xf[:, K:]
        _lib.check(lib.b200_sim_gsu_forward(_lib.ptr(Gp), Gp.stride(0), K, _lib.ptr(items_d), _lib.ptr(long_seqs),
                                            long_seqs.stride(0), _lib.ptr(long_lens), L, k, R, _lib.ptr(sel),
                                            _lib.ptr(pooled), xf.stride(0), st))
        sel_idx = torch.gather(long_seqs, 1, sel.to(torch.int64)).reshape(-1).to(torch.int64)
        Xsel = torch.empty((R * k, K), dtype=f32, device=dev)
        _lib.check(lib.b200_gather_rows(_lib.ptr(Gp), Gp.stride(0), K, _lib.ptr(sel_idx), R * k, _lib.ptr(Xsel), K,
                                        st))

        def core(qq, kk, vv):
            o = torch.empty((R, K), dtype=f32, device=dev)
            P = torch.empty(R * H * k, dtype=f32, device=dev)
            _lib.check(lib.b200_sim_esu_forward(_lib.ptr(qq), qq.stride(0), _lib.ptr(kk), _lib.ptr(vv), K,
                                                _lib.ptr(sel), _lib.ptr(long_lens), R, K, H, k, _lib.ptr(o), K,
                                                _lib.ptr(P), st))
            return o, P

        long_out, mha = self._mha_forward("sim_", q, core, kv=Xsel)
        x = torch.empty((R, F * K + 2 * K), dtype=f32, device=dev)
        feat_forward(self.spec.layout, self.tables, users_d, items_d, R, concat=x)
        x[:, F * K:F * K + K] = long_out
        short_idx = short_seqs.reshape(-1).to(torch.int64)
        Sg = torch.empty((R * S, K), dtype=f32, device=dev)
        _lib.check(lib.b200_gather_rows(_lib.ptr(Gp), Gp.stride(0), K, _lib.ptr(short_idx), R * S, _lib.ptr(Sg), K,
                                        st))
        so = x[:, F * K + K:]
        rows = torch.arange(R, dtype=torch.int64, device=dev)
        slots = rows.to(torch.int32)
        _lib.check(lib.b200_transformer_target_attention(_lib.ptr(q), K, _lib.ptr(Sg), S, K, _lib.ptr(short_lens),
                                                         _lib.ptr(slots), _lib.ptr(rows), R, 0, 0, _lib.ptr(so),
                                                         x.stride(0), st))
        h2, c2 = self._stack_forward("", self.n_layers, x)
        z2 = self._dense1_forward(h2)
        h1, c1 = self._stack_forward("fs_", self.n_fs, xf)
        z1 = self._dense1_forward(h1, "first_stage_out_")
        logit = torch.zeros(R, dtype=f32, device=dev)
        _lib.check(lib.b200_axpy(_lib.ptr(logit), _lib.ptr(z1), self.alpha, R, st))
        _lib.check(lib.b200_axpy(_lib.ptr(logit), _lib.ptr(z2), self.beta, R, st))
        self._cache = dict(R=R, L=L, S=S, users=users_d, items=items_d, long_seqs=long_seqs, long_lens=long_lens,
                           short_idx=short_idx, short_lens=short_lens, G=G, q=q, sel=sel, Sg=Sg, mha=mha, c2=c2,
                           h2=h2, c1=c1, h1=h1, logit=logit)
        return logit

    def backward(self, labels_d):
        """Loss + every gradient buffer filled (before the optimiser); returns the device loss."""
        torch = self._torch
        lib, st, p, g = _lib.lib, _lib.current_stream(), self.params, self.grads
        K, F, H, k = self.K, self.F, self.H, self.topk
        c = self._cache
        R, L, S = c["R"], c["L"], c["S"]
        f32, dev = torch.float32, self.device
        loss = torch.empty((), dtype=f32, device=dev)
        dlogit = torch.empty(R, dtype=f32, device=dev)
        _lib.check(lib.b200_pointwise_loss(_lib.ptr(c["logit"]), _lib.ptr(labels_d), R, SIM_LOSSES[self.loss_type],
                                           0.25, 2.0, _lib.ptr(loss), _lib.ptr(dlogit), _lib.ptr(self._lws),
                                           self._lws.numel(), st))
        dz1 = torch.zeros(R, dtype=f32, device=dev)
        dz2 = torch.zeros(R, dtype=f32, device=dev)
        _lib.check(lib.b200_axpy(_lib.ptr(dz1), _lib.ptr(dlogit), self.alpha, R, st))
        _lib.check(lib.b200_axpy(_lib.ptr(dz2), _lib.ptr(dlogit), self.beta, R, st))
        # second stage
        _, dh2 = self._dense1_backward(c["h2"], None, None, dlogit=dz2)
        dx = self._stack_backward("", self.n_layers, c["c2"], dh2)
        feat_backward(self.spec.layout, self.tables, c["users"], c["items"], R, g, dconcat=dx)
        q, sel, ll = c["q"], c["sel"], c["long_lens"]
        dq = torch.empty((R, K), dtype=f32, device=dev)
        dSg = torch.empty((R * S, K), dtype=f32, device=dev)
        dso = dx[:, F * K + K:]
        _lib.check(lib.b200_transformer_target_attention_backward(
            _lib.ptr(q), K, _lib.ptr(c["Sg"]), S, K, _lib.ptr(c["short_lens"]), _lib.ptr(dso), dx.stride(0), R,
            _lib.ptr(dq), K, _lib.ptr(dSg), st))

        def core_backward(m, dO):
            dqh = torch.empty((R, K), dtype=f32, device=dev)
            dk, dv = (torch.empty((R * k, K), dtype=f32, device=dev) for _ in range(2))
            _lib.check(lib.b200_sim_esu_backward(_lib.ptr(m["q"]), m["q"].stride(0), _lib.ptr(m["k"]),
                                                 _lib.ptr(m["v"]), K, _lib.ptr(sel), _lib.ptr(ll), R, K, H, k, _lib.ptr(m["lse"]),
                                                 _lib.ptr(dO), dO.stride(0), _lib.ptr(dqh), K, _lib.ptr(dk),
                                                 _lib.ptr(dv), K, st))
            return dqh, dk, dv

        dq_esu, dXsel = self._mha_backward("sim_", c["mha"], dx[:, F * K:F * K + K].contiguous(), core_backward)
        # first stage
        _, dh1 = self._dense1_backward(c["h1"], None, None, "first_stage_out_", dlogit=dz1)
        dxf = self._stack_backward("fs_", self.n_fs, c["c1"], dh1)
        self._axpy(dq, dq_esu)
        self._axpy(dq, dxf[:, :K].contiguous())
        # dGp: the query rows, the short keys, the selected and the pooled rows
        n = self.n_items + 1
        dGp = torch.zeros((n, K), dtype=f32, device=dev)
        _lib.check(lib.b200_scatter_add_rows(_lib.ptr(dGp), K, K, _lib.ptr(c["items"]), R, _lib.ptr(dq), K, st))
        _lib.check(lib.b200_scatter_add_rows(_lib.ptr(dGp), K, K, _lib.ptr(c["short_idx"]), R * S, _lib.ptr(dSg), K,
                                             st))
        dpooled = dxf[:, K:]
        _lib.check(lib.b200_sim_long_backward(_lib.ptr(c["long_seqs"]), c["long_seqs"].stride(0), _lib.ptr(ll), L,
                                              _lib.ptr(sel), k, R, K, _lib.ptr(dpooled), dxf.stride(0),
                                              _lib.ptr(dXsel), dXsel.stride(0), _lib.ptr(dGp), K, st))
        # Gp = G Wp
        G = c["G"]
        g["seq_projT"] += _weight_grad(dGp, G)
        self._fold_dG(linear(dGp, p["seq_projT"].t().contiguous(), None, ACT_NONE, cache_split=False))
        return loss

    def step(self, users_d, items_d, long_seqs, long_lens, short_seqs, short_lens, labels_d):
        """One optimisation step; returns the device loss."""
        torch = self._torch
        L, S = int(long_seqs.shape[1]), int(short_seqs.shape[1])
        self._check_batch(L, S)
        i32 = torch.int32
        self.forward(users_d.to(torch.int64).contiguous(), items_d.to(torch.int64).contiguous(),
                     long_seqs.to(i32).contiguous(), long_lens.to(i32).clamp(1, L).contiguous(),
                     short_seqs.to(i32).contiguous(), short_lens.to(i32).clamp(1, S).contiguous())
        loss = self.backward(labels_d.to(torch.float32).contiguous())
        self._adam_update()
        self._cache = None
        return loss

    def export_weights(self):
        """The raw variables in the scheme they came in, both stages."""
        p, K = self.params, self.K
        w = super().export_weights()
        inv = np.argsort(self.perm)
        w["mlp"]["kernels"][0] = w["mlp"]["kernels"][0][inv]
        if self.use_bn:
            w["mlp"]["bn_in"] = {k: v[inv] for k, v in w["mlp"]["bn_in"].items()}
        w.update(sim_scheme=self.scheme, num_heads=self.H,
                 seq_proj=np.ascontiguousarray(p["seq_projT"].cpu().numpy().T), sim_mha=self._export_mha("sim_", K, K), first_stage_mlp=self._export_stack("fs_", self.n_fs),
                 first_stage_out_kernel=p["first_stage_out_kernel"].cpu().numpy().reshape(-1, 1),
                 first_stage_out_bias=p["first_stage_out_bias"].cpu().numpy().reshape(1),
                 out_kernel=w["out_kernel"].reshape(-1, 1),
                 out_bias=np.asarray(w["out_bias"], dtype=np.float32).reshape(1))
        if self._combiner is not None:
            w["multi_sparse_combiner"] = self._combiner
        return w

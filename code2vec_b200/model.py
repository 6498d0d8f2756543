"""Drop-in `Code2Vec` for the reference's `model/model.py`, backed by the sm_90a kernels.

Boundary mirrored:
  * constructor `Code2Vec(option)` reads the same Option fields (model.py:18-42) and creates
    the same submodules in the same order, so `torch.manual_seed(s); Code2Vec(option)` gives
    bit-identical initial weights and `state_dict()` keys/shapes interchange with the reference;
  * `forward(starts, paths, ends, label) -> (outputs, code_vector, attention)` (model.py:44-88),
    int64 [b, L] inputs, fp32 outputs, autograd-connected to every parameter;
  * `model.train()/eval()` toggle dropout only (model.py:60-61);
  * `from code2vec_b200.model import *` also exports `nn`, `F`, `torch`, `math`, `Parameter`,
    `NINF`, because the reference's main.py uses `nn` / `F` from that star import
    (main.py:22, :130, :261).

There is no CPU path: parameters and inputs must live on a CUDA (H100) device.
"""
import math

import os

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.nn.parameter import Parameter

from . import _lib
from . import functional as CF

NINF = - 3.4 * math.pow(10, 38)  # model.py:12

__all__ = ["Code2Vec", "NINF", "torch", "nn", "F", "Parameter", "math"]


class _EncodeFn(torch.autograd.Function):
    """gathers -> concat -> input_linear -> LayerNorm -> tanh -> dropout -> attention -> code vector."""

    @staticmethod
    def forward(ctx, emb_t, emb_p, W, ln_g, ln_b, attn, starts, paths, ends, dims, drop_p, training, seed, algo, cache,
                sparse=(False, False)):
        params = CF.make_params(emb_t, emb_p, W, ln_g, ln_b, attn)
        # when a gradient will be asked for, keep x = c . W^T (105 MB per 1024 x 200 batch at encode_size 128) so that
        # the backward neither re-gathers the embedding rows nor redoes the input_linear GEMM
        stash = any(ctx.needs_input_grad[:6]) and os.environ.get("C2V_NO_STASH", "0") != "1"
        # a PackedBags batch comes in the `starts` position (paths = ends = None); its attention is [N]
        ctx.bags = starts if isinstance(starts, CF.PackedBags) else None
        if ctx.bags is not None:
            res = CF.encode_forward_packed(dims, params, ctx.bags, drop_p, training, seed, algo, cache=cache, weight=W,
                                           stash=stash)
            starts = None
        else:
            res = CF.encode_forward(dims, params, starts, paths, ends, drop_p, training, seed, algo,
                                    cache=cache, weight=W, stash=stash)
        cv, att = res[0], res[1]
        ctx.x_stash = res[2] if stash else None
        # sparse embedding gradients (nn.Embedding.sparse): the row map of each such table is built here, where the indices
        # are at hand; the backward needs U on the host only to shape the final sparse tensor, so U travels to pinned
        # memory behind an event and the backward's one host wait is on that event
        ctx.row_maps = None
        want = (sparse[0] and ctx.needs_input_grad[0], sparse[1] and ctx.needs_input_grad[1])
        if any(want):
            s_, p_, e_ = (ctx.bags.starts, ctx.bags.paths, ctx.bags.ends) if ctx.bags is not None else (starts, paths, ends)
            with torch.cuda.device(s_.device):       # row maps, copies and event all on the stream of the batch's device
                maps = (CF.sparse_rows([s_, e_], dims.terminal_count) if want[0] else None,
                        CF.sparse_rows([p_], dims.path_count) if want[1] else None)
                counts = torch.zeros(2, dtype=torch.int64, pin_memory=True)
                for i, m in enumerate(maps):
                    if m is not None:
                        counts[i:i + 1].copy_(m[2], non_blocking=True)
                ready = torch.cuda.Event()
                ready.record(torch.cuda.current_stream(s_.device))
            # kept with the graph (freed with it), so that a backward with retain_graph=True can run again
            ctx.row_maps = (maps, counts, ready)
        ctx.save_for_backward(emb_t, emb_p, W, ln_g, ln_b, attn, starts, paths, ends, cv, att)
        ctx.cfg = (dims, drop_p, training, seed)
        ctx.cache = cache
        return cv, att

    @staticmethod
    def backward(ctx, d_cv, d_att):
        emb_t, emb_p, W, ln_g, ln_b, attn, starts, paths, ends, cv, att = ctx.saved_tensors
        dims, drop_p, training, seed = ctx.cfg
        if ctx.cache is not None:
            ctx.cache.raise_deferred()               # bad indices in the forward this backward belongs to
        params = CF.make_params(emb_t, emb_p, W, ln_g, ln_b, attn)
        shapes = {"terminal_embedding": emb_t.shape, "path_embedding": emb_p.shape, "input_linear": W.shape,
                  "ln_weight": ln_g.shape, "ln_bias": ln_b.shape, "attention": attn.shape}
        if d_cv is None:
            d_cv = torch.zeros_like(cv)
        # Fused gradient accumulation (opt-in, Code2Vec.fuse_grad_accumulation; what ddp_step switches on for the flat
        # optimizers): the embedding-table and input_linear gradients -- 99.9 % of the bytes -- are scatter-added straight into
        # the existing dense .grad buffers instead of into fresh zero-filled tensors that autograd would then add to .grad
        # (at cfg2: a 360 MB fill plus a 1.1 GB read-modify-write per step).  Autograd gets None for those three inputs.
        # sparse tables: the backward accumulates their rows into compact [U_max, E] buffers (row r -> row slot[r])
        maps = ctx.row_maps[0] if ctx.row_maps is not None else (None, None)
        compact = {k: torch.zeros((m[1].numel(), t.shape[1]), dtype=torch.float32, device=cv.device)
                   for k, m, t in (("terminal_embedding", maps[0], emb_t), ("path_embedding", maps[1], emb_p))
                   if m is not None}
        big = tuple((k, t) for k, t in (("terminal_embedding", emb_t), ("path_embedding", emb_p), ("input_linear", W))
                    if k not in compact)
        fuse = bool(getattr(ctx.cache, "fuse_grad_accumulation", False)) and all(
            t.grad is not None and t.grad.dtype == torch.float32 and t.grad.is_contiguous() and t.grad.shape == t.shape
            and t.grad.device == t.device for _, t in big)
        grads_out = None
        if fuse:
            grads_out = {k: t.grad for k, t in big}
            for k in ("ln_weight", "ln_bias", "attention"):
                grads_out[k] = torch.empty(shapes[k], dtype=torch.float32, device=cv.device)   # overwritten by the kernels
        elif compact:                                # (no dense buffer for a sparse table: its rows go to `compact`)
            grads_out = {k: torch.zeros(s, dtype=torch.float32, device=cv.device) for k, s in shapes.items()
                         if k not in compact}
        if compact:
            grads_out.update(compact)
        hook = getattr(ctx.cache, "on_path_grads_ready", None) if fuse and maps[1] is None else None
        slots = tuple(m[0] if m is not None else None for m in maps) if compact else None
        if ctx.bags is not None:
            g = CF.encode_backward_packed(dims, params, ctx.bags, cv, att, d_cv, d_att, shapes, drop_p, training, seed,
                                          grads_out=grads_out, x_stash=ctx.x_stash, between_phases=hook, slots=slots)
        else:
            g = CF.encode_backward(dims, params, starts, paths, ends, cv, att, d_cv, d_att, shapes, drop_p, training, seed,
                                   grads_out=grads_out, x_stash=ctx.x_stash, between_phases=hook, slots=slots)
        ctx.x_stash = None
        out = {k: (None if fuse else g[k]) for k in ("terminal_embedding", "path_embedding", "input_linear")}
        if compact:
            _, counts, ready = ctx.row_maps
            ready.synchronize()                      # U of each sparse table (the row maps were built in the forward)
            for i, (k, t) in enumerate((("terminal_embedding", emb_t), ("path_embedding", emb_p))):
                if k in compact:
                    U = int(counts[i])
                    rows = maps[i][1][:U].view(1, U)
                    out[k] = torch.sparse_coo_tensor(rows, compact[k][:U], t.shape, is_coalesced=True, check_invariants=False)
                    if ctx.cache is not None:            # what Code2Vec's post-accumulate hook recognises (is_coalesced)
                        ctx.cache.sparse_indices[k] = (rows.data_ptr(), U)
        return (out["terminal_embedding"], out["path_embedding"], out["input_linear"], g["ln_weight"], g["ln_bias"],
                g["attention"], None, None, None, None, None, None, None, None, None, None)


class _LabelFn(torch.autograd.Function):
    """outputs = cv . W_out^T + b   (model.py:83)"""

    @staticmethod
    def forward(ctx, cv, w_out, b_out, dims, algo, cache):
        params = CF.make_params(w_out=w_out, b_out=b_out)
        if any(ctx.needs_input_grad[:3]):
            algo = int(algo) | CF.NO_PDL            # the calls that feed autograd use plain stream-ordered launches
        out = CF.label_logits(dims, params, cv, algo, cache=cache, weight=w_out)
        ctx.save_for_backward(cv, w_out)
        ctx.dims, ctx.cache, ctx.algo = dims, cache, int(algo) & 0xff
        return out

    @staticmethod
    def backward(ctx, d_out):
        cv, w_out = ctx.saved_tensors
        params = CF.make_params(w_out=w_out)
        d_cv, d_w, d_b = CF.label_backward(ctx.dims, params, cv, d_out, ctx.needs_input_grad[0],
                                           ctx.needs_input_grad[1], ctx.needs_input_grad[2], algo=ctx.algo, cache=ctx.cache,
                                           weight=w_out)
        return d_cv, d_w, d_b, None, None, None


class _AngularFn(torch.autograd.Function):
    """angular-margin head (model.py:71-80) with its hand-written backward (c2v_angular_backward)"""

    @staticmethod
    def forward(ctx, cv, w_out, label, dims, margin, inverse_temp):
        params = CF.make_params(w_out=w_out)
        out, cos, inv = CF.angular_forward_train(dims, params, cv, label, margin, inverse_temp)
        ctx.save_for_backward(cv, w_out, label, cos, inv)
        ctx.cfg = (dims, margin, inverse_temp)
        return out

    @staticmethod
    def backward(ctx, d_out):
        cv, w_out, label, cos, inv = ctx.saved_tensors
        dims, margin, inverse_temp = ctx.cfg
        params = CF.make_params(w_out=w_out)
        d_cv, d_w = CF.angular_backward(dims, params, cv, label, margin, inverse_temp, cos, inv, d_out,
                                        ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        return d_cv, d_w, None, None, None, None


class _LabelLossFn(torch.autograd.Function):
    """mean NLL of log_softmax over the label head's logits (+ main.py:251-264) without materialising them: the label
    GEMM's epilogue produces loss / logsumexp / arg-max; the backward recomputes G = d loss / d logits tile by tile and
    runs the label backward on it.  angular=None: the plain head cv . W_out^T + b (model.py:83).
    angular=(margin, inverse_temp), b_out=None: the angular-margin head (model.py:71-80), whose G is d loss / d (cv . W^T)
    and whose backward then projects through F.normalize."""

    @staticmethod
    def forward(ctx, cv, w_out, b_out, label, dims, algo, cache, angular):
        params = CF.make_params(w_out=w_out, b_out=b_out)
        if any(ctx.needs_input_grad[:3]):
            algo = int(algo) | CF.NO_PDL            # the calls that feed autograd use plain stream-ordered launches
        if angular is None:
            loss, lse, am, mx, _ = CF.label_loss(dims, params, cv, label, algo=algo, cache=cache, weight=w_out)
            inv = None
        else:
            loss, lse, am, mx, inv, _ = CF.angular_loss(dims, params, cv, label, *angular, algo=algo, cache=cache, weight=w_out)
        ctx.save_for_backward(cv, w_out, b_out, label, lse, inv)
        ctx.dims, ctx.cache, ctx.algo, ctx.angular = dims, cache, algo, angular
        ctx.mark_non_differentiable(am, mx)
        return loss, am, mx

    @staticmethod
    def backward(ctx, d_loss, _d_am, _d_mx):
        cv, w_out, b_out, label, lse, inv = ctx.saved_tensors
        params = CF.make_params(w_out=w_out, b_out=b_out)
        dlogits = dict(scale_device=d_loss.reshape(1), algo=ctx.algo, cache=ctx.cache, weight=w_out)
        bw = dict(algo=int(ctx.algo) & 0xff, cache=ctx.cache, weight=w_out, absmax_ready=True)
        need, scale = ctx.needs_input_grad, 1.0 / cv.shape[0]
        if ctx.angular is None:
            g = CF.label_dlogits(ctx.dims, params, cv, label, lse, scale, **dlogits)
            d_cv, d_w, d_b = CF.label_backward(ctx.dims, params, cv, g, need[0], need[1], need[2], **bw)
        else:
            g = CF.angular_dlogits(ctx.dims, params, cv, label, lse, inv, *ctx.angular, scale, **dlogits)
            d_cv, d_w = CF.angular_backward_ws(ctx.dims, params, cv, g, inv, need[0], need[1], **bw)
            d_b = None
        return d_cv, d_w, d_b, None, None, None, None, None


class Code2Vec(nn.Module):
    """the code2vec model (H100-native drop-in for model.py:15-105)"""

    def __init__(self, option, algo="auto"):
        super(Code2Vec, self).__init__()
        self.option = option
        # same submodules, same order => same RNG consumption as model.py:21-42
        self.terminal_embedding = nn.Embedding(option.terminal_count, option.terminal_embed_size)
        self.path_embedding = nn.Embedding(option.path_count, option.path_embed_size)
        self.input_linear = nn.Linear(option.terminal_embed_size * 2 + option.path_embed_size, option.encode_size, bias=False)
        self.input_layer_norm = nn.LayerNorm(option.encode_size)

        if 0.0 < option.dropout_prob < 1.0:
            self.input_dropout = nn.Dropout(p=option.dropout_prob)   # holds p; the mask is made in-kernel
        else:
            self.input_dropout = None

        self.attention_parameter = Parameter(torch.nn.init.xavier_normal_(torch.zeros(option.encode_size, 1, dtype=torch.float32, requires_grad=True)).view(-1), requires_grad=True)

        if option.angular_margin_loss:
            self.output_linear = Parameter(torch.empty(option.label_count, option.encode_size, dtype=torch.float32))
            nn.init.xavier_uniform_(self.output_linear)
            self.cos_m = math.cos(option.angular_margin)
            self.sin_m = math.sin(option.angular_margin)
            self.th = math.cos(math.pi - option.angular_margin)
            self.mm = math.sin(math.pi - option.angular_margin) * option.angular_margin
        else:
            self.output_linear = nn.Linear(option.encode_size, option.label_count, bias=True)
            self.output_linear.bias.data.fill_(0.0)

        self.algo = {"auto": _lib.ALGO_AUTO, "ffma": _lib.ALGO_FFMA, "tcgen05": _lib.ALGO_TCGEN05}[algo]
        # the label head takes the tensor cores wherever its shape allows them, unless algo="ffma"
        self._label_algo = _lib.ALGO_FFMA if self.algo == _lib.ALGO_FFMA else _lib.ALGO_AUTO
        self._dropout_calls = 0
        # persistent workspaces: the hi/lo split images of input_linear / output_linear are rebuilt
        # only when the optimizer changed the weights (tracked by the tensors' version counters)
        self._enc_cache = CF.PrepCache(mirror_errors=True)
        # True: the backward adds the table / input_linear gradients directly into the parameters' existing .grad buffers
        # (see _EncodeFn.backward); needs dense fp32 .grad tensors to exist before the backward, e.g. a flat gradient bucket
        self.fuse_grad_accumulation = False
        # callable run by the backward once path_embedding's gradient is complete (fused accumulation only): the sharded
        # optimizer starts that table's data-parallel reduction there (ShardedFlatAdam.early_step)
        self.on_path_grads_ready = None
        self._lab_cache = CF.PrepCache()
        # sparse embedding gradients (opt-in: terminal_embedding.sparse / path_embedding.sparse, as on nn.Embedding)
        self._enc_cache.sparse_indices = {}
        self._sparse_hooks = None

    # -- helpers ---------------------------------------------------------------------------
    def _dims(self):
        o = self.option
        return CF.make_dims(o.terminal_count, o.path_count, o.label_count, o.terminal_embed_size,
                            o.path_embed_size, o.encode_size)

    def _next_seed(self):
        # one Philox key per training forward, drawn from torch's CPU generator so that
        # torch.manual_seed (main.py:120) makes runs repeatable
        self._dropout_calls += 1
        return int(torch.randint(0, 2 ** 62, (1,)).item())

    def _head(self):
        """-> (W_out, b_out) of the label head; the angular-margin head has no bias"""
        if self.option.angular_margin_loss:
            return self.output_linear, None
        return self.output_linear.weight, self.output_linear.bias

    def _encode(self, starts, paths, ends):
        """the encode of forward() / forward_loss(), autograd-connected -> (code_vector, attention, dims)"""
        self._enc_cache.raise_deferred()
        self._enc_cache.fuse_grad_accumulation = self.fuse_grad_accumulation
        self._enc_cache.on_path_grads_ready = self.on_path_grads_ready
        dims = self._dims()
        training = self.training and self.input_dropout is not None
        drop_p = float(self.option.dropout_prob) if training else 0.0
        seed = self._next_seed() if training else 0
        sparse = (bool(self.terminal_embedding.sparse), bool(self.path_embedding.sparse))
        if any(sparse):
            self._watch_sparse_grads()
        code_vector, attention = _EncodeFn.apply(
            self.terminal_embedding.weight, self.path_embedding.weight, self.input_linear.weight,
            self.input_layer_norm.weight, self.input_layer_norm.bias, self.attention_parameter,
            starts, paths, ends, dims, drop_p, training, seed, self.algo, self._enc_cache, sparse)
        return code_vector, attention, dims

    def _watch_sparse_grads(self):
        """Sparse embedding gradients leave the backward coalesced, but torch's AccumulateGrad drops that flag when it
        makes the tensor the parameter's .grad.  A post-accumulate hook on each table sets it back when .grad's indices are
        the very tensor the backward produced (a first backward into an empty .grad); after accumulation over several
        backwards the flag stays whatever torch made it.  Registered once, on the first forward with a sparse table."""
        if self._sparse_hooks:
            return
        cache = self._enc_cache

        def mark(key):
            def hook(p):
                g, made = p.grad, cache.sparse_indices.pop(key, None)
                if g is not None and g.is_sparse and made is not None and not g.is_coalesced():
                    ind = g._indices()
                    if (ind.data_ptr(), ind.shape[1]) == made:
                        g._coalesced_(True)
            return hook
        self._sparse_hooks = [self.terminal_embedding.weight.register_post_accumulate_grad_hook(mark("terminal_embedding")),
                              self.path_embedding.weight.register_post_accumulate_grad_hook(mark("path_embedding"))]

    def _encode_eval(self, starts, paths, ends):
        """the encode of predict() / predict_topk(), without autograd or dropout -> (code_vector, attention, dims)"""
        self._enc_cache.raise_deferred()
        dims = self._dims()
        params = CF.make_params(self.terminal_embedding.weight, self.path_embedding.weight, self.input_linear.weight,
                                self.input_layer_norm.weight, self.input_layer_norm.bias, self.attention_parameter)
        if isinstance(starts, CF.PackedBags):
            code_vector, attention = CF.encode_forward_packed(dims, params, starts, algo=self.algo, cache=self._enc_cache,
                                                              weight=self.input_linear.weight)
        else:
            code_vector, attention = CF.encode_forward(dims, params, starts, paths, ends, algo=self.algo,
                                                       cache=self._enc_cache, weight=self.input_linear.weight)
        return code_vector, attention, dims

    def _head_logits(self, code_vector, label, dims):
        """forward()'s logits: model.py:83, or the angular-margin head (model.py:71-80) on the CUDA cores"""
        option = self.option
        if not option.angular_margin_loss:
            return _LabelFn.apply(code_vector, *self._head(), dims, self._label_algo, self._lab_cache)
        if torch.is_grad_enabled() and (code_vector.requires_grad or self.output_linear.requires_grad):
            return _AngularFn.apply(code_vector, self.output_linear, label, dims, option.angular_margin, option.inverse_temp)
        params = CF.make_params(w_out=self.output_linear)
        return CF.angular_logits(dims, params, code_vector, label, option.angular_margin, option.inverse_temp)

    @staticmethod
    def _eager_loss(outputs, label):
        """forward_loss() from materialised logits: eager log_softmax / NLL (main.py:251-264) + torch.max (main.py:285)"""
        loss = F.nll_loss(F.log_softmax(outputs, dim=1), label)
        mx, am = torch.max(outputs.detach(), dim=1)
        return loss, am, mx

    # -- the reference surface -------------------------------------------------------------
    def check_indices(self):
        """Synchronise and raise IndexError if any forward so far saw an index outside the embedding tables
        (`forward` itself raises it one call late, without synchronising: see functional.PrepCache.raise_deferred)."""
        self._enc_cache.raise_deferred(synchronize=True)

    # Every entry point below also takes a functional.PackedBags batch in place of `starts`, with paths = ends = None: the
    # encode then runs over its N contexts only (no padding rows), attention comes back as [N], aligned with the packed
    # contexts, and the label heads run unchanged on the [b, H] code vectors.
    def forward(self, starts, paths, ends, label):
        code_vector, attention, dims = self._encode(starts, paths, ends)
        return self._head_logits(code_vector, label, dims), code_vector, attention

    # -- additive fast path: forward + calculate_loss (main.py:251-264) + torch.max (main.py:285) -----
    def forward_loss(self, starts, paths, ends, label):
        """-> (loss, pred_label [b], pred_score [b], code_vector [b,H], attention [b,L]); loss is the mean NLL the
        reference's `calculate_loss(preds, label, criterion, option)` returns (criterion weights are all
        1) and is autograd-connected; the [b, C] logits are never written.  Both label heads: with
        option.angular_margin_loss the loss, arg-max and max are those of the angular-margin logits (model.py:71-80).
        Shapes the fused kernel does not take, and algo="ffma", fall back to forward()'s head + eager log_softmax / NLL +
        torch.max."""
        code_vector, attention, dims = self._encode(starts, paths, ends)
        if self.algo != _lib.ALGO_FFMA and CF.label_loss_supported(dims, code_vector.shape[0]):
            o = self.option
            angular = (o.angular_margin, o.inverse_temp) if o.angular_margin_loss else None
            loss, am, mx = _LabelLossFn.apply(code_vector, *self._head(), label, dims, self._label_algo, self._lab_cache,
                                              angular)
        else:
            loss, am, mx = self._eager_loss(self._head_logits(code_vector, label, dims), label)
        return loss, am, mx, code_vector, attention

    # -- additive convenience (the reference does torch.max(preds, dim=1) at main.py:285) ----
    @torch.no_grad()
    def predict(self, starts, paths, ends):
        """-> (pred_label [b], pred_score [b], code_vector [b,H], attention [b,L])"""
        if self.option.angular_margin_loss:
            raise NotImplementedError("predict() needs the plain label head (the angular head needs labels)")
        code_vector, attention, dims = self._encode_eval(starts, paths, ends)
        w_out, b_out = self._head()
        _, am, mx = CF.label_logits_argmax(dims, CF.make_params(w_out=w_out, b_out=b_out), code_vector, self._label_algo,
                                           cache=self._lab_cache, weight=w_out, want_logits=False)
        return am, mx, code_vector, attention

    _TOPK_ROWS = 2048                   # rows per fused top-k call (c2v_label_topk_supported)

    @torch.no_grad()
    def predict_topk(self, starts, paths, ends, k=10, probs=True):
        """-> (pred_labels int64 [b, k], pred_scores [b, k], pred_probs [b, k] or None, code_vector [b,H], attention [b,L]):
        the k best labels of every method, best first, ranked as torch.sort(logits, 1, descending=True, stable=True) ranks
        them (equal scores: the lower label index first; k=1 is predict()), their scores and, with probs=True, their softmax
        probabilities.  Plain head: the logits of forward().  Angular-margin head: inverse_temp * cos(code_vector, W_c),
        without the margin, so no label is needed (predict_topk(k=1) is that head's prediction).
        The label GEMM keeps a running top-k in its epilogue and never writes the [b, C] logits (b is cut into chunks of
        2048 rows).  k > _lib.TOPK_MAX, encode sizes the fused kernel does not take and algo="ffma" materialise the
        logits and sort them instead."""
        k = int(k)
        C = self.option.label_count
        if not 1 <= k <= C:
            raise ValueError(f"predict_topk: k = {k} is outside [1, label_count = {C}]")
        code_vector, attention, dims = self._encode_eval(starts, paths, ends)
        angular = self.option.angular_margin_loss
        w_out, b_out = self._head()
        params = CF.make_params(w_out=w_out, b_out=b_out)
        b = code_vector.shape[0]
        if self.algo != _lib.ALGO_FFMA and CF.label_topk_supported(dims, min(b, self._TOPK_ROWS), k):
            parts = []
            for i in range(0, b, self._TOPK_ROWS):
                cv = code_vector[i:i + self._TOPK_ROWS]
                if angular:
                    parts.append(CF.angular_topk(dims, params, cv, k, self.option.inverse_temp, want_probs=probs,
                                                 cache=self._lab_cache, weight=w_out))
                else:
                    parts.append(CF.label_topk(dims, params, cv, k, want_probs=probs, cache=self._lab_cache, weight=w_out))
            idx, val, prob = (torch.cat(t) if t[0] is not None else None for t in zip(*parts))
            return idx, val, prob, code_vector, attention
        if angular:
            logits = self.option.inverse_temp * F.linear(F.normalize(code_vector), F.normalize(w_out))
        else:
            logits = CF.label_logits(dims, params, code_vector, self._label_algo, cache=self._lab_cache, weight=w_out)
        val, idx = torch.sort(logits, dim=1, descending=True, stable=True)
        val, idx = val[:, :k].contiguous(), idx[:, :k].contiguous()
        prob = torch.softmax(logits, dim=1).gather(1, idx) if probs else None
        return idx, val, prob, code_vector, attention

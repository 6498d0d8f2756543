"""torch-facing wrappers over the C ABI: device memory, streams and autograd plumbing only.
All arithmetic happens inside libc2v_b200.so."""
import ctypes
import os

import torch

from . import _lib
from ._lib import Dims, Dropout, Grads, Params, RowSlots


# C2V_POISON=1: every buffer handed to the library uninitialised (workspaces, outputs, stashes) is filled with 0xFF bytes
# (fp32 NaN / int -1) first, so that a read of memory the current call did not write shows up as NaN instead of hiding
# behind whatever an earlier, identical call left there (debugging aid).
_POISON = os.environ.get("C2V_POISON", "0") == "1"


def _empty(shape, dtype, device):
    t = torch.empty(shape, dtype=dtype, device=device)
    if _POISON:
        if t.numel():
            t.reshape(-1).view(torch.uint8).fill_(255)
    return t


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _need_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise _lib.C2VError(
                "code2vec_b200 runs on CUDA (sm_90a) only and has no CPU fallback: got a "
                f"{t.device} tensor. Move the module and its inputs to an H100 device.")


def _f32c(t, name):
    """contiguous fp32 CUDA tensor (the caller keeps the returned object alive across the library call)"""
    if t.dtype != torch.float32 or not t.is_cuda:
        raise TypeError(f"{name} must be a float32 CUDA tensor, got {t.dtype} on {t.device}")
    return t.contiguous()


def _idx(t, name, shape=None):
    if t.dtype != torch.int64:
        raise TypeError(f"{name} must be int64 (dataset_builder.py:206-209), got {t.dtype}")
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise ValueError(f"{name} has shape {tuple(t.shape)}, expected {tuple(shape)}")
    return t.contiguous()


def make_dims(T, P, C, Et, Ep, H):
    return Dims(int(T), int(P), int(C), int(Et), int(Ep), int(H), 0)


def make_params(emb_t=None, emb_p=None, W=None, ln_g=None, ln_b=None, attn=None, w_out=None, b_out=None):
    for t in (emb_t, emb_p, W, ln_g, ln_b, attn, w_out, b_out):
        if t is not None and (t.dtype != torch.float32 or not t.is_contiguous()):
            raise TypeError("parameters must be contiguous fp32")
    p = Params(_ptr(emb_t), _ptr(emb_p), _ptr(W), _ptr(ln_g), _ptr(ln_b), _ptr(attn), _ptr(w_out), _ptr(b_out))
    p._keep = (emb_t, emb_p, W, ln_g, ln_b, attn, w_out, b_out)   # the struct holds raw pointers: pin the tensors
    return p


REUSE_PREP = 0x100
NO_PDL = 0x200
GRAD_ABSMAX_READY = 0x400


class PrepCache:
    """A persistent workspace whose derived weight images (split / transposed copies of a weight
    matrix) are rebuilt only when the weight changed: keyed on (data_ptr, _version, size)."""

    def __init__(self, mirror_errors=False):
        self.buf, self.key = None, None
        # encode workspaces: a pinned host word the finalize kernel adds its out-of-range index count to
        # (c2v_workspace_set_status_mirror), polled by raise_deferred() at the next call on this cache
        self.mirror_errors, self.err = mirror_errors, None       # (pinned memory needs the driver: allocated on first use)

    def get(self, nbytes, device, weight):
        key = (weight.data_ptr(), weight._version, str(device))
        fresh = self.buf is None or self.buf.numel() < nbytes or self.buf.device != device
        if fresh:
            self.buf = _empty((nbytes,), torch.uint8, device)
            if self.mirror_errors:
                if self.err is None:
                    self.err = torch.zeros(1, dtype=torch.int64).pin_memory()
                lib = _lib.load()
                with torch.cuda.device(device):
                    _lib.check(lib.c2v_workspace_set_status_mirror(_ptr(self.buf), ctypes.c_void_p(self.err.data_ptr()),
                                                                   _stream(device)), "c2v_workspace_set_status_mirror")
        reuse = (not fresh) and key == self.key
        self.key = key
        return self.buf, reuse

    def raise_deferred(self, synchronize=False):
        """IndexError for out-of-range indices of an EARLIER forward on this cache (the kernels clamp them to row 0 and
        count; the reference raises IndexError on CPU and device-asserts -- equally late -- on CUDA).  No sync unless asked."""
        if self.err is None:
            return
        if synchronize and self.buf is not None:
            torch.cuda.synchronize(self.buf.device)
        n = int(self.err[0])
        if n:
            self.err[0] = 0
            raise IndexError(f"index out of range in self ({n} start/path/end indices outside the embedding tables in an "
                             "earlier forward of this module; they were read as row 0)")


def encode_forward(dims, params, starts, paths, ends, drop_p=0.0, training=False, seed=0, algo=_lib.ALGO_AUTO,
                   check_indices=False, cache=None, weight=None, stash=False):
    """-> (code_vector [B,H], attention [B,L]); model.py:48-69 + 90-96.
    stash=True (training): also returns x = c . W^T [B*L, H] for encode_backward(x_stash=...), which then skips the
    re-gather and the recompute GEMM."""
    lib = _lib.load()
    _need_cuda(starts, paths, ends)
    B, L = starts.shape
    starts = _idx(starts, "starts"); paths = _idx(paths, "paths", (B, L)); ends = _idx(ends, "ends", (B, L))
    dev = starts.device
    with torch.cuda.device(dev):
        cv = _empty((B, dims.encode), torch.float32, dev)
        att = _empty((B, L), torch.float32, dev)
        nbytes = lib.c2v_encode_workspace_bytes(ctypes.byref(dims), B, L)
        if cache is not None and weight is not None:
            ws, reuse = cache.get(nbytes, dev, weight)
            if reuse:
                algo = int(algo) | REUSE_PREP
        else:
            ws = _empty((nbytes,), torch.uint8, dev)
        drop = Dropout(float(drop_p), 1 if training else 0, int(seed))
        xs = _empty((B * L, dims.encode), torch.float32, dev) if stash else None
        rc = lib.c2v_encode_forward_stash(ctypes.byref(dims), ctypes.byref(params), _ptr(starts), _ptr(paths), _ptr(ends),
                                          B, L, ctypes.byref(drop), _ptr(cv), _ptr(att), _ptr(xs), _ptr(ws), ws.numel(),
                                          int(algo), _stream(dev))
        _lib.check(rc, "c2v_encode_forward")
        if check_indices:
            bad = lib.c2v_workspace_status(_ptr(ws), _stream(dev))
            if bad > 0:
                raise IndexError("index out of range in self")
            if bad < 0:
                _lib.check(int(bad), "c2v_workspace_status")
    if stash:
        return cv, att, xs
    return cv, att


class PackedBags:
    """A batch of variable-length bags in CSR form, without padding rows: bag b is contexts offsets[b] .. offsets[b+1]-1
    of starts / paths / ends (int64 [N]).  Bag b is row b of the [B, L] batch without its zero-padded suffix, so every bag
    holds 1 .. max_path_length contexts; a method with no contexts is a bag of one pad context (0, 0, 0).

    The offsets (int64 [B + 1]) are validated on the host here -- offsets[0] = 0, non-decreasing, offsets[B] = N, every
    bag length in [1, max_path_length] -- so that no malformed batch reaches a kernel.  Given as a host tensor / array /
    list that costs nothing; given as a CUDA tensor it costs one device-to-host copy (and a synchronisation).
    DeviceCorpus.build_packed computes them on the host and never pays it.

    device_offsets: the same offsets already on the device of starts (no upload then); the caller guarantees that they hold
    the values of `offsets`, which are the ones validated.

    Attributes: starts / paths / ends [N] and offsets [B + 1] on the device of starts; offsets_host (numpy int64), B, N,
    L (= max_path_length)."""

    def __init__(self, starts, paths, ends, offsets, max_path_length, device_offsets=None):
        import numpy as np
        L = int(max_path_length)
        if L < 1:
            raise ValueError(f"PackedBags: max_path_length = {L} < 1")
        if isinstance(offsets, torch.Tensor):
            host = offsets.detach().to("cpu", torch.int64).numpy()
        else:
            host = np.asarray(offsets, dtype=np.int64)
        host = np.ascontiguousarray(host, dtype=np.int64)
        for name, t in (("starts", starts), ("paths", paths), ("ends", ends)):
            if not isinstance(t, torch.Tensor) or t.dim() != 1:
                raise ValueError(f"PackedBags: {name} must be a 1-D int64 tensor [N]")
        N = int(starts.numel())
        if paths.numel() != N or ends.numel() != N:
            raise ValueError(f"PackedBags: starts / paths / ends hold {N} / {paths.numel()} / {ends.numel()} contexts")
        if host.ndim != 1 or host.size < 2:
            raise ValueError("PackedBags: offsets must be 1-D with B + 1 >= 2 entries")
        if host[0] != 0 or host[-1] != N:
            raise ValueError(f"PackedBags: offsets[0] = {host[0]} and offsets[B] = {host[-1]} must be 0 and N = {N}")
        n = np.diff(host)
        if (n < 1).any() or (n > L).any():
            b = int(np.flatnonzero((n < 1) | (n > L))[0])
            raise ValueError(f"PackedBags: bag {b} holds {int(n[b])} contexts; every bag needs 1 .. {L} "
                             "(offsets must increase)")
        self.starts = _idx(starts, "starts"); self.paths = _idx(paths, "paths"); self.ends = _idx(ends, "ends")
        self.offsets_host = host
        if device_offsets is not None:
            if device_offsets.dtype != torch.int64 or device_offsets.device != starts.device or \
                    tuple(device_offsets.shape) != host.shape:
                raise ValueError("PackedBags: device_offsets must be int64 [B + 1] on the device of starts")
            self.offsets = device_offsets.contiguous()
        elif isinstance(offsets, torch.Tensor):
            self.offsets = offsets.to(device=starts.device, dtype=torch.int64).contiguous()
        else:
            self.offsets = torch.from_numpy(host.copy()).to(starts.device)
        self.B, self.N, self.L = int(host.size - 1), N, L

    @property
    def device(self):
        return self.starts.device

    def lengths(self):
        """host numpy int64 [B]: contexts per bag"""
        import numpy as np
        return np.diff(self.offsets_host)

    def padded(self):
        """-> (starts, paths, ends) int64 [B, L] on the device: the same batch with a zero-padded suffix per bag"""
        import numpy as np
        n = self.lengths()
        rows = np.repeat(np.arange(self.B), n)
        cols = np.arange(self.N) - np.repeat(self.offsets_host[:-1], n)
        flat = torch.from_numpy(rows * self.L + cols).to(self.device)
        out = []
        for t in (self.starts, self.paths, self.ends):
            p = torch.zeros(self.B * self.L, dtype=torch.int64, device=self.device)
            p[flat] = t
            out.append(p.view(self.B, self.L))
        return tuple(out)


def encode_forward_packed(dims, params, bags, drop_p=0.0, training=False, seed=0, algo=_lib.ALGO_AUTO,
                          check_indices=False, cache=None, weight=None, stash=False):
    """encode_forward for a PackedBags batch -> (code_vector [B,H], attention [N]) (+ x_stash [N, H] with stash=True).
    The code vector of a bag equals the [B, L] result of the same bag up to fp32 summation order; packed context j of bag
    b draws the dropout mask of padded row b * L + j."""
    lib = _lib.load()
    _need_cuda(bags.starts, bags.paths, bags.ends, bags.offsets)
    B, N, L = bags.B, bags.N, bags.L
    dev = bags.device
    with torch.cuda.device(dev):
        cv = _empty((B, dims.encode), torch.float32, dev)
        att = _empty((N,), torch.float32, dev)
        nbytes = lib.c2v_encode_packed_workspace_bytes(ctypes.byref(dims), B, N)
        if cache is not None and weight is not None:
            ws, reuse = cache.get(nbytes, dev, weight)
            if reuse:
                algo = int(algo) | REUSE_PREP
        else:
            ws = _empty((nbytes,), torch.uint8, dev)
        drop = Dropout(float(drop_p), 1 if training else 0, int(seed))
        xs = _empty((N, dims.encode), torch.float32, dev) if stash else None
        rc = lib.c2v_encode_forward_packed(ctypes.byref(dims), ctypes.byref(params), _ptr(bags.starts), _ptr(bags.paths),
                                           _ptr(bags.ends), _ptr(bags.offsets), B, N, L, ctypes.byref(drop), _ptr(cv),
                                           _ptr(att), _ptr(xs), _ptr(ws), ws.numel(), int(algo), _stream(dev))
        _lib.check(rc, "c2v_encode_forward_packed")
        if check_indices:
            bad = lib.c2v_workspace_status(_ptr(ws), _stream(dev))
            if bad > 0:
                raise IndexError("index out of range in self")
            if bad < 0:
                _lib.check(int(bad), "c2v_workspace_status")
    if stash:
        return cv, att, xs
    return cv, att


def _label_ws(dims, B, dev, algo, cache, weight, nbytes=None, absmax_ready=False, fresh=True):
    """-> (workspace, algo with its flags) of a label-head call.  With a cache (and its weight, W_out) the cache's persistent
    workspace, plus REUSE_PREP while its W_out image is current and GRAD_ABSMAX_READY if absmax_ready.  Without one a fresh
    workspace, or None if not fresh (the backward calls then run on the CUDA cores)."""
    if nbytes is None:
        nbytes = _lib.load().c2v_label_workspace_bytes(ctypes.byref(dims), B)
    if cache is not None and weight is not None:
        ws, reuse = cache.get(nbytes, dev, weight)
        return ws, int(algo) | (REUSE_PREP if reuse else 0) | (GRAD_ABSMAX_READY if absmax_ready else 0)
    return (_empty((nbytes,), torch.uint8, dev) if fresh else None), int(algo)


def label_logits(dims, params, cv, algo=_lib.ALGO_AUTO, cache=None, weight=None):
    """model.py:83"""
    lib = _lib.load()
    _need_cuda(cv)
    B = cv.shape[0]
    dev = cv.device
    with torch.cuda.device(dev):
        out = _empty((B, dims.label_count), torch.float32, dev)
        ws, algo = _label_ws(dims, B, dev, algo, cache, weight)
        cv = _f32c(cv, "code_vector")          # bound to a local: the pointer must outlive the launch
        rc = lib.c2v_label_logits(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), B, _ptr(out),
                                  _ptr(ws), ws.numel(), int(algo), _stream(dev))
        _lib.check(rc, "c2v_label_logits")
    return out


def label_logits_argmax(dims, params, cv, algo=_lib.ALGO_AUTO, cache=None, weight=None, want_logits=True):
    """model.py:83 + main.py:285 fused -> (outputs [B,C] or None, argmax int64 [B], maxval [B])"""
    lib = _lib.load()
    _need_cuda(cv)
    B = cv.shape[0]
    dev = cv.device
    if not want_logits and ((int(algo) & 0xff) == _lib.ALGO_FFMA or not label_loss_supported(dims, B)):
        want_logits = True                      # the CUDA-core / B > 2048 paths take the arg-max from stored logits
    with torch.cuda.device(dev):
        out = _empty((B, dims.label_count), torch.float32, dev) if want_logits else None
        am = _empty((B,), torch.int64, dev)
        mx = _empty((B,), torch.float32, dev)
        ws, algo = _label_ws(dims, B, dev, algo, cache, weight)
        cv = _f32c(cv, "code_vector")
        rc = lib.c2v_label_logits_argmax(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), B, _ptr(out),
                                         _ptr(am), _ptr(mx), _ptr(ws), ws.numel(), int(algo), _stream(dev))
        _lib.check(rc, "c2v_label_logits_argmax")
    return out, am, mx


def label_loss_supported(dims, B):
    return bool(_lib.load().c2v_label_loss_supported(ctypes.byref(dims), int(B)))


def label_loss(dims, params, cv, label, want_logits=False, algo=_lib.ALGO_AUTO, cache=None, weight=None):
    """model.py:83 + main.py:251-264 + main.py:285 in one pass over the label GEMM's accumulators
    -> (loss 0-d, lse [B], argmax int64 [B], maxval [B], outputs [B, C] or None).  With want_logits=False the [B, C]
    logits are never written (nor re-read)."""
    lib = _lib.load()
    _need_cuda(cv, label)
    B = cv.shape[0]
    dev = cv.device
    label = _idx(label, "label", (B,))
    with torch.cuda.device(dev):
        out = _empty((B, dims.label_count), torch.float32, dev) if want_logits else None
        loss = _empty((), torch.float32, dev)
        lse = _empty((B,), torch.float32, dev)
        am = _empty((B,), torch.int64, dev)
        mx = _empty((B,), torch.float32, dev)
        ws, algo = _label_ws(dims, B, dev, algo, cache, weight)
        cv = _f32c(cv, "code_vector")
        rc = lib.c2v_label_loss_argmax(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), _ptr(label), B, _ptr(out),
                                       _ptr(loss), _ptr(lse), _ptr(am), _ptr(mx), _ptr(ws), ws.numel(), int(algo),
                                       _stream(dev))
        _lib.check(rc, "c2v_label_loss_argmax")
    return loss, lse, am, mx, out


def label_dlogits(dims, params, cv, label, lse, scale, scale_device=None, algo=_lib.ALGO_AUTO, cache=None, weight=None):
    """d(mean NLL)/d(outputs) [B, C] = (softmax - onehot) * scale (* scale_device[0]), recomputed from cv and W_out"""
    lib = _lib.load()
    B = cv.shape[0]
    dev = cv.device
    with torch.cuda.device(dev):
        dout = _empty((B, dims.label_count), torch.float32, dev)
        ws, algo = _label_ws(dims, B, dev, algo, cache, weight)
        cv = _f32c(cv, "code_vector"); lse = _f32c(lse, "lse")
        sd = _f32c(scale_device, "scale_device") if scale_device is not None else None
        rc = lib.c2v_label_dlogits(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), _ptr(label), _ptr(lse), B,
                                   float(scale), _ptr(sd), _ptr(dout), _ptr(ws), ws.numel(), int(algo), _stream(dev))
        _lib.check(rc, "c2v_label_dlogits")
    return dout


def angular_loss(dims, params, cv, label, margin, inverse_temp, want_logits=False, algo=_lib.ALGO_AUTO, cache=None,
                 weight=None):
    """model.py:71-80 + main.py:251-264 + main.py:285 in one pass over the label GEMM's accumulators
    -> (loss 0-d, lse [B], argmax int64 [B], maxval [B], inv_norms [B + C], outputs [B, C] or None).  inv_norms is what
    angular_dlogits / angular_backward_ws need; with want_logits=False the [B, C] logits are never written."""
    lib = _lib.load()
    _need_cuda(cv, label)
    B = cv.shape[0]
    dev = cv.device
    label = _idx(label, "label", (B,))
    with torch.cuda.device(dev):
        out = _empty((B, dims.label_count), torch.float32, dev) if want_logits else None
        loss = _empty((), torch.float32, dev)
        lse = _empty((B,), torch.float32, dev)
        am = _empty((B,), torch.int64, dev)
        mx = _empty((B,), torch.float32, dev)
        inv = _empty((B + dims.label_count,), torch.float32, dev)
        ws, algo = _label_ws(dims, B, dev, algo, cache, weight)
        cv = _f32c(cv, "code_vector")
        rc = lib.c2v_angular_loss_argmax(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), _ptr(label), B, float(margin),
                                         float(inverse_temp), _ptr(out), _ptr(loss), _ptr(lse), _ptr(am), _ptr(mx), _ptr(inv),
                                         _ptr(ws), ws.numel(), int(algo), _stream(dev))
        _lib.check(rc, "c2v_angular_loss_argmax")
    return loss, lse, am, mx, inv, out


def label_topk_supported(dims, B, k):
    return bool(_lib.load().c2v_label_topk_supported(ctypes.byref(dims), int(B), int(k)))


def _topk(fn, dims, params, cv, k, want_probs, algo, cache, weight, *head_args):
    lib = _lib.load()
    _need_cuda(cv)
    B, k = cv.shape[0], int(k)
    dev = cv.device
    with torch.cuda.device(dev):
        idx = _empty((B, k), torch.int64, dev)
        val = _empty((B, k), torch.float32, dev)
        prob = _empty((B, k), torch.float32, dev) if want_probs else None
        ws = None                    # a call the library will refuse must not mark the cache's weight image as current
        if (int(algo) & 0xff) != _lib.ALGO_FFMA and label_topk_supported(dims, B, k):
            nbytes = lib.c2v_label_topk_workspace_bytes(ctypes.byref(dims), B, k)
            ws, algo = _label_ws(dims, B, dev, algo, cache, weight, nbytes=nbytes)
        cv = _f32c(cv, "code_vector")
        rc = getattr(lib, fn)(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), B, k, *head_args, _ptr(idx), _ptr(val),
                              _ptr(prob), _ptr(ws), ws.numel() if ws is not None else 0, int(algo), _stream(dev))
        _lib.check(rc, fn)
    return idx, val, prob


def label_topk(dims, params, cv, k, want_probs=True, algo=_lib.ALGO_AUTO, cache=None, weight=None):
    """the k largest logits of model.py:83 per row, ranked as torch.sort(descending=True, stable=True) ranks them, from
    the label GEMM's epilogue (the [B, C] logits are never written) -> (indices int64 [B, k], values [B, k],
    softmax probabilities [B, k] or None).  B <= 2048 and k <= _lib.TOPK_MAX (label_topk_supported)."""
    return _topk("c2v_label_topk", dims, params, cv, k, want_probs, algo, cache, weight)


def angular_topk(dims, params, cv, k, inverse_temp, want_probs=True, algo=_lib.ALGO_AUTO, cache=None, weight=None):
    """label_topk for the angular head (model.py:71-80) without its margin: logits inverse_temp * cos(cv, W_c), no label"""
    return _topk("c2v_angular_topk", dims, params, cv, k, want_probs, algo, cache, weight, ctypes.c_float(inverse_temp))


def angular_dlogits(dims, params, cv, label, lse, inv_norms, margin, inverse_temp, scale, scale_device=None,
                    algo=_lib.ALGO_AUTO, cache=None, weight=None):
    """d(mean NLL)/d(cv . W^T) [B, C] of the angular head (scale and scale_device as in label_dlogits), recomputed from
    cv and W_out"""
    lib = _lib.load()
    B = cv.shape[0]
    dev = cv.device
    label = _idx(label, "label", (B,))
    with torch.cuda.device(dev):
        g = _empty((B, dims.label_count), torch.float32, dev)
        ws, algo = _label_ws(dims, B, dev, algo, cache, weight)
        cv = _f32c(cv, "code_vector"); lse = _f32c(lse, "lse"); inv = _f32c(inv_norms, "inv_norms")
        sd = _f32c(scale_device, "scale_device") if scale_device is not None else None
        rc = lib.c2v_angular_dlogits(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), _ptr(label), _ptr(lse), _ptr(inv), B,
                                     float(margin), float(inverse_temp), float(scale), _ptr(sd), _ptr(g), _ptr(ws), ws.numel(),
                                     int(algo), _stream(dev))
        _lib.check(rc, "c2v_angular_dlogits")
    return g


def angular_backward_ws(dims, params, cv, d_dot, inv_norms, need_cv=True, need_w=True, algo=_lib.ALGO_AUTO, cache=None,
                        weight=None, absmax_ready=False):
    """backward of the angular head from G = angular_dlogits(...) -> (d_code_vector, d_output_weight).  With the label
    PrepCache of the forward (cache + weight) the contractions run on the tensor cores and stream the cached W_out image;
    absmax_ready: d_dot is the tensor angular_dlogits just returned for the same cache."""
    lib = _lib.load()
    B = cv.shape[0]
    dev = cv.device
    with torch.cuda.device(dev):
        d_cv = torch.empty_like(cv) if need_cv else None
        d_w = _empty((dims.label_count, dims.encode), torch.float32, dev) if need_w else None
        cv = _f32c(cv, "code_vector"); d_dot = _f32c(d_dot, "d_dot"); inv = _f32c(inv_norms, "inv_norms")
        ws, flags = _label_ws(dims, B, dev, algo, cache, weight, absmax_ready=absmax_ready, fresh=False)
        rc = lib.c2v_angular_backward_ws(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), _ptr(d_dot), _ptr(inv), B,
                                         _ptr(d_cv), _ptr(d_w), _ptr(ws), ws.numel() if ws is not None else 0, flags,
                                         _stream(dev))
        _lib.check(rc, "c2v_angular_backward_ws")
    return d_cv, d_w


def angular_logits(dims, params, cv, label, margin, inverse_temp):
    """model.py:71-80"""
    lib = _lib.load()
    _need_cuda(cv, label)
    B = cv.shape[0]
    dev = cv.device
    label = _idx(label, "label", (B,))
    with torch.cuda.device(dev):
        out = _empty((B, dims.label_count), torch.float32, dev)
        cv = _f32c(cv, "code_vector")
        rc = lib.c2v_angular_logits(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), _ptr(label), B,
                                    float(margin), float(inverse_temp), _ptr(out), _stream(dev))
        _lib.check(rc, "c2v_angular_logits")
    return out


def angular_forward_train(dims, params, cv, label, margin, inverse_temp):
    """model.py:71-80 for a forward that will be differentiated -> (outputs, cosine [B, C], inv_norms [B + C])"""
    lib = _lib.load()
    _need_cuda(cv, label)
    B = cv.shape[0]
    dev = cv.device
    label = _idx(label, "label", (B,))
    with torch.cuda.device(dev):
        out = _empty((B, dims.label_count), torch.float32, dev)
        cos = _empty((B, dims.label_count), torch.float32, dev)
        inv = _empty((B + dims.label_count,), torch.float32, dev)
        cv = _f32c(cv, "code_vector")
        rc = lib.c2v_angular_forward_train(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), _ptr(label), B, float(margin),
                                           float(inverse_temp), _ptr(out), _ptr(cos), _ptr(inv), _stream(dev))
        _lib.check(rc, "c2v_angular_forward_train")
    return out, cos, inv


def angular_backward(dims, params, cv, label, margin, inverse_temp, cos, inv, d_out, need_cv=True, need_w=True):
    """-> (d_code_vector, d_output_weight); d_out is consumed (overwritten)"""
    lib = _lib.load()
    B = cv.shape[0]
    dev = cv.device
    with torch.cuda.device(dev):
        d_out = _f32c(d_out, "d_outputs").clone()            # the kernel overwrites it; autograd's grad tensor is not ours
        d_cv = torch.empty_like(cv) if need_cv else None
        d_w = _empty((dims.label_count, dims.encode), torch.float32, dev) if need_w else None
        scratch = _empty((B + dims.label_count,), torch.float32, dev)
        cv = _f32c(cv, "code_vector")
        rc = lib.c2v_angular_backward(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), _ptr(label), B, float(margin),
                                      float(inverse_temp), _ptr(cos), _ptr(inv), _ptr(d_out), _ptr(d_cv), _ptr(d_w),
                                      _ptr(scratch), _stream(dev))
        _lib.check(rc, "c2v_angular_backward")
    return d_cv, d_w


def loss_argmax(outputs, label=None, want_grad=False):
    """main.py:251-264 + main.py:285 -> (loss 0-d or None, argmax [B], maxval [B], d_outputs or None)"""
    lib = _lib.load()
    _need_cuda(outputs)
    B, C = outputs.shape
    dev = outputs.device
    outputs = outputs.contiguous()
    with torch.cuda.device(dev):
        am = _empty((B,), torch.int64, dev)
        mx = _empty((B,), torch.float32, dev)
        loss = _empty((), torch.float32, dev) if label is not None else None
        dout = torch.empty_like(outputs) if (want_grad and label is not None) else None
        if label is not None:
            label = _idx(label, "label", (B,))
        rc = lib.c2v_loss_argmax(_ptr(outputs), _ptr(label), B, C, _ptr(loss), _ptr(am), _ptr(mx), _ptr(dout),
                                 _stream(dev))
        _lib.check(rc, "c2v_loss_argmax")
    return loss, am, mx, dout


def label_backward(dims, params, cv, d_out, need_cv=True, need_w=True, need_b=True, algo=_lib.ALGO_AUTO, cache=None,
                   weight=None, absmax_ready=False):
    """backward of model.py:83 -> (d_code_vector, d_output_weight, d_output_bias).  With the label PrepCache of the
    forward (cache + weight) the two contractions run on the tensor cores and stream the cached W_out image.
    absmax_ready: d_out is the tensor label_dlogits just returned for the same cache (skips the max |d_out| pass)."""
    lib = _lib.load()
    B = cv.shape[0]
    dev = cv.device
    with torch.cuda.device(dev):
        d_cv = torch.empty_like(cv) if need_cv else None
        d_w = _empty((dims.label_count, dims.encode), torch.float32, dev) if (need_w or need_b) else None
        d_b = _empty((dims.label_count,), torch.float32, dev) if need_b else None
        cv = _f32c(cv, "code_vector"); d_out = _f32c(d_out, "d_outputs")
        ws, flags = _label_ws(dims, B, dev, algo, cache, weight, absmax_ready=absmax_ready, fresh=False)
        if ws is not None:
            rc = lib.c2v_label_backward_ws(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), _ptr(d_out), B, _ptr(d_cv),
                                           _ptr(d_w), _ptr(d_b), _ptr(ws), ws.numel(), flags, _stream(dev))
            _lib.check(rc, "c2v_label_backward_ws")
        else:
            rc = lib.c2v_label_backward(ctypes.byref(dims), ctypes.byref(params), _ptr(cv),
                                        _ptr(d_out), B, _ptr(d_cv), _ptr(d_w), _ptr(d_b), _stream(dev))
            _lib.check(rc, "c2v_label_backward")
    return d_cv, (d_w if need_w else None), d_b


def _row_slots(slots):
    """(terminal slot map or None, path slot map or None) -> c2v_row_slots (the tensors stay with the caller)"""
    return RowSlots(_ptr(slots[0]), _ptr(slots[1]))


def encode_backward(dims, params, starts, paths, ends, cv, att, d_cv, d_att, shapes, drop_p=0.0, training=False,
                    seed=0, grads_out=None, x_stash=None, between_phases=None, slots=None):
    """Gradients of the six encode parameters; returns dict name -> tensor.  x_stash: what encode_forward(stash=True)
    returned for this batch (skips the re-gather + recompute GEMM).  slots: (terminal, path) slot maps of sparse_rows()
    for this batch, None for a dense table; grads_out then holds the zero-filled compact [U, E] buffer of every table
    with a slot map (c2v_encode_backward_sparse)."""
    lib = _lib.load()
    B, L = starts.shape
    dev = starts.device
    with torch.cuda.device(dev):
        g = grads_out or {k: torch.zeros(s, dtype=torch.float32, device=dev) for k, s in shapes.items()}
        grads = Grads(_ptr(g["terminal_embedding"]), _ptr(g["path_embedding"]), _ptr(g["input_linear"]),
                      _ptr(g["ln_weight"]), _ptr(g["ln_bias"]), _ptr(g["attention"]))
        nbytes = lib.c2v_encode_backward_workspace_bytes(ctypes.byref(dims), B, L)
        ws = _empty((nbytes,), torch.uint8, dev)
        drop = Dropout(float(drop_p), 1 if training else 0, int(seed))
        # contiguous copies (if any were needed) are bound to locals so that they outlive the launch
        cv = _f32c(cv, "code_vector"); att = _f32c(att, "attention")
        d_cv = _f32c(d_cv, "d_code_vector")
        d_att = _f32c(d_att, "d_attention") if d_att is not None else None
        # between_phases: called after the path sub-vector's gradients are complete (c2v_encode_backward_phased), e.g. to
        # start their data-parallel reduction on another stream while start / end / dW are still being computed
        for phase in ((1, 2) if between_phases is not None else (0,)):
            args = (ctypes.byref(dims), ctypes.byref(params), _ptr(starts), _ptr(paths), _ptr(ends), B, L, ctypes.byref(drop),
                    _ptr(cv), _ptr(att), _ptr(x_stash), _ptr(d_cv), _ptr(d_att), ctypes.byref(grads))
            if slots is None:
                rc = lib.c2v_encode_backward_phased(*args, _ptr(ws), nbytes, phase, _stream(dev))
            else:
                rc = lib.c2v_encode_backward_sparse(*args, ctypes.byref(_row_slots(slots)), _ptr(ws), nbytes, phase,
                                                    _stream(dev))
            _lib.check(rc, "c2v_encode_backward")
            if phase == 1:
                between_phases()
    return g


def encode_backward_packed(dims, params, bags, cv, att, d_cv, d_att, shapes, drop_p=0.0, training=False, seed=0,
                           grads_out=None, x_stash=None, between_phases=None, slots=None):
    """encode_backward for a PackedBags batch: att / d_att [N], x_stash [N, H] from encode_forward_packed(stash=True)."""
    lib = _lib.load()
    B, N, L = bags.B, bags.N, bags.L
    dev = bags.device
    with torch.cuda.device(dev):
        g = grads_out or {k: torch.zeros(s, dtype=torch.float32, device=dev) for k, s in shapes.items()}
        grads = Grads(_ptr(g["terminal_embedding"]), _ptr(g["path_embedding"]), _ptr(g["input_linear"]),
                      _ptr(g["ln_weight"]), _ptr(g["ln_bias"]), _ptr(g["attention"]))
        nbytes = lib.c2v_encode_backward_packed_workspace_bytes(ctypes.byref(dims), B, N)
        ws = _empty((nbytes,), torch.uint8, dev)
        drop = Dropout(float(drop_p), 1 if training else 0, int(seed))
        cv = _f32c(cv, "code_vector"); att = _f32c(att, "attention")
        d_cv = _f32c(d_cv, "d_code_vector")
        d_att = _f32c(d_att, "d_attention") if d_att is not None else None
        for phase in ((1, 2) if between_phases is not None else (0,)):
            args = (ctypes.byref(dims), ctypes.byref(params), _ptr(bags.starts), _ptr(bags.paths), _ptr(bags.ends),
                    _ptr(bags.offsets), B, N, L, ctypes.byref(drop), _ptr(cv), _ptr(att), _ptr(x_stash), _ptr(d_cv),
                    _ptr(d_att), ctypes.byref(grads))
            if slots is None:
                rc = lib.c2v_encode_backward_packed(*args, _ptr(ws), nbytes, phase, _stream(dev))
            else:
                rc = lib.c2v_encode_backward_packed_sparse(*args, ctypes.byref(_row_slots(slots)), _ptr(ws), nbytes, phase,
                                                           _stream(dev))
            _lib.check(rc, "c2v_encode_backward_packed")
            if phase == 1:
                between_phases()
    return g


def sparse_rows(indices, vocab):
    """Row map of one embedding table for one batch (c2v_sparse_rows): indices is a list of one or two int64 CUDA tensors
    (any shape; e.g. [starts, ends] for the terminal table) -> (slot int32 [vocab], rows int64 [min(vocab, n)] whose
    first U entries are the distinct rows the batch indexes, ascending, count int64 [1] = U), all on the device and
    enqueued on the current stream.  Out-of-range indices count as row 0, as the encode reads them."""
    lib = _lib.load()
    idx = [_idx(t, "indices").reshape(-1) for t in indices]
    if not 1 <= len(idx) <= 2:
        raise ValueError("sparse_rows takes one or two index tensors")
    _need_cuda(*idx)
    a = idx[0]
    b = idx[1] if len(idx) == 2 else None
    n_a, n_b = a.numel(), (b.numel() if b is not None else 0)
    vocab = int(vocab)
    dev = a.device
    nbytes = lib.c2v_sparse_rows_workspace_bytes(vocab)
    if nbytes == 0:
        raise ValueError(f"sparse_rows: vocab = {vocab} outside [1, 2^31)")
    with torch.cuda.device(dev):
        slot = _empty((vocab,), torch.int32, dev)
        rows = _empty((min(vocab, n_a + n_b),), torch.int64, dev)
        count = _empty((1,), torch.int64, dev)
        ws = _empty((nbytes,), torch.uint8, dev)
        rc = lib.c2v_sparse_rows(_ptr(a) if n_a else None, n_a, _ptr(b) if n_b else None, n_b, vocab, _ptr(slot),
                                 _ptr(rows) if rows.numel() else None, _ptr(count), _ptr(ws), nbytes, _stream(dev))
        _lib.check(rc, "c2v_sparse_rows")
    return slot, rows, count


def sparse_adam_step(param, exp_avg, exp_avg_sq, values, rows, lr, beta1, beta2, eps, step):
    """torch.optim.SparseAdam's update of param / exp_avg / exp_avg_sq [n, E] (contiguous fp32 CUDA) at the distinct rows
    `rows` (int64 [U]) from the gradient values [U, E] of a coalesced sparse gradient (c2v_sparse_adam_step); step is
    the step count after this step."""
    lib = _lib.load()
    _need_cuda(param, exp_avg, exp_avg_sq, values, rows)
    for t, name in ((param, "param"), (exp_avg, "exp_avg"), (exp_avg_sq, "exp_avg_sq")):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.shape != param.shape:
            raise TypeError(f"{name} must be contiguous fp32 of the parameter's shape")
    n, E = param.shape[0], param[0].numel()
    values = _f32c(values, "values").reshape(-1, E)
    rows = _idx(rows, "rows").reshape(-1)
    if values.shape[0] != rows.numel():
        raise ValueError(f"sparse_adam_step: {values.shape[0]} value rows for {rows.numel()} indices")
    dev = param.device
    with torch.cuda.device(dev):
        rc = lib.c2v_sparse_adam_step(_ptr(param), _ptr(exp_avg), _ptr(exp_avg_sq), _ptr(values), _ptr(rows), rows.numel(),
                                      n, E, float(lr), float(beta1), float(beta2), float(eps), int(step), _stream(dev))
        _lib.check(rc, "c2v_sparse_adam_step")

"""torch-facing wrappers over the C ABI: device memory, streams and autograd plumbing only.
All arithmetic happens inside libc2v_b200.so."""
import ctypes
import os
import threading

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


_det = threading.local()


def sync_deterministic():
    """Set the library's deterministic mode (c2v_set_deterministic) of the calling thread from
    torch.are_deterministic_algorithms_enabled(); the library is called only when the value changed.  The mode is per host
    thread and autograd runs backwards on threads of its own, so every training-path wrapper calls this before it sizes a
    workspace.  Returns the mode."""
    on = torch.are_deterministic_algorithms_enabled()
    if getattr(_det, "on", False) != on:
        _lib.load().c2v_set_deterministic(1 if on else 0)
        _det.on = on
    return on


def torch_matmul_tf32():
    """True while torch lets its fp32 CUDA matmuls use TF32: torch.backends.cuda.matmul.fp32_precision == "tf32", what
    torch.set_float32_matmul_precision("high" / "medium"), allow_tf32 = True and the fp32_precision setters (this one and
    torch.backends.fp32_precision) select.  The legacy getters (allow_tf32, get_float32_matmul_precision()) are not read:
    they raise once a setter of the new API has been used."""
    return torch.backends.cuda.matmul.fp32_precision == "tf32"


def sync_matmul_precision():
    """Set the library's matmul precision (c2v_set_matmul_precision) of the calling thread from torch's switch:
    C2V_MATMUL_TF32 while torch_matmul_tf32(), C2V_MATMUL_IEEE otherwise.  Like sync_deterministic the mode is per host
    thread and the library is called only when the value changed; every wrapper that can reach a tensor-core GEMM calls
    this.  Returns True in TF32 mode."""
    on = torch_matmul_tf32()
    if getattr(_det, "tf32", False) != on:
        _lib.check(_lib.load().c2v_set_matmul_precision(_lib.MATMUL_TF32 if on else _lib.MATMUL_IEEE),
                   "c2v_set_matmul_precision")
        _det.tf32 = on
    return on


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


def capturing():
    """True while the current CUDA stream is being captured into a CUDA graph"""
    return torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()


def capture_flags(algo):
    """`algo` of a library call made under capture: plain stream-ordered launches (no programmatic dependent launch)"""
    return int(algo) | NO_PDL if capturing() else int(algo)


def next_dropout_key(rng_state):
    """A fresh int64 [1] device tensor holding the next dropout key of rng_state (int64 [2] {base, counter} on the
    device): c2v_next_dropout_key, enqueued on the current stream (capturable)."""
    lib = _lib.load()
    dev = rng_state.device
    with torch.cuda.device(dev):
        key = torch.empty(1, dtype=torch.int64, device=dev)
        _lib.check(lib.c2v_next_dropout_key(_ptr(rng_state), _ptr(key), _stream(dev)), "c2v_next_dropout_key")
    return key


def _dropout(drop_p, training, seed):
    """c2v_dropout: `seed` is an int (the key, by value) or an int64 [1] device tensor holding it
    (C2V_DROPOUT_SEED_ON_DEVICE; the caller keeps the tensor alive until the kernels have run)"""
    if isinstance(seed, torch.Tensor):
        return Dropout(float(drop_p), (1 if training else 0) | _lib.DROPOUT_SEED_ON_DEVICE, seed.data_ptr())
    return Dropout(float(drop_p), 1 if training else 0, int(seed))


class PrepCache:
    """A persistent workspace whose derived weight images (split / transposed copies of a weight
    matrix) are rebuilt only when the weight changed: keyed on (data_ptr, _version, size)."""

    def __init__(self, mirror_errors=False):
        self.buf, self.key = None, None
        # CUDA graphs: a replay neither bumps version counters nor knows whether the weights changed since the capture, so
        # a call under capture rebuilds the images (no REUSE_PREP), and once the owner has captured a training step the
        # counters are not trusted at all (trust_versions = False).  A graph keeps the raw address of the workspace it
        # was captured with: graph_bufs keeps every such buffer alive even after a larger one replaces it.
        self.trust_versions, self.graph_bufs = True, []
        # encode workspaces: a pinned host word the finalize kernel adds its out-of-range index count to
        # (c2v_workspace_set_status_mirror), polled by raise_deferred() at the next call on this cache
        self.mirror_errors, self.err = mirror_errors, None       # (pinned memory needs the driver: allocated on first use)

    def get(self, nbytes, device, weight):
        key = (weight.data_ptr(), weight._version, str(device))
        fresh = self.buf is None or self.buf.numel() < nbytes or self.buf.device != device
        cap = capturing()
        if fresh and cap:
            raise RuntimeError("a persistent workspace would be allocated under CUDA-graph capture: run the same call once "
                               "eagerly at this batch shape before capturing it")
        if fresh:
            self.buf = _empty((nbytes,), torch.uint8, device)
            if self.mirror_errors:
                if self.err is None:
                    self.err = torch.zeros(1, dtype=torch.int64).pin_memory()
                lib = _lib.load()
                with torch.cuda.device(device):
                    _lib.check(lib.c2v_workspace_set_status_mirror(_ptr(self.buf), ctypes.c_void_p(self.err.data_ptr()),
                                                                   _stream(device)), "c2v_workspace_set_status_mirror")
        reuse = (not fresh) and key == self.key and self.trust_versions and not cap
        self.key = key
        if cap and not any(b is self.buf for b in self.graph_bufs):
            self.graph_bufs.append(self.buf)
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
    sync_matmul_precision()
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
        drop = _dropout(drop_p, training, seed)
        algo = capture_flags(algo)
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
    if capturing():
        raise RuntimeError("PackedBags batches cannot be captured into a CUDA graph: their context count N changes from "
                           "batch to batch; capture padded [B, L] batches")
    lib = _lib.load()
    sync_matmul_precision()
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
        drop = _dropout(drop_p, training, seed)
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
    sync_deterministic()
    sync_matmul_precision()
    if nbytes is None:
        nbytes = _lib.load().c2v_label_workspace_bytes(ctypes.byref(dims), B)
    algo = capture_flags(algo)
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


class LossCriterion:
    """The criterion of the fused loss, read from an nn.NLLLoss / nn.CrossEntropyLoss (c2v_loss_options):
    F.cross_entropy(logits, label, weight, ignore_index, reduction, label_smoothing) on the head's logits."""

    def __init__(self, criterion, label_count, device):
        if type(criterion) not in (torch.nn.NLLLoss, torch.nn.CrossEntropyLoss):
            raise TypeError("criterion must be exactly torch.nn.NLLLoss (applied, as in the reference, to log_softmax of the "
                            "logits) or torch.nn.CrossEntropyLoss, not a subclass or another loss: got "
                            f"{type(criterion).__name__}")
        w = criterion.weight
        if w is not None and (w.dtype != torch.float32 or w.device != torch.device(device) or
                              tuple(w.shape) != (int(label_count),)):
            raise ValueError(f"criterion weight must be float32 of shape [{int(label_count)}] on {device}, got "
                             f"{w.dtype} {tuple(w.shape)} on {w.device}")
        if criterion.reduction not in _lib.REDUCTIONS:
            raise ValueError(f"{criterion.reduction} is not a valid value for reduction")
        self.weight = w.contiguous() if w is not None else None    # (the same tensor when contiguous: in-place updates show)
        self.ignore_index = int(criterion.ignore_index)
        self.label_smoothing = float(getattr(criterion, "label_smoothing", 0.0))
        self.reduction = criterion.reduction

    def options(self, row_grad=None):
        o = _lib.LossOptions(_ptr(self.weight), self.ignore_index, self.label_smoothing, _lib.REDUCTIONS[self.reduction],
                             _ptr(row_grad))
        o._keep = (self.weight, row_grad)
        return o

    def loss_shape(self, B):
        return (B,) if self.reduction == "none" else ()


def label_loss_opts(dims, params, cv, label, crit, angular=None, algo=_lib.ALGO_AUTO, cache=None, weight=None):
    """label_loss / angular_loss (angular = (margin, inverse_temp)) with a LossCriterion
    -> (loss 0-d or [B], lse [B], argmax [B], maxval [B], coef [2 B + 1], inv_norms [B + C] or None).  coef holds the row
    coefficients the matching dlogits call reads on the device."""
    lib = _lib.load()
    _need_cuda(cv, label)
    B = cv.shape[0]
    dev = cv.device
    label = _idx(label, "label", (B,))
    with torch.cuda.device(dev):
        loss = _empty(crit.loss_shape(B), torch.float32, dev)
        lse = _empty((B,), torch.float32, dev)
        am = _empty((B,), torch.int64, dev)
        mx = _empty((B,), torch.float32, dev)
        coef = _empty((2 * B + 1,), torch.float32, dev)
        inv = _empty((B + dims.label_count,), torch.float32, dev) if angular is not None else None
        sync_deterministic()                     # (the size depends on the mode)
        nbytes = lib.c2v_label_loss_opts_workspace_bytes(ctypes.byref(dims), B)
        ws, algo = _label_ws(dims, B, dev, algo, cache, weight, nbytes=nbytes)
        cv = _f32c(cv, "code_vector")
        opts = crit.options()
        if angular is None:
            rc = lib.c2v_label_loss_argmax_opts(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), _ptr(label), B,
                                                ctypes.byref(opts), None, _ptr(loss), _ptr(lse), _ptr(coef), _ptr(am),
                                                _ptr(mx), _ptr(ws), ws.numel(), int(algo), _stream(dev))
        else:
            rc = lib.c2v_angular_loss_argmax_opts(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), _ptr(label), B,
                                                  float(angular[0]), float(angular[1]), ctypes.byref(opts), None, _ptr(loss),
                                                  _ptr(lse), _ptr(coef), _ptr(am), _ptr(mx), _ptr(inv), _ptr(ws), ws.numel(),
                                                  int(algo), _stream(dev))
        _lib.check(rc, "c2v_label_loss_argmax_opts" if angular is None else "c2v_angular_loss_argmax_opts")
    return loss, lse, am, mx, coef, inv


def label_dlogits_opts(dims, params, cv, label, lse, coef, crit, d_loss, inv_norms=None, angular=None,
                       algo=_lib.ALGO_AUTO, cache=None, weight=None):
    """d loss / d logits [B, C] (angular: d loss / d (cv . W^T)) of label_loss_opts' loss for its upstream gradient d_loss
    (0-d, or [B] for reduction none), recomputed from cv and W_out"""
    lib = _lib.load()
    B = cv.shape[0]
    dev = cv.device
    label = _idx(label, "label", (B,))
    with torch.cuda.device(dev):
        g = _empty((B, dims.label_count), torch.float32, dev)
        ws, algo = _label_ws(dims, B, dev, algo, cache, weight)
        cv = _f32c(cv, "code_vector"); lse = _f32c(lse, "lse"); d_loss = _f32c(d_loss, "d_loss")
        none = crit.reduction == "none"
        opts = crit.options(row_grad=d_loss if none else None)
        sd = None if none else d_loss.reshape(1)
        if angular is None:
            rc = lib.c2v_label_dlogits_opts(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), _ptr(label), _ptr(lse),
                                            _ptr(coef), B, ctypes.byref(opts), 1.0, _ptr(sd), _ptr(g), _ptr(ws), ws.numel(),
                                            int(algo), _stream(dev))
        else:
            inv = _f32c(inv_norms, "inv_norms")
            rc = lib.c2v_angular_dlogits_opts(ctypes.byref(dims), ctypes.byref(params), _ptr(cv), _ptr(label), _ptr(lse),
                                              _ptr(coef), _ptr(inv), B, float(angular[0]), float(angular[1]),
                                              ctypes.byref(opts), 1.0, _ptr(sd), _ptr(g), _ptr(ws), ws.numel(), int(algo),
                                              _stream(dev))
        _lib.check(rc, "c2v_label_dlogits_opts" if angular is None else "c2v_angular_dlogits_opts")
    return g


def loss_argmax_opts(outputs, label, crit, want_grad=False):
    """loss_argmax with a LossCriterion -> (loss 0-d or [B], argmax [B], maxval [B], d_outputs or None); d_outputs is the
    gradient for a unit upstream gradient (of the scalar loss, or of every row loss for reduction none)"""
    lib = _lib.load()
    sync_deterministic()
    _need_cuda(outputs, label)
    B, C = outputs.shape
    dev = outputs.device
    outputs = outputs.contiguous()
    label = _idx(label, "label", (B,))
    with torch.cuda.device(dev):
        am = _empty((B,), torch.int64, dev)
        mx = _empty((B,), torch.float32, dev)
        loss = _empty(crit.loss_shape(B), torch.float32, dev)
        dout = torch.empty_like(outputs) if want_grad else None
        opts = crit.options()
        rc = lib.c2v_loss_argmax_opts(_ptr(outputs), _ptr(label), B, C, ctypes.byref(opts), _ptr(loss), _ptr(am), _ptr(mx),
                                      _ptr(dout), _stream(dev))
        _lib.check(rc, "c2v_loss_argmax_opts")
    return loss, am, mx, dout


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
            sync_deterministic()                 # (the size depends on the mode)
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
    sync_deterministic()
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
    sync_deterministic()
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
    sync_deterministic()
    sync_matmul_precision()
    B, L = starts.shape
    dev = starts.device
    with torch.cuda.device(dev):
        g = grads_out or {k: torch.zeros(s, dtype=torch.float32, device=dev) for k, s in shapes.items()}
        grads = Grads(_ptr(g["terminal_embedding"]), _ptr(g["path_embedding"]), _ptr(g["input_linear"]),
                      _ptr(g["ln_weight"]), _ptr(g["ln_bias"]), _ptr(g["attention"]))
        nbytes = lib.c2v_encode_backward_workspace_bytes(ctypes.byref(dims), B, L)
        ws = _empty((nbytes,), torch.uint8, dev)
        drop = _dropout(drop_p, training, seed)
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
    sync_deterministic()
    sync_matmul_precision()
    B, N, L = bags.B, bags.N, bags.L
    dev = bags.device
    with torch.cuda.device(dev):
        g = grads_out or {k: torch.zeros(s, dtype=torch.float32, device=dev) for k, s in shapes.items()}
        grads = Grads(_ptr(g["terminal_embedding"]), _ptr(g["path_embedding"]), _ptr(g["input_linear"]),
                      _ptr(g["ln_weight"]), _ptr(g["ln_bias"]), _ptr(g["attention"]))
        nbytes = lib.c2v_encode_backward_packed_workspace_bytes(ctypes.byref(dims), B, N)
        ws = _empty((nbytes,), torch.uint8, dev)
        drop = _dropout(drop_p, training, seed)
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


def _gathered_lists(rows, counts):
    rows = _idx(rows, "rows")
    counts = _idx(counts, "counts")
    if rows.dim() != 2 or tuple(counts.shape) != (rows.shape[0],):
        raise ValueError(f"rows must be [world, u_max] and counts [world], got {tuple(rows.shape)} and "
                         f"{tuple(counts.shape)}")
    return rows, counts


def sparse_union_rows(rows, counts, vocab):
    """The union of W ascending row lists (c2v_sparse_union_rows): rows int64 [W, u_max], list r valid up to counts[r]
    (int64 [W], on the device; negative = empty), as the ranks of a data-parallel step all-gathered them ->
    (union_rows int64 [min(vocab, W * u_max)] whose first U entries are the union, ascending, count int64 [1] = U), on
    the device and enqueued on the current stream; U is not read on the host."""
    lib = _lib.load()
    rows, counts = _gathered_lists(rows, counts)
    _need_cuda(rows, counts)
    world, u_max, vocab = rows.shape[0], rows.shape[1], int(vocab)
    nbytes = lib.c2v_sparse_union_rows_workspace_bytes(vocab)
    if nbytes == 0:
        raise ValueError(f"sparse_union_rows: vocab = {vocab} outside [1, 2^31)")
    dev = rows.device
    with torch.cuda.device(dev):
        union = _empty((min(vocab, world * u_max),), torch.int64, dev)
        count = _empty((1,), torch.int64, dev)
        ws = _empty((nbytes,), torch.uint8, dev)
        rc = lib.c2v_sparse_union_rows(_ptr(rows) if u_max else None, _ptr(counts), world, u_max, vocab,
                                       _ptr(union) if union.numel() else None, _ptr(count), _ptr(ws), nbytes, _stream(dev))
        _lib.check(rc, "c2v_sparse_union_rows")
    return union, count


def sparse_adam_step_merged(param, exp_avg, exp_avg_sq, values, rows, counts, union_rows, union_count, lr, beta1,
                            beta2, eps, step, scale):
    """sparse_adam_step on the merged gradient of W ranks (c2v_sparse_adam_step_merged): values fp32 [W, u_max, E] and
    rows / counts as in sparse_union_rows, union_rows / union_count what it returned for them.  Each union row's gradient
    is the sum of the ranks' rows, in fp32 in rank order, times `scale` (the fp32 1/W of the mean, negated for
    maximize); it is applied without being written.  No host read."""
    lib = _lib.load()
    _need_cuda(param, exp_avg, exp_avg_sq, values, rows, counts, union_rows, union_count)
    for t, name in ((param, "param"), (exp_avg, "exp_avg"), (exp_avg_sq, "exp_avg_sq")):
        if t.dtype != torch.float32 or not t.is_contiguous() or t.shape != param.shape:
            raise TypeError(f"{name} must be contiguous fp32 of the parameter's shape")
    rows, counts = _gathered_lists(rows, counts)
    n, E = param.shape[0], param[0].numel()
    world, u_max = rows.shape
    values = _f32c(values, "values")
    if values.numel() != world * u_max * E:
        raise ValueError(f"sparse_adam_step_merged: values has {values.numel()} elements, rows {tuple(rows.shape)} with "
                         f"E = {E} need {world * u_max * E}")
    union_rows, union_count = _idx(union_rows, "union_rows"), _idx(union_count, "union_count")
    dev = param.device
    with torch.cuda.device(dev):
        rc = lib.c2v_sparse_adam_step_merged(
            _ptr(param), _ptr(exp_avg), _ptr(exp_avg_sq), _ptr(values) if u_max else None, _ptr(rows) if u_max else None,
            _ptr(counts), world, u_max, _ptr(union_rows) if union_rows.numel() else None, _ptr(union_count), n, E,
            float(scale), float(lr), float(beta1), float(beta2), float(eps), int(step), _stream(dev))
        _lib.check(rc, "c2v_sparse_adam_step_merged")


class SampledSoftmax:
    """The proposal distribution of a sampled-softmax loss (Code2Vec.forward_sampled_loss) over `label_count` labels:
    q(c) = counts[c]^power / sum_k counts[k]^power, uniform when counts is None.  Every step draws num_sampled candidates
    i.i.d. with replacement from q.  The usual counts are the training set's label frequencies
    (Vocab.get_freq_list()); pass counts + 1 when some label never occurs, since the true label's correction log q needs
    q > 0.

    The fp64 CDF (numpy.cumsum of the weights over their total) and log q [label_count] are built once on the host and
    uploaded to each device on its first use.  ValueError: label_count < 1, num_sampled outside [1, 65536], counts not
    1-D of length label_count or with a non-finite or non-positive entry, power not finite and > 0."""

    def __init__(self, label_count, num_sampled, counts=None, power=1.0):
        import math
        import numpy as np
        C, S, power = int(label_count), int(num_sampled), float(power)
        if C < 1:
            raise ValueError(f"SampledSoftmax: label_count = {C} < 1")
        if not 1 <= S <= _lib.SAMPLED_MAX:
            raise ValueError(f"SampledSoftmax: num_sampled = {S} outside [1, {_lib.SAMPLED_MAX}]")
        if not (math.isfinite(power) and power > 0):
            raise ValueError(f"SampledSoftmax: power = {power} must be finite and > 0")
        if counts is None:
            w = np.ones(C, dtype=np.float64)
        else:
            if isinstance(counts, torch.Tensor):
                counts = counts.detach().cpu().numpy()
            n = np.asarray(counts, dtype=np.float64)
            if n.ndim != 1 or n.shape[0] != C:
                raise ValueError(f"SampledSoftmax: counts must be 1-D of length label_count = {C}, got shape {n.shape}")
            if not (np.isfinite(n).all() and (n > 0).all()):
                raise ValueError("SampledSoftmax: every count must be finite and > 0 (pass counts + 1 when some label "
                                 "never occurs)")
            with np.errstate(over="ignore", under="ignore"):
                w = n ** power
            if not (np.isfinite(w).all() and (w > 0).all()):
                raise ValueError(f"SampledSoftmax: counts ** {power} leaves the finite positive fp64 range")
        cdf = np.cumsum(w)
        total = cdf[-1]
        if not math.isfinite(total):
            raise ValueError("SampledSoftmax: the sum of counts ** power is not finite in fp64")
        self.label_count, self.num_sampled, self.power = C, S, power
        self.cdf_host = cdf / total                  # cdf_host[-1] == 1 exactly
        self.log_q_host = np.log(w) - np.log(total)
        self._dev = {}

    def device_tables(self, device):
        """-> (cdf fp64 [C], log_q fp64 [C]) on `device`, uploaded on its first use there"""
        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        t = self._dev.get(device)
        if t is None:
            if capturing():
                raise RuntimeError("SampledSoftmax: the proposal tables would be uploaded under CUDA-graph capture: run "
                                   "one step eagerly on this device first")
            t = (torch.from_numpy(self.cdf_host).to(device), torch.from_numpy(self.log_q_host).to(device))
            self._dev[device] = t
        return t

    def sample(self, key, device=None):
        """-> int64 [num_sampled] candidate ids drawn from q with Philox key `key` (c2v_sampled_candidates): an int, or an
        int64 [1] CUDA tensor holding it (read on the device when the kernel runs).  device: where to draw (the key
        tensor's device, else the current CUDA device)."""
        lib = _lib.load()
        key_dev = key if isinstance(key, torch.Tensor) else None
        if key_dev is not None:
            _need_cuda(key_dev)
            if key_dev.dtype != torch.int64 or key_dev.numel() != 1:
                raise TypeError("SampledSoftmax.sample: a key tensor must be int64 with one element")
            device = key_dev.device
        elif device is None:
            device = torch.device("cuda", torch.cuda.current_device())
        cdf, _ = self.device_tables(device)
        with torch.cuda.device(cdf.device):
            out = _empty((self.num_sampled,), torch.int64, cdf.device)
            k = 0 if key_dev is not None else int(key) & 0xFFFFFFFFFFFFFFFF
            rc = lib.c2v_sampled_candidates(_ptr(cdf), self.label_count, self.num_sampled, k, _ptr(key_dev), _ptr(out),
                                            _stream(cdf.device))
            _lib.check(rc, "c2v_sampled_candidates")
        return out


def sampled_gather(w_out, b_out, log_q, candidates, label):
    """-> (ids int64 [S + B], w_hat [S + B, H], b_hat [S + B]) of the compact head (c2v_sampled_gather)"""
    lib = _lib.load()
    _need_cuda(w_out, b_out, log_q, candidates, label)
    C, H = w_out.shape
    S, B = candidates.numel(), label.numel()
    dev = w_out.device
    w_out, b_out = _f32c(w_out, "output_weight"), _f32c(b_out, "output_bias")
    candidates, label = _idx(candidates, "candidates"), _idx(label, "label")
    with torch.cuda.device(dev):
        ids = _empty((S + B,), torch.int64, dev)
        w_hat = _empty((S + B, H), torch.float32, dev)
        b_hat = _empty((S + B,), torch.float32, dev)
        rc = lib.c2v_sampled_gather(_ptr(w_out), _ptr(b_out), _ptr(log_q), C, H, _ptr(candidates), S, _ptr(label), B,
                                    _ptr(w_hat), _ptr(b_hat), _ptr(ids), _stream(dev))
        _lib.check(rc, "c2v_sampled_gather")
    return ids, w_hat, b_hat


def sampled_loss(logits, ids, S):
    """-> (loss 0-d, lse [B]) of the compact logits [B, S + B] (c2v_sampled_loss)"""
    lib = _lib.load()
    B = logits.shape[0]
    dev = logits.device
    with torch.cuda.device(dev):
        lse = _empty((B,), torch.float32, dev)
        loss = _empty((), torch.float32, dev)
        rc = lib.c2v_sampled_loss(_ptr(logits), _ptr(ids), int(S), B, _ptr(lse), _ptr(loss), _stream(dev))
        _lib.check(rc, "c2v_sampled_loss")
    return loss, lse


def sampled_dlogits_(logits, ids, lse, S, scale, scale_device=None):
    """overwrites the compact logits [B, S + B] with d loss / d logits (c2v_sampled_dlogits); returns them"""
    lib = _lib.load()
    B = logits.shape[0]
    dev = logits.device
    sd = _f32c(scale_device, "scale_device") if scale_device is not None else None
    with torch.cuda.device(dev):
        rc = lib.c2v_sampled_dlogits(_ptr(logits), _ptr(ids), _ptr(lse), int(S), B, float(scale), _ptr(sd), _stream(dev))
        _lib.check(rc, "c2v_sampled_dlogits")
    return logits


def scatter_rows_add(ids, rows, bias, dst, dst_bias):
    """dst[ids[e]] += rows[e] and dst_bias[ids[e]] += bias[e] in a fixed order (c2v_scatter_rows_add); either pair may
    be None"""
    lib = _lib.load()
    n = ids.numel()
    ref = dst if dst is not None else dst_bias
    C = ref.shape[0]
    H = dst.shape[1] if dst is not None else 1
    dev = ref.device
    rows = _f32c(rows, "rows") if rows is not None else None
    bias = _f32c(bias, "bias") if bias is not None else None
    nbytes = lib.c2v_scatter_rows_add_workspace_bytes(n)
    if nbytes == 0:
        raise ValueError(f"scatter_rows_add: {n} ids outside [1, 2^31)")
    with torch.cuda.device(dev):
        ws = _empty((nbytes,), torch.uint8, dev)
        rc = lib.c2v_scatter_rows_add(_ptr(ids), n, _ptr(rows), _ptr(bias), H, C, _ptr(dst), _ptr(dst_bias), _ptr(ws),
                                      nbytes, _stream(dev))
        _lib.check(rc, "c2v_scatter_rows_add")

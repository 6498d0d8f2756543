"""ctypes binding of oracle/c2v_oracle.c plus a torch-CPU restatement used as the
timed CPU baseline.  TEST INFRASTRUCTURE ONLY (see c2v_oracle.c header).

Every function cites the reference lines it follows (model.py = /root/reference/model/model.py).
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libc2v_oracle.so")
_lib = None

_i64p = ctypes.POINTER(ctypes.c_int64)
_f32p = ctypes.POINTER(ctypes.c_float)


def build(force=False):
    """gcc-compile the C oracle in-tree (oracle/_build/, git-ignored)."""
    src = os.path.join(_HERE, "c2v_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-s", "-C", _HERE, "-B" if force else "-s"])
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_SO)
    return _lib


def _f(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a, a.ctypes.data_as(_f32p)


def _i(a):
    a = np.ascontiguousarray(a, dtype=np.int64)
    return a, a.ctypes.data_as(_i64p)


def encode_forward(starts, paths, ends, emb_t, emb_p, W, ln_g, ln_b, attn, dropmask=None,
                   ln_eps=1e-5, want_ctx=False):
    """model.py:44-69 + 90-96.  Returns (code_vector [B,H], attention [B,L][, ctx_h])."""
    starts, ps = _i(starts); paths, pp = _i(paths); ends, pe = _i(ends)
    B, L = starts.shape
    emb_t, pt = _f(emb_t); emb_p, ppp = _f(emb_p); W, pw = _f(W)
    ln_g, pg = _f(ln_g); ln_b, pb = _f(ln_b); attn, pa = _f(attn)
    H = W.shape[0]
    assert W.shape[1] == 2 * emb_t.shape[1] + emb_p.shape[1]
    cv = np.empty((B, H), np.float32); at = np.empty((B, L), np.float32)
    ctx = np.empty((B, L, H), np.float32) if want_ctx else None
    dm = pdm = None
    if dropmask is not None:
        dm, pdm = _f(dropmask)
    rc = lib().c2v_oracle_encode_forward(
        ps, pp, pe, ctypes.c_int(B), ctypes.c_int(L),
        pt, ctypes.c_int64(emb_t.shape[0]), ctypes.c_int(emb_t.shape[1]),
        ppp, ctypes.c_int64(emb_p.shape[0]), ctypes.c_int(emb_p.shape[1]),
        pw, ctypes.c_int(H), pg, pb, ctypes.c_float(ln_eps), pa, pdm,
        cv.ctypes.data_as(_f32p), at.ctypes.data_as(_f32p),
        ctx.ctypes.data_as(_f32p) if want_ctx else None)
    if rc == -1:
        raise IndexError("index out of range in self")   # what nn.Embedding raises
    if rc != 0:
        raise MemoryError("oracle allocation failed")
    return (cv, at, ctx) if want_ctx else (cv, at)


def label_logits(cv, Wout, bias):
    """model.py:83."""
    cv, pc = _f(cv); Wout, pw = _f(Wout)
    B, H = cv.shape; C = Wout.shape[0]
    pbias = None
    if bias is not None:
        bias, pbias = _f(bias)
    out = np.empty((B, C), np.float32)
    lib().c2v_oracle_label_logits(pc, ctypes.c_int(B), ctypes.c_int(H), pw, pbias,
                                  ctypes.c_int64(C), out.ctypes.data_as(_f32p))
    return out


def angular_logits(cv, Wout, label, margin, inverse_temp):
    """model.py:71-80."""
    cv, pc = _f(cv); Wout, pw = _f(Wout); label, pl = _i(label)
    B, H = cv.shape; C = Wout.shape[0]
    out = np.empty((B, C), np.float32)
    lib().c2v_oracle_angular_logits(pc, ctypes.c_int(B), ctypes.c_int(H), pw, ctypes.c_int64(C), pl,
                                    ctypes.c_float(margin), ctypes.c_float(inverse_temp),
                                    out.ctypes.data_as(_f32p))
    return out


def loss_argmax(logits, label):
    """main.py:251-264 (mean NLL of log_softmax; weights are all 1) and main.py:285."""
    logits, pl = _f(logits)
    B, C = logits.shape
    lab = plab = None
    if label is not None:
        lab, plab = _i(label)
    loss = ctypes.c_float(0.0)
    am = np.empty((B,), np.int64); mx = np.empty((B,), np.float32)
    lib().c2v_oracle_loss_argmax(pl, ctypes.c_int(B), ctypes.c_int64(C), plab, ctypes.byref(loss),
                                 am.ctypes.data_as(_i64p), mx.ctypes.data_as(_f32p))
    return float(loss.value), am, mx


def forward(params, starts, paths, ends, label=None, dropmask=None, angular=None):
    """Whole Code2Vec.forward (model.py:44-88) -> (outputs, code_vector, attention).
    params: dict with the reference state_dict keys (numpy arrays)."""
    cv, at = encode_forward(starts, paths, ends, params["terminal_embedding.weight"],
                            params["path_embedding.weight"], params["input_linear.weight"],
                            params["input_layer_norm.weight"], params["input_layer_norm.bias"],
                            params["attention_parameter"], dropmask)
    if angular is not None:
        out = angular_logits(cv, params["output_linear"], label, angular["margin"], angular["inverse_temp"])
    else:
        out = label_logits(cv, params["output_linear.weight"], params["output_linear.bias"])
    return out, cv, at


def backward(params, starts, paths, ends, g_logits, dropmask=None, ln_eps=1e-5):
    """Gradients of every parameter given dLoss/doutputs; plain head."""
    starts, ps = _i(starts); paths, pp = _i(paths); ends, pe = _i(ends)
    B, L = starts.shape
    emb_t, pt = _f(params["terminal_embedding.weight"]); emb_p, ppp = _f(params["path_embedding.weight"])
    W, pw = _f(params["input_linear.weight"]); g, pg = _f(params["input_layer_norm.weight"])
    b, pb = _f(params["input_layer_norm.bias"]); a, pa = _f(params["attention_parameter"])
    Wo, pwo = _f(params["output_linear.weight"]); gl, pgl = _f(g_logits)
    H = W.shape[0]; C = Wo.shape[0]
    dm = pdm = None
    if dropmask is not None:
        dm, pdm = _f(dropmask)
    outs = {
        "terminal_embedding.weight": np.empty_like(emb_t), "path_embedding.weight": np.empty_like(emb_p),
        "input_linear.weight": np.empty_like(W), "input_layer_norm.weight": np.empty_like(g),
        "input_layer_norm.bias": np.empty_like(b), "attention_parameter": np.empty_like(a),
        "output_linear.weight": np.empty_like(Wo), "output_linear.bias": np.empty((C,), np.float32),
    }
    ptr = lambda k: outs[k].ctypes.data_as(_f32p)
    rc = lib().c2v_oracle_backward(
        ps, pp, pe, ctypes.c_int(B), ctypes.c_int(L),
        pt, ctypes.c_int64(emb_t.shape[0]), ctypes.c_int(emb_t.shape[1]),
        ppp, ctypes.c_int64(emb_p.shape[0]), ctypes.c_int(emb_p.shape[1]),
        pw, ctypes.c_int(H), pg, pb, ctypes.c_float(ln_eps), pa, pdm, pwo, ctypes.c_int64(C), pgl,
        ptr("terminal_embedding.weight"), ptr("path_embedding.weight"), ptr("input_linear.weight"),
        ptr("input_layer_norm.weight"), ptr("input_layer_norm.bias"), ptr("attention_parameter"),
        ptr("output_linear.weight"), ptr("output_linear.bias"))
    if rc != 0:
        raise MemoryError("oracle allocation failed")
    return outs


def num_threads():
    return int(lib().c2v_oracle_num_threads())


# --------------------------------------------------------------------------------------
# torch-CPU restatement: the same ATen CPU kernels the reference's eager forward
# dispatches, written functionally.  This is what
# bench.py times as the CPU baseline (kind="port"): the C file above is the
# arithmetic checker, this is the fastest faithful CPU path (MKL sgemm, oneDNN LN).
# --------------------------------------------------------------------------------------
def torch_forward(p, starts, paths, ends, label=None, angular=None, drop_p=0.0, training=False, dropmask=None,
                  taps=None):
    """-> (outputs, code_vector, attention) in the dtype and on the device of `p`.
    dropmask: a given multiplicative mask [B, L, encode] applied to the tanh output instead of a random F.dropout (what
    `forward(..., dropmask=)` does), e.g. the kernels' Philox mask rebuilt by tests/philox_ref.py.
    taps: a dict that receives the intermediates "x" (input_linear output, before the LayerNorm), "ln" (LayerNorm
    output), "z" (masked attention scores), "cv", "logits" and, angular head only, "cos", so that a caller can
    retain_grad() them and read the gradient at every stage."""
    import math
    import torch
    import torch.nn.functional as F
    es = F.embedding(starts, p["terminal_embedding.weight"])            # model.py:48
    ep = F.embedding(paths, p["path_embedding.weight"])                 # model.py:49
    ee = F.embedding(ends, p["terminal_embedding.weight"])              # model.py:50
    c = torch.cat((es, ep, ee), dim=2)                                  # model.py:51
    x = F.linear(c, p["input_linear.weight"])                           # model.py:54
    if taps is not None:
        taps["x"] = x
    H = x.shape[-1]
    x = F.layer_norm(x.view(-1, H), (H,), p["input_layer_norm.weight"],
                     p["input_layer_norm.bias"], 1e-5).view(x.shape)    # model.py:55-56
    if taps is not None:
        taps["ln"] = x
    h = torch.tanh(x)                                                   # model.py:57
    if dropmask is not None:
        h = h * dropmask                                                # model.py:60-61 with a given mask
    elif training and 0.0 < drop_p < 1.0:
        h = F.dropout(h, drop_p, True)                                  # model.py:60-61
    mask = (starts > 0).float()                                         # model.py:64
    z = (h * p["attention_parameter"]).sum(2) * mask + (1 - mask) * (-3.4e38)   # model.py:92-93
    att = F.softmax(z, dim=1)                                           # model.py:96
    cv = (h * att.unsqueeze(-1)).sum(1)                                 # model.py:68-69
    if angular is not None:                                             # model.py:71-80
        cos = F.linear(F.normalize(cv), F.normalize(p["output_linear"]))
        sin = torch.sqrt(1.0 - cos * cos)
        phi = cos * math.cos(angular["margin"]) - sin * math.sin(angular["margin"])
        phi = torch.where(cos > 0, phi, cos)
        oh = torch.zeros_like(cos).scatter_(1, label.view(-1, 1), 1)
        out = (oh * phi + (1.0 - oh) * cos) * angular["inverse_temp"]
    else:
        out = F.linear(cv, p["output_linear.weight"], p["output_linear.bias"])  # model.py:83
    if taps is not None:
        taps.update(z=z, cv=cv, logits=out)
        if angular is not None:
            taps["cos"] = cos
    return out, cv, att

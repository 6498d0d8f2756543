"""CPU-side checks of the plain label head's entry points (c2v_label_logits, _logits_argmax, _loss_argmax, _dlogits,
c2v_label_backward, _backward_ws): bad arguments are rejected with C2V_EINVAL, shapes the tensor-core GEMM does not take
with C2V_EUNSUPPORTED and a missing workspace with C2V_EWORKSPACE, each with a message and before any CUDA call."""
import ctypes

import pytest

from code2vec_b200 import _lib

V = ctypes.c_void_p
FAKE = V(0x1000)          # never dereferenced: every call below fails its argument checks first
BIG = 1 << 40             # a workspace size that passes the size check

# argument order of every entry point (include/c2v_b200.h); `out` is each call's [B, C] output, `d_out` an input gradient
ARGS = {
    "c2v_label_logits": ["d", "p", "cv", "B", "out", "ws", "ws_bytes", "algo", "stream"],
    "c2v_label_logits_argmax": ["d", "p", "cv", "B", "out", "am", "mx", "ws", "ws_bytes", "algo", "stream"],
    "c2v_label_loss_argmax": ["d", "p", "cv", "label", "B", "out", "loss", "lse", "am", "mx", "ws", "ws_bytes", "algo",
                              "stream"],
    "c2v_label_dlogits": ["d", "p", "cv", "label", "lse", "B", "scale", "scale_device", "out", "ws", "ws_bytes", "algo",
                          "stream"],
    "c2v_label_backward": ["d", "p", "cv", "d_out", "B", "d_cv", "d_w", "d_b", "stream"],
    "c2v_label_backward_ws": ["d", "p", "cv", "d_out", "B", "d_cv", "d_w", "d_b", "ws", "ws_bytes", "algo", "stream"],
}
FNS = list(ARGS)


def _dims(H=128, C=64):
    return _lib.Dims(1000, 800, C, H, H, H, 0)


def _params(w=FAKE):
    return _lib.Params(None, None, None, None, None, None, w, FAKE)


def _call(name, **kw):
    lib = _lib.load()
    a = dict(d=_dims(), p=_params(), cv=FAKE, B=8, out=FAKE, am=FAKE, mx=FAKE, label=FAKE, loss=FAKE, lse=FAKE, scale=0.125,
             scale_device=None, d_out=FAKE, d_cv=FAKE, d_w=FAKE, d_b=FAKE, ws=FAKE, ws_bytes=BIG, algo=_lib.ALGO_AUTO,
             stream=None)
    a.update(kw)
    a["d"] = None if a["d"] == "null" else ctypes.byref(a["d"])
    a["p"] = None if a["p"] == "null" else ctypes.byref(a["p"])
    # a message no call below writes, so that a call which sets none is caught instead of passing on an earlier one
    lib.c2v_loss_argmax(None, None, 0, 0, None, None, None, None, None)
    stale = lib.c2v_last_error()
    rc = getattr(lib, name)(*(a[k] for k in ARGS[name]))
    return rc, stale


def _expect(got, code, name, named=True):
    rc, stale = got
    assert rc == code
    msg = _lib.load().c2v_last_error()
    assert msg and msg != stale, msg
    if named:
        assert name.encode() in msg, msg


NULLS = {
    "params": dict(p="null"), "output_weight": dict(p=_params(None)), "code_vector": dict(cv=None),
    "outputs": dict(out=None), "label": dict(label=None), "lse": dict(lse=None), "d_outputs": dict(d_out=None),
    "outputs+argmax+maxval": dict(out=None, am=None, mx=None), "loss+lse": dict(loss=None, lse=None),
}
CHECKED = {
    "c2v_label_logits": ["params", "output_weight", "code_vector", "outputs"],
    "c2v_label_logits_argmax": ["params", "output_weight", "code_vector", "outputs+argmax+maxval"],
    "c2v_label_loss_argmax": ["params", "output_weight", "code_vector", "label", "loss+lse"],
    "c2v_label_dlogits": ["params", "output_weight", "code_vector", "label", "lse", "outputs"],
    "c2v_label_backward": ["params", "output_weight", "code_vector", "d_outputs"],
    "c2v_label_backward_ws": ["params", "output_weight", "code_vector", "d_outputs"],
}


@pytest.mark.parametrize("fn,case", [(f, c) for f in FNS for c in CHECKED[f]])
def test_label_rejects_null_pointers(fn, case):
    _expect(_call(fn, **NULLS[case]), _lib.C2V_EINVAL, fn)


@pytest.mark.parametrize("fn", FNS)
def test_label_rejects_null_dims(fn):
    _expect(_call(fn, d="null"), _lib.C2V_EINVAL, fn, named=False)


@pytest.mark.parametrize("fn", FNS)
def test_label_rejects_empty_batch(fn):
    _expect(_call(fn, B=0), _lib.C2V_EINVAL, fn)


TC = _lib.ALGO_TCGEN05
UNSUPPORTED = [
    # (entry point, arguments, message names the entry point)
    ("c2v_label_logits", dict(d=_dims(H=30), algo=TC), False),
    ("c2v_label_logits", dict(d=_dims(H=260), algo=TC), False),
    ("c2v_label_logits_argmax", dict(d=_dims(H=30), algo=TC), False),
    ("c2v_label_logits_argmax", dict(d=_dims(H=30), out=None), True),
    ("c2v_label_logits_argmax", dict(d=_dims(H=260), out=None), True),
    ("c2v_label_logits_argmax", dict(B=2049, out=None), True),
    ("c2v_label_loss_argmax", dict(d=_dims(H=30)), True),
    ("c2v_label_loss_argmax", dict(d=_dims(H=260)), True),
    ("c2v_label_loss_argmax", dict(B=2049), True),
    ("c2v_label_dlogits", dict(d=_dims(H=30)), True),
    ("c2v_label_dlogits", dict(d=_dims(H=260)), True),
    ("c2v_label_backward_ws", dict(ws=None, ws_bytes=0, algo=TC), False),
    ("c2v_label_backward_ws", dict(d=_dims(H=30), algo=TC), False),
]


@pytest.mark.parametrize("fn,kw,named", UNSUPPORTED)
def test_label_reports_unsupported_shapes(fn, kw, named):
    _expect(_call(fn, **kw), _lib.C2V_EUNSUPPORTED, fn, named)


def test_label_logits_argmax_without_logits_rejects_cuda_cores():
    _expect(_call("c2v_label_logits_argmax", out=None, algo=_lib.ALGO_FFMA), _lib.C2V_EINVAL, "c2v_label_logits_argmax",
            named=False)


@pytest.mark.parametrize("fn,algo", [("c2v_label_logits", TC), ("c2v_label_logits_argmax", TC),
                                     ("c2v_label_loss_argmax", _lib.ALGO_AUTO), ("c2v_label_dlogits", _lib.ALGO_AUTO)])
def test_label_gemm_reports_a_missing_workspace(fn, algo):
    _expect(_call(fn, ws=None, ws_bytes=0, algo=algo), _lib.C2V_EWORKSPACE, fn, named=False)

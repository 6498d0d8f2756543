"""CPU-side checks of the fused angular-margin entry points (c2v_angular_loss_argmax / _dlogits / _backward_ws): bad
arguments are rejected with C2V_EINVAL and a message before any CUDA call, unsupported shapes with C2V_EUNSUPPORTED."""
import ctypes

from code2vec_b200 import _lib

V = ctypes.c_void_p
FAKE = V(0x1000)          # never dereferenced: every call below fails its argument checks first


def _dims(H=128, C=64):
    return _lib.Dims(1000, 800, C, H, H, H, 0)


def _params():
    return _lib.Params(None, None, None, None, None, None, FAKE, None)


def _einval(rc, name):
    assert rc == _lib.C2V_EINVAL
    msg = _lib.load().c2v_last_error()
    assert name.encode() in msg and msg


def test_angular_loss_argmax_rejects_null_arguments():
    lib = _lib.load()
    d, p = _dims(), _params()
    args = dict(cv=FAKE, label=FAKE, loss=FAKE, lse=FAKE, inv=FAKE)
    for missing in ("params", "cv", "label", "inv", "loss+lse"):
        a = dict(args)
        if missing == "loss+lse":
            a["loss"] = a["lse"] = None
        elif missing != "params":
            a[missing] = None
        rc = lib.c2v_angular_loss_argmax(ctypes.byref(d), None if missing == "params" else ctypes.byref(p), a["cv"],
                                         a["label"], 8, 0.5, 30.0, None, a["loss"], a["lse"], None, None, a["inv"], FAKE,
                                         1 << 20, 0, None)
        _einval(rc, "c2v_angular_loss_argmax")
    rc = lib.c2v_angular_loss_argmax(ctypes.byref(d), ctypes.byref(p), FAKE, FAKE, 0, 0.5, 30.0, None, FAKE, FAKE, None, None,
                                     FAKE, FAKE, 1 << 20, 0, None)
    _einval(rc, "c2v_angular_loss_argmax")                                  # B < 1


def test_angular_loss_argmax_reports_unsupported_shapes():
    lib = _lib.load()
    p = _params()
    for d, B in ((_dims(H=30), 8), (_dims(), 4096)):          # encode_size % 4 != 0; B > 2048
        rc = lib.c2v_angular_loss_argmax(ctypes.byref(d), ctypes.byref(p), FAKE, FAKE, B, 0.5, 30.0, None, FAKE, FAKE, None,
                                         None, FAKE, FAKE, 1 << 20, 0, None)
        assert rc == _lib.C2V_EUNSUPPORTED
        assert b"c2v_angular_loss_argmax" in lib.c2v_last_error()


def test_angular_dlogits_rejects_null_arguments():
    lib = _lib.load()
    d, p = _dims(), _params()
    full = [FAKE, FAKE, FAKE, FAKE]                              # code_vector, label, lse, inv_norms
    for i in range(5):
        a = list(full) + [FAKE]                                  # ... d_dot
        a[i] = None
        rc = lib.c2v_angular_dlogits(ctypes.byref(d), ctypes.byref(p), a[0], a[1], a[2], a[3], 8, 0.5, 30.0, 0.125, None,
                                     a[4], FAKE, 1 << 20, 0, None)
        _einval(rc, "c2v_angular_dlogits")
    rc = lib.c2v_angular_dlogits(ctypes.byref(d), None, FAKE, FAKE, FAKE, FAKE, 8, 0.5, 30.0, 0.125, None, FAKE, FAKE,
                                 1 << 20, 0, None)
    _einval(rc, "c2v_angular_dlogits")
    rc = lib.c2v_angular_dlogits(ctypes.byref(_dims(H=30)), ctypes.byref(p), FAKE, FAKE, FAKE, FAKE, 8, 0.5, 30.0, 0.125,
                                 None, FAKE, FAKE, 1 << 20, 0, None)
    assert rc == _lib.C2V_EUNSUPPORTED


def test_angular_backward_ws_rejects_null_arguments():
    lib = _lib.load()
    d, p = _dims(), _params()
    for i in range(3):                                           # code_vector, d_dot, inv_norms
        a = [FAKE, FAKE, FAKE]
        a[i] = None
        rc = lib.c2v_angular_backward_ws(ctypes.byref(d), ctypes.byref(p), a[0], a[1], a[2], 8, FAKE, FAKE, FAKE, 1 << 20, 0,
                                         None)
        _einval(rc, "c2v_angular_backward_ws")
    rc = lib.c2v_angular_backward_ws(ctypes.byref(d), None, FAKE, FAKE, FAKE, 8, FAKE, FAKE, FAKE, 1 << 20, 0, None)
    _einval(rc, "c2v_angular_backward_ws")
    rc = lib.c2v_angular_backward_ws(ctypes.byref(d), ctypes.byref(p), FAKE, FAKE, FAKE, 0, FAKE, FAKE, FAKE, 1 << 20, 0, None)
    _einval(rc, "c2v_angular_backward_ws")

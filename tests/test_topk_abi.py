"""CPU-side checks of the fused top-k entry points (c2v_label_topk / c2v_angular_topk): bad arguments are rejected with
C2V_EINVAL, shapes the fused kernel does not take with C2V_EUNSUPPORTED and short workspaces with C2V_EWORKSPACE, each
with a message and before any CUDA call."""
import ctypes
import os
import re

import pytest

from code2vec_b200 import _lib

V = ctypes.c_void_p
FAKE = V(0x1000)          # never dereferenced: every call below fails its argument checks first
BIG = 1 << 40             # a workspace size that passes the size check


def _dims(H=128, C=64):
    return _lib.Dims(1000, 800, C, H, H, H, 0)


def _params(w=FAKE):
    return _lib.Params(None, None, None, None, None, None, w, None)


def _call(name, d=None, p=None, cv=FAKE, B=8, k=4, idx=FAKE, val=FAKE, prob=None, ws=FAKE, ws_bytes=BIG, algo=0):
    lib = _lib.load()
    d = _dims() if d is None else d
    p = _params() if p is None else p
    dp = None if d == "null" else ctypes.byref(d)
    pp = None if p == "null" else ctypes.byref(p)
    if name == "c2v_label_topk":
        return lib.c2v_label_topk(dp, pp, cv, B, k, idx, val, prob, ws, ws_bytes, algo, None)
    return lib.c2v_angular_topk(dp, pp, cv, B, k, 30.0, idx, val, prob, ws, ws_bytes, algo, None)


def _expect(rc, code, name):
    assert rc == code
    msg = _lib.load().c2v_last_error()
    assert msg and name.encode() in msg, msg


FNS = ["c2v_label_topk", "c2v_angular_topk"]


@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("case", ["dims", "params", "output_weight", "code_vector", "indices", "values", "B<1", "k<1", "k>C"])
def test_topk_rejects_bad_arguments(fn, case):
    kw = {"dims": dict(d="null"), "params": dict(p="null"), "output_weight": dict(p=_params(None)),
          "code_vector": dict(cv=None), "indices": dict(idx=None), "values": dict(val=None), "B<1": dict(B=0),
          "k<1": dict(k=0), "k>C": dict(d=_dims(C=3), k=4)}[case]
    _expect(_call(fn, **kw), _lib.C2V_EINVAL, fn)


@pytest.mark.parametrize("fn", FNS)
@pytest.mark.parametrize("case", ["encode%4", "encode>256", "B>2048", "k>TOPK_MAX", "ffma"])
def test_topk_reports_unsupported_shapes(fn, case):
    kw = {"encode%4": dict(d=_dims(H=30)), "encode>256": dict(d=_dims(H=260)), "B>2048": dict(B=2049),
          "k>TOPK_MAX": dict(k=_lib.TOPK_MAX + 1), "ffma": dict(algo=_lib.ALGO_FFMA)}[case]
    _expect(_call(fn, **kw), _lib.C2V_EUNSUPPORTED, fn)


@pytest.mark.parametrize("fn", FNS)
def test_topk_reports_a_short_workspace(fn):
    lib = _lib.load()
    d = _dims()
    need = lib.c2v_label_topk_workspace_bytes(ctypes.byref(d), 8, 4)
    _expect(_call(fn, ws_bytes=need - 1), _lib.C2V_EWORKSPACE, fn)
    _expect(_call(fn, ws=None), _lib.C2V_EWORKSPACE, fn)


def test_topk_support_and_workspace_size():
    lib = _lib.load()
    header = open(os.path.join(os.path.dirname(_lib._HERE), "include", "c2v_b200.h")).read()
    assert int(re.search(r"#define C2V_TOPK_MAX (\d+)", header).group(1)) == _lib.TOPK_MAX
    d = _dims(C=195299, H=100)
    for B in (1, 1024, 2048):
        base = lib.c2v_label_workspace_bytes(ctypes.byref(d), B)
        for k in (1, 10, _lib.TOPK_MAX):
            assert lib.c2v_label_topk_supported(ctypes.byref(d), B, k) == 1
            assert lib.c2v_label_topk_workspace_bytes(ctypes.byref(d), B, k) >= base
    assert lib.c2v_label_topk_supported(ctypes.byref(d), 2049, 10) == 0
    assert lib.c2v_label_topk_supported(ctypes.byref(d), 8, _lib.TOPK_MAX + 1) == 0
    assert lib.c2v_label_topk_supported(ctypes.byref(d), 8, 0) == 0
    assert lib.c2v_label_topk_supported(ctypes.byref(_dims(H=30)), 8, 4) == 0
    assert lib.c2v_label_topk_supported(ctypes.byref(_dims(C=3)), 8, 4) == 0
    assert lib.c2v_label_topk_workspace_bytes(ctypes.byref(d), 8, _lib.TOPK_MAX + 1) == 0

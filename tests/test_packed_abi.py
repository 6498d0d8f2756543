"""CPU-side checks of the packed (CSR) batch entry points: argument checks before any CUDA call, workspace sizes, the host
bag-offsets function of the builder and PackedBags' validation of the offsets."""
import ctypes

import numpy as np
import pytest
import torch

from code2vec_b200 import _lib
from code2vec_b200 import functional as CF
from code2vec_b200.batch_builder import packed_offsets

D = _lib.Dims(1000, 800, 64, 128, 128, 128, 0)
P = _lib.Params(*([ctypes.c_void_p(16)] * 8))       # never dereferenced: every call below fails its checks first
G = _lib.Grads(*([ctypes.c_void_p(16)] * 6))
X = ctypes.c_void_p(16)                              # a stand-in device pointer


def _err():
    return _lib.load().c2v_last_error().decode()


def _fwd(B=4, N=10, L=7, ws_bytes=1 << 30, algo=0, nulls=()):
    a = {k: (None if k in nulls else X) for k in ("starts", "paths", "ends", "offsets", "cv", "att", "ws")}
    return _lib.load().c2v_encode_forward_packed(ctypes.byref(D), ctypes.byref(P), a["starts"], a["paths"], a["ends"],
                                                 a["offsets"], B, N, L, None, a["cv"], a["att"], None, a["ws"], ws_bytes,
                                                 algo, None)


def _bwd(B=4, N=10, L=7, ws_bytes=1 << 30, phase=0, nulls=()):
    a = {k: (None if k in nulls else X) for k in ("starts", "paths", "ends", "offsets", "cv", "att", "dcv", "ws")}
    return _lib.load().c2v_encode_backward_packed(ctypes.byref(D), ctypes.byref(P), a["starts"], a["paths"], a["ends"],
                                                  a["offsets"], B, N, L, None, a["cv"], a["att"], None, a["dcv"], None,
                                                  ctypes.byref(G), a["ws"], ws_bytes, phase, None)


@pytest.mark.parametrize("null", ["starts", "paths", "ends", "offsets", "cv", "att", "ws"])
def test_forward_rejects_null_pointers(null):
    assert _fwd(nulls=(null,)) == _lib.C2V_EINVAL
    assert "NULL" in _err()


@pytest.mark.parametrize("B,N,L", [(0, 10, 7), (4, 3, 7), (4, 10, 0), (4, 29, 7)])
def test_forward_rejects_bad_shapes(B, N, L):
    assert _fwd(B, N, L) == _lib.C2V_EINVAL
    assert "B <= N <= B * L" in _err()


def test_forward_rejects_small_workspace_and_unknown_algo():
    need = _lib.load().c2v_encode_packed_workspace_bytes(ctypes.byref(D), 4, 10)
    assert _fwd(ws_bytes=need - 1) == _lib.C2V_EWORKSPACE
    assert "workspace too small" in _err()
    assert _fwd(ws_bytes=need, algo=7) == _lib.C2V_EINVAL
    assert "unknown algo 7" in _err()


@pytest.mark.parametrize("null", ["starts", "paths", "ends", "offsets", "cv", "att", "dcv", "ws"])
def test_backward_rejects_null_pointers(null):
    assert _bwd(nulls=(null,)) == _lib.C2V_EINVAL
    assert "NULL" in _err()


def test_backward_rejects_bad_shapes_phase_and_small_workspace():
    for B, N, L in [(0, 10, 7), (4, 3, 7), (4, 10, 0), (4, 29, 7)]:
        assert _bwd(B, N, L) == _lib.C2V_EINVAL
        assert "B <= N <= B * L" in _err()
    assert _bwd(phase=3) == _lib.C2V_EINVAL
    assert "phase 3" in _err()
    need = _lib.load().c2v_encode_backward_packed_workspace_bytes(ctypes.byref(D), 4, 10)
    assert _bwd(ws_bytes=need - 1) == _lib.C2V_EWORKSPACE
    assert "workspace too small" in _err()


def test_build_batch_packed_rejects_bad_arguments():
    lib = _lib.load()
    args = dict(offsets=X, contexts=X, n_items=5, ids=X, bag_off=X, B=4, L=7)
    for bad in ({"offsets": None}, {"contexts": None}, {"ids": None}, {"bag_off": None}, {"n_items": 0}, {"B": 0},
                {"L": 0}):
        a = {**args, **bad}
        rc = lib.c2v_build_batch_packed(a["offsets"], a["contexts"], a["n_items"], a["ids"], None, a["B"], a["L"], 0, 2, 1,
                                        a["bag_off"], X, X, X, None, None)
        assert rc == _lib.C2V_EINVAL, bad
        assert "c2v_build_batch_packed: bad argument" in _err()


def test_workspace_sizes_grow_with_n_and_ignore_l():
    lib = _lib.load()
    for fn in (lib.c2v_encode_packed_workspace_bytes, lib.c2v_encode_backward_packed_workspace_bytes):
        sizes = [fn(ctypes.byref(D), 64, n) for n in (64, 2000, 12800)]
        assert all(s > 0 and s % 1024 == 0 for s in sizes)
        assert sizes[0] < sizes[1] < sizes[2]
        assert fn(ctypes.byref(D), 64, 63) == 0 and fn(ctypes.byref(D), 0, 64) == 0
    # the packed sizes take no L: a full packed batch is no larger than the [B, L] workspace plus its int32 row map
    full = lib.c2v_encode_packed_workspace_bytes(ctypes.byref(D), 64, 64 * 200)
    assert full <= lib.c2v_encode_workspace_bytes(ctypes.byref(D), 64, 200) + 64 * 200 * 4 + 1024
    fb = lib.c2v_encode_backward_packed_workspace_bytes(ctypes.byref(D), 64, 64 * 200)
    assert fb <= lib.c2v_encode_backward_workspace_bytes(ctypes.byref(D), 64, 200) + 64 * 200 * 4 + 1024


def test_packed_offsets_truncate_and_pad():
    counts = np.array([5, 0, 300, 200, 1, 199])
    off = packed_offsets(counts, [0, 1, 2, 3, 4, 5, -1, 6, 2], 200)
    assert off.dtype == np.int64
    assert np.diff(off).tolist() == [5, 1, 200, 200, 1, 199, 1, 1, 200]
    assert off[0] == 0 and off[-1] == np.diff(off).sum()
    assert packed_offsets(counts, [], 200).tolist() == [0]


def _bags(offsets, L=4, N=None):
    n = int(np.asarray(offsets)[-1]) if N is None else N
    t = torch.zeros(n, dtype=torch.int64)
    return CF.PackedBags(t, t.clone(), t.clone(), offsets, L)


@pytest.mark.parametrize("offsets,N,msg", [
    ([1, 3, 5], 5, "offsets\\[0\\]"),          # does not start at 0
    ([0, 3, 2, 5], 5, "bag 1 holds -1"),        # decreasing
    ([0, 3, 3, 5], 5, "bag 1 holds 0"),         # empty bag
    ([0, 5, 7], 7, "bag 0 holds 5"),            # longer than L
    ([0], 0, "B \\+ 1 >= 2"),                   # no bag
    ([[0, 1], [1, 2]], 2, "1-D"),
])
def test_packed_bags_rejects_malformed_offsets(offsets, N, msg, monkeypatch):
    def no_library():
        raise AssertionError("the library must not be reached")
    monkeypatch.setattr(_lib, "load", no_library)
    with pytest.raises(ValueError, match=msg):
        _bags(offsets, N=N)


def test_packed_bags_rejects_mismatched_n_and_accepts_a_valid_batch():
    with pytest.raises(ValueError, match="offsets\\[B\\]"):
        _bags([0, 2, 4], N=5)
    t = torch.zeros(5, dtype=torch.int64)
    with pytest.raises(ValueError, match="contexts"):
        CF.PackedBags(t, t[:4], t, [0, 2, 5], 4)
    b = _bags(torch.tensor([0, 1, 4, 5]), L=4)
    assert (b.B, b.N, b.L) == (3, 5, 4)
    assert b.lengths().tolist() == [1, 3, 1]
    s, p, e = CF.PackedBags(torch.arange(1, 6), torch.arange(1, 6), torch.arange(1, 6), [0, 1, 4, 5], 4).padded()
    assert s.tolist() == [[1, 0, 0, 0], [2, 3, 4, 0], [5, 0, 0, 0]]

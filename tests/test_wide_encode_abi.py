"""No GPU: the encode backward's envelope above encode_size 256 (up to 512) as the host side sees it.

  * the backward workspace queries of every training case of tests/shape_envelope.py, in both deterministic modes, are
    the bytes the library reserved before the envelope grew (recorded from that build), so shapes up to 256 and the
    260-wide forward-only case keep their layout;
  * the queries are positive for the shapes between 257 and 512;
  * above 512 every encode-backward entry point still reports C2V_EUNSUPPORTED (NotImplementedError through
    _lib.check) with a message naming the limit, before it touches the device.
"""
import ctypes

import pytest

from code2vec_b200 import _lib
from code2vec_b200 import functional as CF
import shape_envelope as SE

# case -> (padded, packed at N = B * L) bytes with the deterministic mode off, then on
WORKSPACE = {
    "e4-4-h100-b1x1": (795648, 796672, 2771968, 2772992),
    "e4-4-h100-b129x33": (2497536, 2514944, 4833280, 4850688),
    "e4-4-h100-b7x333": (1727488, 1737728, 3898368, 3908608),
    "e124-124-h128-b1x1": (980992, 982016, 15012864, 15013888),
    "e124-124-h128-b129x33": (3160064, 3177472, 23936000, 23953408),
    "e124-124-h128-b7x333": (2173952, 2184192, 19896320, 19906560),
    "e132-132-h256-b1x1": (1196032, 1197056, 29777920, 29778944),
    "e132-132-h256-b129x33": (5554176, 5571584, 41306112, 41323520),
    "e132-132-h256-b7x333": (3581952, 3592192, 36085760, 36096000),
    "e256-256-h256-b1x1": (1576960, 1577984, 54539264, 54540288),
    "e256-256-h256-b129x33": (5935104, 5952512, 72664064, 72681472),
    "e256-256-h256-b7x333": (3962880, 3973120, 64458752, 64468992),
    "e200-200-h192-b1x1": (1251328, 1252352, 32979968, 32980992),
    "e200-200-h192-b129x33": (4519936, 4537344, 47036416, 47053824),
    "e200-200-h192-b7x333": (3041280, 3051520, 40673280, 40683520),
    "e64-64-h60-b1x1": (836608, 837632, 5209088, 5210112),
    "e64-64-h60-b129x33": (1857536, 1874944, 9782272, 9799680),
    "e64-64-h60-b7x333": (1395712, 1405952, 7710720, 7720960),
    "e128-128-h4-b1x1": (796672, 797696, 2270208, 2271232),
    "e128-128-h4-b129x33": (864256, 881664, 9294848, 9312256),
    "e128-128-h4-b7x333": (833536, 843776, 6113280, 6123520),
    "e256-256-h252-b1x1": (1564672, 1565696, 53715968, 53716992),
    "e256-256-h252-b129x33": (5855232, 5872640, 71773184, 71790592),
    "e256-256-h252-b7x333": (3913728, 3923968, 63598592, 63608832),
    "e128-96-h128-b1x1": (970752, 971776, 14347264, 14348288),
    "e128-96-h128-b129x33": (3149824, 3167232, 22938624, 22956032),
    "e128-96-h128-b7x333": (2163712, 2173952, 19048448, 19058688),
    "e37-29-h45-b1x1": (811008, 812032, 3329024, 3330048),
    "e37-29-h45-b129x33": (1576960, 1594368, 6074368, 6091776),
    "e37-29-h45-b7x333": (1229824, 1240064, 4829184, 4839424),
    "e128-128-h260-b1x1": (1190912, 1191936, 29403136, 29404160),
    "e128-128-h260-b129x33": (5616640, 5634048, 40785920, 40803328),
    "e128-128-h260-b7x333": (3613696, 3623936, 35632128, 35642368),
    "e124-124-h128-b129x33-packed": (3160064, 3177472, 23936000, 23953408),
    "e200-200-h192-b129x33-packed": (4519936, 4537344, 47036416, 47053824),
    "e128-96-h128-b129x33-packed": (3149824, 3167232, 22938624, 22956032),
    "e37-29-h45-b129x33-packed": (1576960, 1594368, 6074368, 6091776),
    "e128-128-h128-b85x200": (9690112, 9758720, 51902464, 51971072),
    "table-past-4GB": (1138688, 1140736, 16046080, 16048128),
}

WIDE = ((128, 128, 384), (128, 128, 260), (100, 100, 300), (124, 124, 508), (256, 256, 512), (128, 96, 384),
        (37, 29, 301))


@pytest.fixture
def det_mode():
    lib = _lib.load()
    saved = lib.c2v_get_deterministic()
    yield lib
    lib.c2v_set_deterministic(saved)


def _queries(lib, c):
    d = CF.make_dims(c["T"], c["P"], c["C"], c["Et"], c["Ep"], c["H"])
    return (lib.c2v_encode_backward_workspace_bytes(ctypes.byref(d), c["B"], c["L"]),
            lib.c2v_encode_backward_packed_workspace_bytes(ctypes.byref(d), c["B"], c["B"] * c["L"]))


def test_every_envelope_case_is_recorded():
    assert set(WORKSPACE) == set(SE.TRAIN)


@pytest.mark.parametrize("case", list(SE.TRAIN))
def test_envelope_workspace_unchanged(case, det_mode):
    lib = det_mode
    got = []
    for det in (0, 1):
        assert lib.c2v_set_deterministic(det) == _lib.C2V_OK
        got += _queries(lib, SE.TRAIN[case])
    assert tuple(got) == WORKSPACE[case]


@pytest.mark.parametrize("shape", WIDE, ids=lambda s: f"e{s[0]}-{s[1]}-h{s[2]}")
def test_wide_workspace_positive(shape, det_mode):
    lib = det_mode
    Et, Ep, H = shape
    for det in (0, 1):
        lib.c2v_set_deterministic(det)
        for B, L in SE.BAGS + ((1024, 200),):
            c = dict(T=SE.T_SMALL, P=SE.P_SMALL, C=SE.C_TRAIN, Et=Et, Ep=Ep, H=H, B=B, L=L)
            padded, packed = _queries(lib, c)
            # at least dx [N, H], the W^T copy [D, H] and (deterministic) the dC rows [N, D]
            floor = 4 * (B * L * H + (2 * Et + Ep) * H + (B * L * (2 * Et + Ep) if det else 0))
            assert padded >= floor and packed >= floor, (det, B, L, padded, packed, floor)


def test_wide_tensor_core_workspace_holds_every_window():
    """256 < H <= 512 with Et = Ep <= 256: the dC kernel's W^T images grow to n_db x n_hb = 2 x 4 (192 KB each); below,
    every shape reserves 2 x 2"""
    lib = _lib.load()
    img = 6 * 2 * (128 * 64 * 2)                            # 6 tiles of {hi, lo} [128 d x 64 h] fp16

    def ws(E, H):
        return lib.c2v_encode_backward_workspace_bytes(ctypes.byref(CF.make_dims(1000, 1000, 10, E, E, H)), 1, 1)

    def grown(E, H):                                        # dx of one context and the W^T copy, 1 KB aligned
        kb = lambda n: -(-n // 1024) * 1024
        return kb(H * 4) - kb(256 * 4) + kb(3 * E * H * 4) - kb(3 * E * 256 * 4)
    assert ws(256, 512) - ws(256, 256) == grown(256, 512) + 4 * img
    assert ws(256, 384) - ws(256, 256) == grown(256, 384) + 2 * img     # 2 x 3
    assert ws(128, 512) - ws(128, 256) == grown(128, 512)   # 1 x 4 images: as many as 2 x 2
    assert ws(100, 300) - ws(100, 256) == grown(100, 300)   # 1 x 3


class _Fake:
    """non-NULL, 16-byte aligned stand-ins for device pointers: the calls below fail before any device access"""
    addr = 1 << 20

    @classmethod
    def ptr(cls):
        cls.addr += 4096
        return ctypes.c_void_p(cls.addr)


def _call_args(H, B=3, L=5):
    d = CF.make_dims(100, 100, 10, 128, 128, H)
    f = _Fake.ptr
    p = _lib.Params(*(f().value for _ in range(8)))
    g = _lib.Grads(*(f().value for _ in range(6)))
    drop = _lib.Dropout(0.25, 1, 7)
    return d, p, g, drop, f


@pytest.mark.parametrize("H", [513, 516, 1024])
def test_above_512_is_unsupported(H):
    lib = _lib.load()
    d, p, g, drop, f = _call_args(H)
    B, L, N = 3, 5, 9
    ws_bytes = 1 << 40
    slots = _lib.RowSlots(f().value, f().value)
    calls = {
        "c2v_encode_backward_phased": lambda: lib.c2v_encode_backward_phased(
            ctypes.byref(d), ctypes.byref(p), f(), f(), f(), B, L, ctypes.byref(drop), f(), f(), f(), f(), f(),
            ctypes.byref(g), f(), ws_bytes, 0, None),
        "c2v_encode_backward_packed": lambda: lib.c2v_encode_backward_packed(
            ctypes.byref(d), ctypes.byref(p), f(), f(), f(), f(), B, N, L, ctypes.byref(drop), f(), f(), f(), f(), f(),
            ctypes.byref(g), f(), ws_bytes, 1, None),
        "c2v_encode_backward_sparse": lambda: lib.c2v_encode_backward_sparse(
            ctypes.byref(d), ctypes.byref(p), f(), f(), f(), B, L, ctypes.byref(drop), f(), f(), None, f(), None,
            ctypes.byref(g), ctypes.byref(slots), f(), ws_bytes, 0, None),
        "c2v_encode_backward_packed_sparse": lambda: lib.c2v_encode_backward_packed_sparse(
            ctypes.byref(d), ctypes.byref(p), f(), f(), f(), f(), B, N, L, ctypes.byref(drop), f(), f(), f(), f(), f(),
            ctypes.byref(g), ctypes.byref(slots), f(), ws_bytes, 2, None),
    }
    for name, call in calls.items():
        rc = call()
        assert rc == _lib.C2V_EUNSUPPORTED, (name, rc, lib.c2v_last_error())
        msg = lib.c2v_last_error().decode()
        assert "512" in msg and str(H) in msg, (name, msg)
        with pytest.raises(NotImplementedError, match="encode_size <= 512"):
            _lib.check(rc, name)

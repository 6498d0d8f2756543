"""No GPU: the shape-envelope case table (tests/shape_envelope.py) against the library's exported dispatch predicates and
workspace-size queries, so that a case whose expected kernels drift from the dispatch rules fails on the CPU."""
import ctypes

import pytest

from code2vec_b200 import _lib
from code2vec_b200 import functional as CF
import shape_envelope as SE


def _dims(T, P, C, Et, Ep, H):
    return CF.make_dims(T, P, C, Et, Ep, H)


def test_every_shape_is_in_the_table_once():
    assert set(SE.SHAPES.values()) == set(SE.GROUPS)
    for shape in SE.PACKED:
        assert shape in SE.SHAPES
    assert {SE.SHAPES[s] for s in SE.PACKED} == set(SE.GROUPS) - {"forward-only"}, "one packed shape per group"
    for name, paths in SE.GROUPS.items():
        assert set(paths) == (set(SE.KERNELS) if name != "forward-only" else {"encode", "label"})


@pytest.mark.parametrize("case", list(SE.TRAIN))
def test_training_case_path_matches_the_predicates(case):
    c = SE.TRAIN[case]
    d = _dims(c["T"], c["P"], c["C"], c["Et"], c["Ep"], c["H"])
    lib = _lib.load()
    tc = SE.TC
    assert bool(lib.c2v_encode_supports_tcgen05(ctypes.byref(d))) == (c["paths"]["encode"] == tc)
    assert CF.label_loss_supported(d, c["B"]) == (c["paths"]["label"] == tc)
    assert CF.label_topk_supported(d, c["B"], 1) == (c["paths"]["label"] == tc)
    # dW / dC are not exported: their rule (shape_envelope's docstring) restated on the case's dims
    E, H = c["Et"], c["H"]
    if "dw" not in c["paths"]:                   # forward only: the encode backward takes H <= 256
        assert H > 256
        return
    fits = c["Et"] == c["Ep"] and E <= 256 and H <= 256 and E % 4 == 0 and H % 4 == 0
    under_4gb = max(c["T"], c["P"]) * E * 4 < 2 ** 32
    assert (fits and under_4gb) == (c["paths"]["dw"] == tc)
    assert (fits and max(c["T"], c["P"]) * (E // 4) < 2 ** 32 - 1) == (c["paths"]["dc"] == tc)
    assert lib.c2v_encode_workspace_bytes(ctypes.byref(d), c["B"], c["L"]) > 0
    assert lib.c2v_encode_backward_workspace_bytes(ctypes.byref(d), c["B"], c["L"]) > 0
    assert lib.c2v_label_workspace_bytes(ctypes.byref(d), c["B"]) > 0
    if c["layout"] == "packed":
        N = c["B"] * c["L"]
        assert lib.c2v_encode_packed_workspace_bytes(ctypes.byref(d), c["B"], N) > 0
        assert lib.c2v_encode_backward_packed_workspace_bytes(ctypes.byref(d), c["B"], N) > 0


@pytest.mark.parametrize("case", list(SE.LABEL))
def test_label_case_runs_on_the_tensor_cores(case):
    c = SE.LABEL[case]
    d = _dims(10, 10, c["C"], c["H"], c["H"], c["H"])
    lib = _lib.load()
    assert CF.label_loss_supported(d, c["B"])
    for k in SE.topk_ks(c["C"]):
        assert CF.label_topk_supported(d, c["B"], k)
        assert lib.c2v_label_topk_workspace_bytes(ctypes.byref(d), c["B"], k) > 0
    assert lib.c2v_label_workspace_bytes(ctypes.byref(d), c["B"]) > 0
    assert lib.c2v_label_loss_opts_workspace_bytes(ctypes.byref(d), c["B"]) > 0


def test_label_envelope_edges():
    """the covering set spans the whole B / C / H envelope, and one step past it leaves the fused kernels"""
    Bs = {c["B"] for c in SE.LABEL.values()}
    Cs = {c["C"] for c in SE.LABEL.values()}
    Hs = {c["H"] for c in SE.LABEL.values()}
    assert Bs == {1, 127, 128, 129, 1793, 1920, 2048}
    assert Cs == {1, 2, 127, 128, 129, 1023, 16896, 16897, 195299}
    assert Hs == {4, 60, 64, 68, 100, 252, 256}
    assert {(SE.LABEL[n]["B"], SE.LABEL[n]["C"]) for n in SE.LABEL_GROUPS_CASES} == {(1793, 16896), (1920, 16897)}
    d = _dims(10, 10, 1000, 128, 128, 128)
    assert CF.label_loss_supported(d, 2048) and not CF.label_loss_supported(d, 2049)
    assert not CF.label_topk_supported(d, 2048, _lib.TOPK_MAX + 1)
    for H in (0, 2, 258, 260):
        assert not CF.label_loss_supported(_dims(10, 10, 1000, 128, 128, H), 128)


def test_default_label_order_at_132_sms():
    """on a 132-SM H100 the groups-order cases take groups order by default and the other cases lanes order"""
    for name, c in SE.LABEL.items():
        want = "groups" if name in SE.LABEL_GROUPS_CASES else "lanes"
        assert SE.default_label_order(c["B"], c["C"], 132) == want, name

"""Host side of the matmul precision (no GPU needed): c2v_set_matmul_precision / c2v_get_matmul_precision are per thread
and reject unknown modes, functional.sync_matmul_precision maps every torch setter of the fp32 matmul switch to the right
mode without raising and calls the library only on a change, the workspace sizes do not depend on the mode, and a
captured graph refuses a changed switch."""
import ctypes
import threading

import pytest
import torch

from code2vec_b200 import _lib
from code2vec_b200 import functional as CF
from code2vec_b200.graphs import GraphedPredict, GraphedTrainStep
from code2vec_b200.model import Code2Vec


class _Opt:
    terminal_count, path_count, label_count = 50, 60, 7
    terminal_embed_size = path_embed_size = 8
    encode_size = 16
    dropout_prob = 0.0
    angular_margin_loss = False
    angular_margin, inverse_temp = 0.5, 30.0


def _batch():
    z = torch.zeros(4, 8, dtype=torch.int64)
    return z, z, z, torch.zeros(4, dtype=torch.int64)


@pytest.fixture
def lib():
    lib = _lib.load()
    yield lib
    lib.c2v_set_matmul_precision(_lib.MATMUL_IEEE)
    CF._det.__dict__.pop("tf32", None)


@pytest.fixture
def torch_switch():
    """restores torch's switch through the new API (the legacy getters raise once it has been used)"""
    saved = torch.backends.fp32_precision, torch.backends.cuda.matmul.fp32_precision
    yield
    torch.backends.fp32_precision = saved[0]
    torch.backends.cuda.matmul.fp32_precision = saved[1]


def test_set_get_is_per_thread(lib):
    assert lib.c2v_get_matmul_precision() == _lib.MATMUL_IEEE
    assert lib.c2v_set_matmul_precision(_lib.MATMUL_TF32) == 0
    assert lib.c2v_get_matmul_precision() == _lib.MATMUL_TF32
    seen = {}

    def other():
        seen["initial"] = lib.c2v_get_matmul_precision()
        lib.c2v_set_matmul_precision(_lib.MATMUL_TF32)
        lib.c2v_set_matmul_precision(_lib.MATMUL_IEEE)
        seen["after"] = lib.c2v_get_matmul_precision()
    t = threading.Thread(target=other)
    t.start()
    t.join()
    assert seen == {"initial": _lib.MATMUL_IEEE, "after": _lib.MATMUL_IEEE}
    assert lib.c2v_get_matmul_precision() == _lib.MATMUL_TF32        # untouched by the other thread
    lib.c2v_set_matmul_precision(_lib.MATMUL_IEEE)
    assert lib.c2v_get_matmul_precision() == _lib.MATMUL_IEEE


@pytest.mark.parametrize("mode", [-1, 2, 3, 1 << 30])
def test_other_modes_are_rejected(lib, mode):
    lib.c2v_set_matmul_precision(_lib.MATMUL_TF32)
    assert lib.c2v_set_matmul_precision(mode) == -1                   # C2V_EINVAL
    assert b"c2v_set_matmul_precision" in lib.c2v_last_error()
    assert lib.c2v_get_matmul_precision() == _lib.MATMUL_TF32        # the mode is left as it was


def _legacy_allow(on):
    torch.backends.cuda.matmul.allow_tf32 = on


def _precision(p):
    torch.set_float32_matmul_precision(p)


def _new_api(p):
    torch.backends.cuda.matmul.fp32_precision = p


def _global(p):
    torch.backends.fp32_precision = p


# (setter, value, expected library mode)
SETTERS = [(_precision, "highest", 0), (_precision, "high", 1), (_precision, "medium", 1),
           (_legacy_allow, False, 0), (_legacy_allow, True, 1),
           (_new_api, "ieee", 0), (_new_api, "tf32", 1), (_new_api, "none", 0),
           (_global, "tf32", 1), (_global, "ieee", 0)]


@pytest.mark.parametrize("setter,value,mode", SETTERS, ids=[f"{s.__name__}-{v}" for s, v, _ in SETTERS])
def test_sync_follows_every_torch_setter(lib, torch_switch, setter, value, mode):
    setter(value)
    assert CF.sync_matmul_precision() is bool(mode)
    assert lib.c2v_get_matmul_precision() == mode


def test_sequence_of_setters(lib, torch_switch):
    """the new-API setters first, then the legacy ones: the getter the library reads never raises"""
    for setter, value, mode in SETTERS[5:] + SETTERS[:5] + SETTERS[5:]:
        setter(value)
        assert CF.sync_matmul_precision() is bool(mode)
        assert lib.c2v_get_matmul_precision() == mode


def test_library_is_called_only_on_a_change(lib, torch_switch, monkeypatch):
    calls = []
    real = _lib.load()

    class Spy:
        def __getattr__(self, name):
            return getattr(real, name)

        def c2v_set_matmul_precision(self, mode):
            calls.append(mode)
            return real.c2v_set_matmul_precision(mode)
    monkeypatch.setattr(_lib, "load", lambda: Spy())
    _new_api("none")
    CF.sync_matmul_precision()
    calls.clear()
    for _ in range(3):
        CF.sync_matmul_precision()
    assert calls == []
    _new_api("tf32")
    for _ in range(3):
        CF.sync_matmul_precision()
    assert calls == [_lib.MATMUL_TF32]
    _precision("highest")
    CF.sync_matmul_precision()
    CF.sync_matmul_precision()
    assert calls == [_lib.MATMUL_TF32, _lib.MATMUL_IEEE]


def _sizes(lib, dims, B, L, N):
    d = ctypes.byref(dims)
    return {"encode": lib.c2v_encode_workspace_bytes(d, B, L),
            "encode_packed": lib.c2v_encode_packed_workspace_bytes(d, B, N),
            "backward": lib.c2v_encode_backward_workspace_bytes(d, B, L),
            "backward_packed": lib.c2v_encode_backward_packed_workspace_bytes(d, B, N),
            "label": lib.c2v_label_workspace_bytes(d, B),
            "label_opts": lib.c2v_label_loss_opts_workspace_bytes(d, B),
            "topk": lib.c2v_label_topk_workspace_bytes(d, B, 5)}


@pytest.mark.parametrize("shape", [(360633, 342846, 8192, 128, 128, 128, 1024, 200), (360633, 342846, 195299, 100, 100, 100, 1024, 200),
                                   (360633, 342846, 8192, 256, 256, 256, 512, 200), (3000, 4000, 257, 37, 29, 45, 48, 33)])
@pytest.mark.parametrize("det", [0, 1])
def test_workspace_sizes_do_not_depend_on_the_mode(lib, shape, det):
    T, P, C, Et, Ep, H, B, L = shape
    dims = CF.make_dims(T, P, C, Et, Ep, H)
    N = B * L // 2
    lib.c2v_set_deterministic(det)
    try:
        ieee = _sizes(lib, dims, B, L, N)
        lib.c2v_set_matmul_precision(_lib.MATMUL_TF32)
        tf32 = _sizes(lib, dims, B, L, N)
    finally:
        lib.c2v_set_deterministic(0)
    assert all(v > 0 for v in ieee.values())
    assert tf32 == ieee


@pytest.mark.parametrize("setter,value", [(_precision, "high"), (_legacy_allow, True), (_new_api, "tf32"), (_global, "tf32")])
def test_similarity_fallback_turns_tf32_off_under_every_setter(torch_switch, setter, value):
    """CodeVectorIndex's torch fallback keeps its fp32 contract in TF32 mode, whichever API turned TF32 on"""
    from code2vec_b200.similarity import _fp32_matmul
    setter(value)
    assert CF.torch_matmul_tf32()
    with _fp32_matmul():
        assert not CF.torch_matmul_tf32()
    assert CF.torch_matmul_tf32()


@pytest.mark.parametrize("matmul", [None, "tf32", "ieee"])
def test_similarity_fallback_restores_the_switch_as_it_was(torch_switch, matmul):
    """after the fallback the matmul setting still follows the global one when it did before, and keeps an explicit
    value otherwise"""
    from code2vec_b200.similarity import _fp32_matmul
    _global("tf32")
    if matmul is not None:
        _new_api(matmul)
    with _fp32_matmul():
        assert not CF.torch_matmul_tf32()
    assert torch.backends.fp32_precision == "tf32"
    assert torch.backends.cuda.matmul.fp32_precision == (matmul or "tf32")
    _global("ieee")
    assert torch.backends.cuda.matmul.fp32_precision == (matmul or "ieee")


@pytest.mark.parametrize("on", [False, True])
def test_similarity_fallback_keeps_the_legacy_api_usable(torch_switch, on):
    """a user of the legacy switch alone can still read it after the fallback ran"""
    from code2vec_b200.similarity import _fp32_matmul
    _legacy_allow(on)
    with _fp32_matmul():
        assert not CF.torch_matmul_tf32()
    assert torch.backends.cuda.matmul.allow_tf32 is on


def test_graphed_step_raises_when_the_switch_changes(torch_switch):
    m = Code2Vec(_Opt())
    step = GraphedTrainStep(m, torch.optim.Adam(m.parameters()), 4, 8)
    step.graph, step._frozen = object(), step._settings()        # as after a capture (no replay is reached below)
    _new_api("tf32")
    with pytest.raises(RuntimeError, match="TF32"):
        step(*_batch())


def test_graphed_predict_raises_when_the_switch_changes(torch_switch):
    m = Code2Vec(_Opt()).eval()
    _new_api("tf32")
    pred = GraphedPredict(m, 4, 8)
    pred.graph, pred._frozen = object(), pred._settings()
    _new_api("ieee")
    with pytest.raises(RuntimeError, match="TF32"):
        pred(*_batch()[:3])

"""CPU-side checks of the criterion options of the fused loss (c2v_loss_options and the c2v_*_opts entry points): the
symbols and their signatures, C2V_EINVAL with a message before any CUDA call for bad options, and the Python-side
TypeError / ValueError / GraphedTrainStep checks of Code2Vec.forward_loss(criterion=...)."""
import ctypes
import math

import pytest
import torch
import torch.nn as nn

from code2vec_b200 import _lib
from code2vec_b200 import functional as CF
from code2vec_b200.graphs import GraphedTrainStep
from code2vec_b200.model import Code2Vec

V = ctypes.c_void_p
FAKE = V(0x1000)          # never dereferenced: every call below fails its argument checks first
B = 8


def _dims(H=128, C=64):
    return _lib.Dims(1000, 800, C, H, H, H, 0)


def _params():
    return _lib.Params(None, None, None, None, None, None, FAKE, None)


def _opts(weight=None, ii=-100, eps=0.0, reduction=_lib.REDUCTION_MEAN, row_grad=None):
    return _lib.LossOptions(weight, ii, eps, reduction, row_grad)


def test_symbols_and_signatures():
    lib = _lib.load()
    P = ctypes.POINTER
    for name in ("c2v_label_loss_opts_workspace_bytes", "c2v_label_loss_argmax_opts", "c2v_label_dlogits_opts",
                 "c2v_angular_loss_argmax_opts", "c2v_angular_dlogits_opts", "c2v_loss_argmax_opts"):
        assert hasattr(lib, name)
        assert P(_lib.LossOptions) in _lib.SYMBOLS[name][1] or name.endswith("workspace_bytes")
    assert [f[0] for f in _lib.LossOptions._fields_] == ["class_weight", "ignore_index", "label_smoothing", "reduction",
                                                         "row_grad"]
    assert ctypes.sizeof(_lib.LossOptions) == 32
    assert _lib.LossOptions.ignore_index.offset == 8 and _lib.LossOptions.row_grad.offset == 24
    d = _dims()
    base = lib.c2v_label_workspace_bytes(ctypes.byref(d), B)
    assert lib.c2v_label_loss_opts_workspace_bytes(ctypes.byref(d), B) > base
    assert lib.c2v_label_loss_opts_workspace_bytes(ctypes.byref(d), 0) == 0


BAD = {"smoothing < 0": dict(eps=-0.1), "smoothing > 1": dict(eps=1.5), "smoothing NaN": dict(eps=math.nan),
       "smoothing inf": dict(eps=math.inf), "reduction -1": dict(reduction=-1), "reduction 3": dict(reduction=3),
       "misaligned weight": dict(weight=V(0x1002))}


def _rc_msg(rc):
    return rc, _lib.load().c2v_last_error()


def _calls(o):
    """every entry point that takes options, with otherwise valid (fake) arguments -> {name: (rc, last error)}"""
    lib = _lib.load()
    d, p = _dims(), _params()
    ws = 1 << 40
    r = {}
    r["c2v_label_loss_argmax_opts"] = _rc_msg(lib.c2v_label_loss_argmax_opts(
        ctypes.byref(d), ctypes.byref(p), FAKE, FAKE, B, ctypes.byref(o), None, FAKE, FAKE, FAKE, None, None, FAKE, ws, 0, None))
    r["c2v_angular_loss_argmax_opts"] = _rc_msg(lib.c2v_angular_loss_argmax_opts(
        ctypes.byref(d), ctypes.byref(p), FAKE, FAKE, B, 0.5, 30.0, ctypes.byref(o), None, FAKE, FAKE, FAKE, None, None, FAKE,
        FAKE, ws, 0, None))
    r["c2v_label_dlogits_opts"] = _rc_msg(lib.c2v_label_dlogits_opts(
        ctypes.byref(d), ctypes.byref(p), FAKE, FAKE, FAKE, FAKE, B, ctypes.byref(o), 1.0, None, FAKE, FAKE, ws, 0, None))
    r["c2v_angular_dlogits_opts"] = _rc_msg(lib.c2v_angular_dlogits_opts(
        ctypes.byref(d), ctypes.byref(p), FAKE, FAKE, FAKE, FAKE, FAKE, B, 0.5, 30.0, ctypes.byref(o), 1.0, None, FAKE, FAKE,
        ws, 0, None))
    r["c2v_loss_argmax_opts"] = _rc_msg(lib.c2v_loss_argmax_opts(FAKE, FAKE, B, 64, ctypes.byref(o), FAKE, None, None, None,
                                                                 None))
    return r


@pytest.mark.parametrize("case", list(BAD))
def test_bad_options_are_rejected_before_any_cuda_call(case):
    for name, (rc, msg) in _calls(_opts(**BAD[case])).items():
        assert rc == _lib.C2V_EINVAL, (name, rc)
        assert name.encode() in msg, (name, msg)


def test_reduction_none_needs_row_grad_in_dlogits():
    lib = _lib.load()
    d, p = _dims(), _params()
    o = _opts(reduction=_lib.REDUCTION_NONE)
    rc = lib.c2v_label_dlogits_opts(ctypes.byref(d), ctypes.byref(p), FAKE, FAKE, FAKE, FAKE, B, ctypes.byref(o), 1.0, None,
                                    FAKE, FAKE, 1 << 40, 0, None)
    assert rc == _lib.C2V_EINVAL and b"row_grad" in lib.c2v_last_error()
    rc = lib.c2v_angular_dlogits_opts(ctypes.byref(d), ctypes.byref(p), FAKE, FAKE, FAKE, FAKE, FAKE, B, 0.5, 30.0,
                                      ctypes.byref(o), 1.0, None, FAKE, FAKE, 1 << 40, 0, None)
    assert rc == _lib.C2V_EINVAL and b"row_grad" in lib.c2v_last_error()


def test_coefficients_and_workspace_are_required():
    lib = _lib.load()
    d, p = _dims(), _params()
    o = _opts()
    rc = lib.c2v_label_loss_argmax_opts(ctypes.byref(d), ctypes.byref(p), FAKE, FAKE, B, ctypes.byref(o), None, FAKE, FAKE,
                                        None, None, None, FAKE, 1 << 40, 0, None)
    assert rc == _lib.C2V_EINVAL and b"coef" in lib.c2v_last_error()
    small = lib.c2v_label_workspace_bytes(ctypes.byref(d), B)          # enough without options, not with them
    rc = lib.c2v_label_loss_argmax_opts(ctypes.byref(d), ctypes.byref(p), FAKE, FAKE, B, ctypes.byref(o), None, FAKE, FAKE,
                                        FAKE, None, None, FAKE, small, 0, None)
    assert rc == _lib.C2V_EWORKSPACE
    rc = lib.c2v_label_dlogits_opts(ctypes.byref(d), ctypes.byref(p), FAKE, FAKE, FAKE, None, B, ctypes.byref(o), 1.0, None,
                                    FAKE, FAKE, 1 << 40, 0, None)
    assert rc == _lib.C2V_EINVAL


# ---- Python-side errors -------------------------------------------------------------------------------------------------
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


class _MyCE(nn.CrossEntropyLoss):
    pass


@pytest.mark.parametrize("crit", [nn.MSELoss(), nn.BCEWithLogitsLoss(), _MyCE(), nn.MultiMarginLoss(), "nll"])
def test_other_criterion_types_raise_type_error(crit):
    with pytest.raises(TypeError, match="criterion"):
        Code2Vec(_Opt()).forward_loss(*_batch(), criterion=crit)


@pytest.mark.parametrize("weight", [torch.ones(7, dtype=torch.float64), torch.ones(6), torch.ones(7, 1), torch.ones(8)])
def test_a_wrong_weight_raises_value_error(weight):
    for cls in (nn.NLLLoss, nn.CrossEntropyLoss):
        with pytest.raises(ValueError, match="weight"):
            Code2Vec(_Opt()).forward_loss(*_batch(), criterion=cls(weight=weight))


def test_loss_criterion_reads_the_settings():
    w = torch.rand(7)
    c = CF.LossCriterion(nn.CrossEntropyLoss(weight=w, ignore_index=3, reduction="sum", label_smoothing=0.25), 7, "cpu")
    assert (c.ignore_index, c.label_smoothing, c.reduction) == (3, 0.25, "sum") and c.weight is w
    c = CF.LossCriterion(nn.NLLLoss(reduction="none"), 7, "cpu")
    assert (c.weight, c.ignore_index, c.label_smoothing, c.reduction, c.loss_shape(5)) == (None, -100, 0.0, "none", (5,))


def _captured_step(crit):
    m = Code2Vec(_Opt())
    step = GraphedTrainStep(m, torch.optim.Adam(m.parameters()), 4, 8, criterion=crit)
    step.graph, step._frozen = object(), step._settings()        # as after a capture (no replay is reached below)
    return step


@pytest.mark.parametrize("change", ["ignore_index", "label_smoothing", "reduction", "weight", "weight shape", "type"])
def test_graphed_step_raises_when_the_criterion_changes(change):
    w = torch.rand(7)
    crit = nn.CrossEntropyLoss(weight=w, label_smoothing=0.1)
    step = _captured_step(crit)
    if change == "ignore_index":
        crit.ignore_index = 2
    elif change == "label_smoothing":
        crit.label_smoothing = 0.2
    elif change == "reduction":
        crit.reduction = "sum"
    elif change == "weight":
        crit.weight = torch.rand(7)
    elif change == "weight shape":
        crit.weight = w[:5]                       # same address, other shape
    else:
        step.criterion = nn.NLLLoss(weight=w)
    with pytest.raises(RuntimeError, match="criterion"):
        step(*_batch())


def test_graphed_step_allows_in_place_weight_updates():
    crit = nn.CrossEntropyLoss(weight=torch.rand(7), label_smoothing=0.1)
    step = _captured_step(crit)
    crit.weight.mul_(2.0)                         # the replays read the values: no new capture needed
    assert step._settings() == step._frozen

"""CPU-side checks of the sampled softmax (functional.SampledSoftmax, Code2Vec.forward_sampled_loss, ddp_step(sampler=)):
the sampler's validation and its CDF / log q against numpy, every new C entry point's argument errors -- returned
before any CUDA call --, and the errors of the model and ddp_step that come before any device work."""
import ctypes
import math
import types

import numpy as np
import pytest
import torch

from code2vec_b200 import _lib, distributed
from code2vec_b200 import functional as CF
from code2vec_b200.model import Code2Vec

V = ctypes.c_void_p
FAKE = V(0x1000)          # never dereferenced: every call below fails its argument checks first
BIG = 1 << 40


def _expect(rc, code, name):
    assert rc == code
    msg = _lib.load().c2v_last_error()
    assert msg and name.encode() in msg, msg


# ---- SampledSoftmax ---------------------------------------------------------------------------------------------------
SAMPLER_BAD = {
    "label_count 0": dict(label_count=0),
    "num_sampled 0": dict(num_sampled=0),
    "num_sampled 65537": dict(num_sampled=65537),
    "counts too short": dict(counts=np.ones(9)),
    "counts 2-D": dict(counts=np.ones((2, 5))),
    "counts with a zero": dict(counts=np.r_[np.ones(9), 0.0]),
    "counts negative": dict(counts=np.r_[np.ones(9), -1.0]),
    "counts NaN": dict(counts=np.r_[np.ones(9), np.nan]),
    "counts inf": dict(counts=np.r_[np.ones(9), np.inf]),
    "power 0": dict(power=0.0),
    "power negative": dict(power=-0.5),
    "power NaN": dict(power=float("nan")),
    "power inf": dict(power=float("inf")),
    "counts ** power overflows": dict(counts=np.full(10, 1e200), power=2.0),
}


@pytest.mark.parametrize("case", list(SAMPLER_BAD))
def test_sampled_softmax_rejects_bad_arguments(case):
    kw = dict(label_count=10, num_sampled=4, counts=None, power=1.0)
    kw.update(SAMPLER_BAD[case])
    with pytest.raises(ValueError):
        CF.SampledSoftmax(**kw)


def test_sampled_softmax_bounds_are_accepted():
    for S in (1, 65536):
        assert CF.SampledSoftmax(3, S).num_sampled == S
    CF.SampledSoftmax(1, 1)
    CF.SampledSoftmax(5, 2, counts=torch.arange(1, 6), power=0.75)       # a tensor of counts


@pytest.mark.parametrize("C,power,kind", [(1, 1.0, "uniform"), (50, 0.75, "zipf"), (50, 1.0, "zipf"),
                                          (1000, 1.0, "uniform"), (195299, 0.75, "zipf"), (7, 0.5, "random")])
def test_cdf_and_log_q_match_numpy(C, power, kind):
    rng = np.random.default_rng(C)
    counts = None if kind == "uniform" else (
        1.0 / np.arange(1, C + 1) * 1e6 if kind == "zipf" else rng.integers(1, 100, C).astype(np.float64))
    s = CF.SampledSoftmax(C, 8, counts=counts, power=power)
    w = np.ones(C) if counts is None else counts.astype(np.float64) ** power
    q = w / w.sum()
    assert s.cdf_host.dtype == np.float64 and s.log_q_host.dtype == np.float64
    assert s.cdf_host[-1] == 1.0
    assert np.all(np.diff(s.cdf_host) > 0) if C > 1 else True
    np.testing.assert_allclose(s.cdf_host, np.cumsum(q), rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(s.log_q_host, np.log(q), rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(np.exp(s.log_q_host).sum(), 1.0, rtol=1e-12)


# ---- C entry points ---------------------------------------------------------------------------------------------------
def _cand(cdf=FAKE, C=100, S=8, key=1, key_dev=None, out=FAKE):
    return _lib.load().c2v_sampled_candidates(cdf, C, S, key, key_dev, out, None)


CAND_BAD = {"C<1": dict(C=0), "S<1": dict(S=0), "S>65536": dict(S=65537), "cdf": dict(cdf=None),
            "candidates": dict(out=None), "misaligned cdf": dict(cdf=V(0x1004)),
            "misaligned candidates": dict(out=V(0x1004)), "misaligned key_device": dict(key_dev=V(0x1004))}


@pytest.mark.parametrize("case", list(CAND_BAD))
def test_sampled_candidates_rejects_bad_arguments(case):
    _expect(_cand(**CAND_BAD[case]), _lib.C2V_EINVAL, "c2v_sampled_candidates")


def _gather(w=FAKE, b=FAKE, lq=FAKE, C=100, H=64, cand=FAKE, S=8, lab=FAKE, B=4, wh=FAKE, bh=FAKE, ids=FAKE):
    return _lib.load().c2v_sampled_gather(w, b, lq, C, H, cand, S, lab, B, wh, bh, ids, None)


GATHER_BAD = {"C<1": dict(C=0), "H<1": dict(H=0), "S<1": dict(S=0), "S>65536": dict(S=65537), "B<1": dict(B=0),
              "S+B>=2^31": dict(B=(1 << 31) - 1), "output_weight": dict(w=None), "output_bias": dict(b=None),
              "log_q": dict(lq=None), "candidates": dict(cand=None), "label": dict(lab=None), "w_hat": dict(wh=None),
              "b_hat": dict(bh=None), "ids": dict(ids=None), "misaligned output_weight": dict(w=V(0x1002)),
              "misaligned log_q": dict(lq=V(0x1004)), "misaligned candidates": dict(cand=V(0x1004)),
              "misaligned label": dict(lab=V(0x1004)), "misaligned w_hat": dict(wh=V(0x1001)),
              "misaligned ids": dict(ids=V(0x1004))}


@pytest.mark.parametrize("case", list(GATHER_BAD))
def test_sampled_gather_rejects_bad_arguments(case):
    _expect(_gather(**GATHER_BAD[case]), _lib.C2V_EINVAL, "c2v_sampled_gather")


def _loss(lg=FAKE, ids=FAKE, S=8, B=4, lse=FAKE, loss=FAKE):
    return _lib.load().c2v_sampled_loss(lg, ids, S, B, lse, loss, None)


LOSS_BAD = {"S<1": dict(S=0), "S>65536": dict(S=65537), "B<1": dict(B=0), "logits": dict(lg=None), "ids": dict(ids=None),
            "lse": dict(lse=None), "loss": dict(loss=None), "misaligned logits": dict(lg=V(0x1002)),
            "misaligned ids": dict(ids=V(0x1004)), "misaligned lse": dict(lse=V(0x1001))}


@pytest.mark.parametrize("case", list(LOSS_BAD))
def test_sampled_loss_rejects_bad_arguments(case):
    _expect(_loss(**LOSS_BAD[case]), _lib.C2V_EINVAL, "c2v_sampled_loss")


def _dlogits(lg=FAKE, ids=FAKE, lse=FAKE, S=8, B=4, scale=0.25, sd=None):
    return _lib.load().c2v_sampled_dlogits(lg, ids, lse, S, B, scale, sd, None)


DLOGITS_BAD = {"S<1": dict(S=0), "S>65536": dict(S=65537), "B<1": dict(B=0), "B>65535": dict(B=65536),
               "logits": dict(lg=None), "ids": dict(ids=None), "lse": dict(lse=None),
               "misaligned logits": dict(lg=V(0x1002)), "misaligned ids": dict(ids=V(0x1004)),
               "misaligned scale_device": dict(sd=V(0x1001))}


@pytest.mark.parametrize("case", list(DLOGITS_BAD))
def test_sampled_dlogits_rejects_bad_arguments(case):
    _expect(_dlogits(**DLOGITS_BAD[case]), _lib.C2V_EINVAL, "c2v_sampled_dlogits")


def _scatter(ids=FAKE, n=16, rows=FAKE, bias=FAKE, H=64, C=100, dst=FAKE, dst_b=FAKE, ws=FAKE, ws_bytes=BIG):
    return _lib.load().c2v_scatter_rows_add(ids, n, rows, bias, H, C, dst, dst_b, ws, ws_bytes, None)


SCATTER_BAD = {"n<1": dict(n=0), "n>=2^31": dict(n=1 << 31), "C<1": dict(C=0), "C>=2^31": dict(C=1 << 31),
               "H<1": dict(H=0), "ids": dict(ids=None), "workspace": dict(ws=None), "rows without dst": dict(dst=None),
               "dst without rows": dict(rows=None), "bias without dst_bias": dict(dst_b=None),
               "dst_bias without bias": dict(bias=None), "neither pair": dict(rows=None, dst=None, bias=None, dst_b=None),
               "misaligned ids": dict(ids=V(0x1004)), "misaligned rows": dict(rows=V(0x1002)),
               "misaligned dst": dict(dst=V(0x1001)), "misaligned workspace": dict(ws=V(0x1008))}


@pytest.mark.parametrize("case", list(SCATTER_BAD))
def test_scatter_rows_add_rejects_bad_arguments(case):
    _expect(_scatter(**SCATTER_BAD[case]), _lib.C2V_EINVAL, "c2v_scatter_rows_add")


def test_scatter_rows_add_workspace():
    lib = _lib.load()
    assert lib.c2v_scatter_rows_add_workspace_bytes(0) == 0
    assert lib.c2v_scatter_rows_add_workspace_bytes(1 << 31) == 0
    for n in (1, 1000, 9216, 65536 + 2048):
        # a double buffer of u64 keys, then one byte per key plus 1 MB for the radix sort
        assert lib.c2v_scatter_rows_add_workspace_bytes(n) == (16 * n + 1023) // 1024 * 1024 + n + (1 << 20)
    need = lib.c2v_scatter_rows_add_workspace_bytes(16)
    _expect(_scatter(ws_bytes=need - 1), _lib.C2V_EWORKSPACE, "c2v_scatter_rows_add")
    # one pair is enough
    _expect(_scatter(rows=None, dst=None, ws_bytes=need - 1), _lib.C2V_EWORKSPACE, "c2v_scatter_rows_add")


# ---- model and ddp_step -----------------------------------------------------------------------------------------------
def _option(C=10, angular=False):
    o = types.SimpleNamespace()
    o.terminal_count, o.path_count, o.label_count = 20, 20, C
    o.terminal_embed_size, o.path_embed_size, o.encode_size = 8, 8, 8
    o.dropout_prob = 0.0
    o.angular_margin_loss, o.angular_margin, o.inverse_temp = angular, 0.5, 30.0
    o.device = torch.device("cpu")
    return o


def _batch():
    z = torch.ones(2, 3, dtype=torch.int64)
    return z, z, z, torch.zeros(2, dtype=torch.int64)


def test_forward_sampled_loss_rejects_the_angular_head():
    m = Code2Vec(_option(angular=True))
    with pytest.raises(NotImplementedError):
        m.forward_sampled_loss(*_batch(), CF.SampledSoftmax(10, 4))


def test_forward_sampled_loss_rejects_a_sampler_of_another_vocabulary():
    m = Code2Vec(_option(C=10))
    with pytest.raises(ValueError):
        m.forward_sampled_loss(*_batch(), CF.SampledSoftmax(11, 4))
    with pytest.raises(TypeError):
        m.forward_sampled_loss(*_batch(), sampler=None)


def test_forward_sampled_loss_has_no_cpu_fallback():
    m = Code2Vec(_option(C=10))
    with pytest.raises(_lib.C2VError, match="CUDA"):
        m.forward_sampled_loss(*_batch(), CF.SampledSoftmax(10, 4))


@pytest.mark.parametrize("kw", [dict(loss_fn=torch.nn.functional.cross_entropy),
                                dict(loss_fn=None, criterion=torch.nn.CrossEntropyLoss())])
def test_ddp_step_rejects_a_sampler_with_another_loss(kw):
    m = Code2Vec(_option(C=10))
    loss_fn = kw.pop("loss_fn")
    with pytest.raises(ValueError, match="sampler"):
        distributed.ddp_step(m, None, None, *_batch(), loss_fn, sampler=CF.SampledSoftmax(10, 4), **kw)


def test_sample_has_no_cpu_fallback():
    with pytest.raises(_lib.C2VError, match="CUDA"):
        CF.SampledSoftmax(10, 4).sample(torch.zeros(1, dtype=torch.int64))
    assert math.isfinite(CF.SampledSoftmax(10, 4).log_q_host[0])

"""-m gpu: top-k prediction fused into the tensor-core label GEMM -- c2v_label_topk / c2v_angular_topk and
Code2Vec.predict_topk -- against torch.sort(descending=True, stable=True) of the logits c2v_label_logits writes (plain
head: the same numbers, so exact), fp64 restatements of the angular head without its margin, and the fallbacks."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden
from gpu_util import cuda, model_from_golden, random_batch, random_params
from code2vec_b200 import _lib
from code2vec_b200 import functional as CF
from code2vec_b200.model import Code2Vec

pytestmark = pytest.mark.gpu

KS = (1, 5, 10, _lib.TOPK_MAX)
S = 30.0

# the shapes of test_label_logits_tcgen05_vs_ffma_vs_oracle and of test_angular_loss_gpu.GRID, then the top11 label count
SHAPES = [(1, 5, 128), (37, 77, 128), (130, 1000, 128), (1024, 8192, 128), (64, 300, 64), (9, 50, 100), (200, 2279, 100),
          (33, 70, 36), (5, 40, 130), (130, 1000, 256), (40, 300, 200), (7, 11, 128), (64, 4097, 100), (33, 260, 256),
          (5, 3, 4), (1024, 19531, 128), (1024, 195299, 100)]


def _dims(C, H):
    return CF.make_dims(10, 10, C, H, H, H)


def _ks(C):
    return sorted({min(k, C) for k in KS})


def _check_plain(dims, params, cv, logits, k):
    B, C = logits.shape
    ref = torch.sort(logits, dim=1, descending=True, stable=True).indices[:, :k]
    idx, val, prob = CF.label_topk(dims, params, cv, k)
    assert idx.dtype == torch.int64 and idx.shape == (B, k) and val.shape == (B, k) and prob.shape == (B, k)
    assert torch.equal(idx, ref), (idx != ref).nonzero()[:5]
    assert torch.equal(val, logits.gather(1, idx))
    lsm = F.log_softmax(logits.double(), 1)
    lse = torch.logsumexp(logits.double(), 1)
    err = (prob.double().log() - lsm.gather(1, idx)).abs().max().item()
    assert err <= 2e-5 * max(1.0, lse.abs().max().item()), err
    idx2, val2, none = CF.label_topk(dims, params, cv, k, want_probs=False)
    assert none is None and torch.equal(idx2, idx) and torch.equal(val2, val)
    if k == 1:
        _, am, mx = CF.label_logits_argmax(dims, params, cv, want_logits=False)       # what predict() returns
        assert torch.equal(idx[:, 0], am) and torch.equal(val[:, 0], mx)


@pytest.mark.parametrize("B,C,H", SHAPES)
def test_plain_topk_is_the_stable_sort_of_the_tensor_core_logits(B, C, H):
    rng = np.random.default_rng(B * 31 + C)
    cv = cuda(np.tanh(rng.standard_normal((B, H))).astype(np.float32))
    w = (rng.standard_normal((C, H)) * 0.7).astype(np.float32)
    bias = (0.3 * rng.standard_normal(C)).astype(np.float32)
    dims, params = _dims(C, H), CF.make_params(None, None, None, None, None, None, cuda(w), cuda(bias))
    if H % 4 or H > 256:
        assert not CF.label_topk_supported(dims, B, 1)
        with pytest.raises(NotImplementedError):
            CF.label_topk(dims, params, cv, 1)
        return
    logits = CF.label_logits(dims, params, cv, algo=_lib.ALGO_TCGEN05)
    for k in _ks(C):
        _check_plain(dims, params, cv, logits, k)


@pytest.mark.parametrize("B,C", [(37, 77), (130, 1000), (1024, 19531), (9, 13)])
def test_ties_rank_the_lower_column_first(B, C):
    rng = np.random.default_rng(C)
    H = 128
    cvn = np.tanh(rng.standard_normal((B, H))).astype(np.float32)
    cvn[0] = 0.0                                               # every logit of row 0 is its bias
    cvn[B // 2] = 0.0
    w = (rng.standard_normal((C, H)) * 0.3).astype(np.float32)
    bias = np.zeros(C, np.float32)
    bias[C // 3:] = 0.25                                       # row 0: columns C // 3 .. C - 1 tie at the top
    for dst, src in ((C - 1, 1), (C // 2, 1), (5, 2), (6, 2), (C - 2, C // 3)):
        w[dst] = w[src]; bias[dst] = bias[src]                 # exact duplicates, the last column among them
    dims = _dims(C, H)
    params = CF.make_params(None, None, None, None, None, None, cuda(w), cuda(bias))
    cv = cuda(cvn)
    logits = CF.label_logits(dims, params, cv, algo=_lib.ALGO_TCGEN05)
    for k in _ks(C):
        _check_plain(dims, params, cv, logits, k)
    k = min(C, _lib.TOPK_MAX)
    idx = CF.label_topk(dims, params, cv, k)[0]
    top = [j for j in range(C) if bias[j] == 0.25][:k]              # the all-zero row: equal logits, in column order
    assert idx[0].tolist()[:len(top)] == top and idx[B // 2].tolist() == idx[0].tolist()


def _ang_case(rng, B, C, H, scale):
    W = (rng.uniform(-1, 1, (C, H)) / np.sqrt(H) * scale).astype(np.float32)
    cv = (rng.standard_normal((B, H)) * 0.5).astype(np.float32)
    return cv, W


def _ang_ref(cv, W):
    return S * F.linear(F.normalize(cuda(cv).double()), F.normalize(cuda(W).double()))


def _check_angular(idx, val, prob, ref, k):
    B = ref.shape[0]
    rs = torch.sort(ref, dim=1, descending=True).values[:, :k]
    assert (val.double() - rs).abs().max().item() <= 3e-6 * max(1.0, rs.abs().max().item())
    got = ref.gather(1, idx)
    assert bool((got >= rs[:, k - 1:k] - 1e-4).all())
    assert all(len(set(r)) == k for r in idx.tolist())
    if prob is not None:
        lse = torch.logsumexp(ref, 1)
        err = (prob.double().log() - (got - lse[:, None])).abs().max().item()
        assert err <= 2e-5 * max(1.0, lse.abs().max().item()), err
    assert idx.shape == (B, k)


@pytest.mark.parametrize("B,C,H,scale", [(7, 11, 128, 1.0), (130, 1000, 128, 8.0), (64, 4097, 100, 4.0), (33, 260, 256, 2.0),
                                         (1024, 8192, 128, 6.0), (5, 3, 4, 1.0), (1024, 195299, 100, 5.0)])
def test_angular_topk_matches_fp64_scaled_cosines(B, C, H, scale):
    rng = np.random.default_rng(B * 7 + C)
    cv, W = _ang_case(rng, B, C, H, scale)
    dims = _dims(C, H)
    params = CF.make_params(None, None, None, None, None, None, cuda(W), None)
    ref = _ang_ref(cv, W)
    for k in _ks(C):
        idx, val, prob = CF.angular_topk(dims, params, cuda(cv), k, S)
        _check_angular(idx, val, prob, ref, k)


# ---- Code2Vec.predict_topk ---------------------------------------------------------------------------------------------
def test_predict_topk_on_the_cfg2_golden():
    rec = load_golden("cfg2_small")
    m = model_from_golden(rec).eval()
    s, p, e = cuda(rec["starts"]), cuda(rec["paths"]), cuda(rec["ends"])
    out = torch.from_numpy(rec["outputs"]).double()
    srt = torch.sort(out, dim=1, descending=True, stable=True).values
    for k in _ks(out.shape[1]):
        idx, val, prob, cv, att = m.predict_topk(s, p, e, k=k)
        got = out.gather(1, idx.cpu())
        assert (val.cpu().double() - srt[:, :k]).abs().max().item() <= 1e-4
        assert bool((got >= srt[:, k - 1:k] - 1e-4).all())
        assert abs(prob.sum(1).max().item()) <= 1.0 + 1e-5
        assert np.abs(cv.cpu().numpy() - rec["code_vector"]).max() <= 2e-5
    am, mx, _, _ = m.predict(s, p, e)
    idx, val = m.predict_topk(s, p, e, k=1, probs=False)[:2]
    assert torch.equal(idx[:, 0], am) and torch.equal(val[:, 0], mx)
    assert np.array_equal(idx[:, 0].cpu().numpy(), rec["outputs"].argmax(1))


def test_predict_topk_on_the_angular_golden():
    rec = load_golden("angular")
    m = model_from_golden(rec).eval()
    s, p, e = cuda(rec["starts"]), cuda(rec["paths"]), cuda(rec["ends"])
    with pytest.raises(NotImplementedError):
        m.predict(s, p, e)                                    # unchanged: the margin needs the label
    W = rec["params"]["output_linear"]
    for k in _ks(W.shape[0]):
        idx, val, prob, cv, att = m.predict_topk(s, p, e, k=k)
        ref = m.option.inverse_temp * F.linear(F.normalize(cv.double()), F.normalize(cuda(W).double()))
        _check_angular(idx, val, prob, ref, k)


def _model(rng, T, P, C, E, H, angular=False, algo="auto"):
    opt = types.SimpleNamespace(terminal_count=T, path_count=P, label_count=C, terminal_embed_size=E, path_embed_size=E,
                                encode_size=H, dropout_prob=0.0, angular_margin_loss=angular, angular_margin=0.5,
                                inverse_temp=S, device=torch.device("cuda:0"))
    prm = random_params(rng, T, P, C, E, E, H)
    if angular:
        prm["output_linear"] = prm.pop("output_linear.weight")
        del prm["output_linear.bias"]
    m = Code2Vec(opt, algo=algo)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in prm.items()}, strict=True)
    return m.to("cuda:0").eval()


@pytest.mark.parametrize("angular", [False, True])
def test_predict_topk_cuts_large_batches_into_chunks(angular):
    rng = np.random.default_rng(4)
    T, P, C, E, H, B, L = 300, 200, 500, 128, 128, 2049, 20
    m = _model(rng, T, P, C, E, H, angular)
    s, p, e, _ = (cuda(x) for x in random_batch(rng, B, L, T, P, C))
    idx, val, prob, cv, _ = m.predict_topk(s, p, e, k=10)
    assert idx.shape == (B, 10) and prob.shape == (B, 10)
    dims = m._dims()
    if angular:
        params = CF.make_params(None, None, None, None, None, None, m.output_linear, None)
        for lo, hi in ((0, 2048), (2048, B)):
            i2, v2, p2 = CF.angular_topk(dims, params, cv[lo:hi], 10, S)
            assert torch.equal(idx[lo:hi], i2) and torch.equal(val[lo:hi], v2) and torch.equal(prob[lo:hi], p2)
    else:
        params = CF.make_params(None, None, None, None, None, None, m.output_linear.weight, m.output_linear.bias)
        logits = CF.label_logits(dims, params, cv, algo=_lib.ALGO_TCGEN05)
        assert torch.equal(idx, torch.sort(logits, dim=1, descending=True, stable=True).indices[:, :10])
        assert torch.equal(val, logits.gather(1, idx))


@pytest.mark.parametrize("angular", [False, True])
@pytest.mark.parametrize("case", ["ffma", "odd_encode", "k_above_max"])
def test_predict_topk_fallbacks_rank_like_the_fused_path(angular, case):
    rng = np.random.default_rng(12)
    T, P, C, L, B = 300, 200, 700, 20, 96
    E, H, algo = (30, 30, "auto") if case == "odd_encode" else (128, 128, "ffma" if case == "ffma" else "auto")
    m = _model(rng, T, P, C, E, H, angular, algo)
    s, p, e, _ = (cuda(x) for x in random_batch(rng, B, L, T, P, C))
    k = _lib.TOPK_MAX + 4 if case == "k_above_max" else 10
    idx, val, prob, cv, _ = m.predict_topk(s, p, e, k=k)
    assert idx.shape == (B, k) and val.shape == (B, k) and prob.shape == (B, k)
    W = m.output_linear if angular else m.output_linear.weight
    if angular:
        ref = S * F.linear(F.normalize(cv.double()), F.normalize(W.double()))
    else:
        ref = cv.double() @ W.double().T + m.output_linear.bias.double()
    ref_idx = torch.sort(ref, dim=1, descending=True, stable=True).indices[:, :k]
    assert torch.equal(idx, ref_idx)                           # random data: no ties, no near-ties at 1e-6
    assert (val.double() - ref.gather(1, idx)).abs().max().item() <= 3e-6 * max(1.0, ref.abs().max().item())
    lse = torch.logsumexp(ref, 1)
    assert (prob.double().log() - (ref.gather(1, idx) - lse[:, None])).abs().max().item() <= 2e-5 * max(1.0, lse.abs().max().item())
    if case == "k_above_max":
        fused = m.predict_topk(s, p, e, k=_lib.TOPK_MAX)
        assert torch.equal(fused[0], idx[:, :_lib.TOPK_MAX])


def test_predict_topk_argument_errors_and_deferred_index_errors():
    rng = np.random.default_rng(2)
    T, P, C, E, H, B, L = 300, 200, 12, 128, 128, 16, 10
    m = _model(rng, T, P, C, E, H)
    s, p, e, _ = (cuda(x) for x in random_batch(rng, B, L, T, P, C))
    for k in (0, C + 1):
        with pytest.raises(ValueError):
            m.predict_topk(s, p, e, k=k)
    assert m.predict_topk(s, p, e, k=C)[0].shape == (B, C)
    bad = s.clone()
    bad[3, 0] = T + 5
    m.predict_topk(bad, p, e, k=3)                              # clamped to row 0 and counted
    torch.cuda.synchronize()
    with pytest.raises(IndexError):                             # raised by the next call, without a sync of its own
        m.predict_topk(s, p, e, k=3)
    m.predict_topk(s, p, e, k=3)


def test_predict_topk_never_writes_the_logits():
    rng = np.random.default_rng(8)
    T, P, C, E, H, B, L = 2000, 1500, 195299, 100, 100, 1024, 200
    m = _model(rng, T, P, C, E, H)
    s, p, e, _ = (cuda(x) for x in random_batch(rng, B, L, T, P, C))
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    idx = m.predict_topk(s, p, e, k=10)[0]
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < B * C * 4 // 2, peak
    # the module keeps reusing its W_out image across predict / predict_topk
    cache = m._lab_cache
    buf = cache.buf
    m.predict(s, p, e)
    idx2 = m.predict_topk(s, p, e, k=10)[0]
    assert cache.buf is buf and torch.equal(idx, idx2)

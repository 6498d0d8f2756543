"""-m gpu: torch's TF32 switch (torch.set_float32_matmul_precision("high"), torch.backends.cuda.matmul.fp32_precision =
"tf32") runs the library's tensor-core GEMMs in one pass (c2v_set_matmul_precision(C2V_MATMUL_TF32)).

  fp64 judge        in TF32 mode the training step (test_train_step_gpu's cases, both heads, encode sizes 100, 128 and 256)
                    and a subset of test_value_range_gpu's trained-range cases (train, train-dc, eval-tc with predict_topk,
                    eval-ffma; encode sizes 100, 128 and 256; padded and PackedBags, with and without a criterion) are
                    judged against fp64 with the plain-precision baseline being torch fp32 WITH TF32 on: per tensor max rho(kernel) <= max(FACTOR * max rho(torch TF32),
                    2^-20), or the entry of LOOSER
  kernels           a profiled training step and predict_topk launch the OnePass instantiation of every converted kernel
                    in TF32 mode and none in IEEE mode; dC and the top-k label GEMM run three passes in both
  default mode      IEEE, TF32, IEEE with the deterministic mode on: the first and third runs are bit-identical, the TF32
                    run differs
  fp32 contracts    CodeVectorIndex.search / pairs and the CUDA-core paths give bit-identical results in both modes; a host-buffer
                    session call follows the mode of the calling thread
  deterministic     deterministic + TF32: repeated runs are bit-identical; a graphed step matches the eager one; a graph
                    refuses a changed switch
  training          25 optimizer steps of the drop-in loop in both modes stay as close as torch's own GPU model in both

Every test sets the switch through the new API and restores torch.backends.cuda.matmul.fp32_precision and
torch.backends.fp32_precision in a finally (the tf32 context manager): the legacy getter (allow_tf32) that other test
files' fixtures read raises while a new-API setter has left a value other than "none".
"""
import contextlib
import ctypes
import json

import numpy as np
import pytest
import torch
import torch.nn as nn

import test_deterministic_gpu as tdg
import test_train_step_gpu as tts
import test_value_range_gpu as tvr
from code2vec_b200 import _lib
from code2vec_b200 import functional as CF
from code2vec_b200.distributed import ShardedFlatAdam, ddp_step
from code2vec_b200.graphs import GraphedTrainStep
from code2vec_b200.model import Code2Vec
from code2vec_b200.similarity import CodeVectorIndex

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


@contextlib.contextmanager
def tf32(on=True):
    saved = torch.backends.fp32_precision, torch.backends.cuda.matmul.fp32_precision
    torch.backends.cuda.matmul.fp32_precision = "tf32" if on else "ieee"
    try:
        yield
    finally:
        torch.backends.fp32_precision = saved[0]
        torch.backends.cuda.matmul.fp32_precision = saved[1]


# ---- fp64 judge ------------------------------------------------------------------------------------------------------
# Tensors that need more than FACTOR in TF32 mode, per case: the worst measured ratio max rho(kernel) / max rho(torch
# TF32) in brackets, on one H100 80GB HBM3 (700 W).  Every other tensor of every case stays below 8 (below 2 for most).
#  * cfg3-angular, margin branch: phi(cos) = cos cos m - sin sin m for cos > 0 and cos otherwise jumps by sin m = 0.48 at
#    cos = 0.  A bag whose target cosine lies within one-pass rounding of 0 takes the other branch than fp64: its target
#    logit moves by s sin m = 14, and with it that bag's loss term, d cv row and the embedding rows it feeds.  Whether a
#    bag lands there depends on the parameters after the first Adam step, which vary with the order of the gradient
#    atomics; two of three runs hit it at step 1 ([233] and [208] on the loss), one did not (worst ratio 4.1 then).
#    torch's TF32 model rounds differently and stayed on fp64's side in all three.
# The OnePass kernels keep fp16's 10 explicit mantissa bits, as TF32 does, but fp16's
# exponent range: an operand split per tile under ONE power-of-two scale (dX of the encode backward, G of the label
# backward) or not scaled at all (gathered embedding rows, code vectors) loses relative precision where its entries fall
# far below that scale (fp16 subnormals), where torch's TF32 keeps 10 bits of every entry -- cases such as
# test_value_range_gpu's "tables-2^-16" or "attention-2^3" are outside what this mode promises.
LOOSER_TRAIN = {"cfg3-angular": {"loss": 512.0,                       # [233]
                                 "dcv": 128.0,                        # [85]
                                 "terminal_embedding.weight": 128.0,  # [51]
                                 "path_embedding.weight": 128.0}}     # [52]
LOOSER_RANGE = {}

TRAIN_CASES = ["cfg2", "cfg3", "cfg4", "cfg3-angular"]


@pytest.mark.parametrize("case", TRAIN_CASES)
def test_tf32_training_step_matches_fp64(case, monkeypatch):
    """test_train_step_gpu's case (ddp_step + ShardedFlatAdam, dropout 0.25, fused loss) in TF32 mode"""
    monkeypatch.setattr(tts, "LOOSER", {case: LOOSER_TRAIN.get(case, {})})
    with tf32():
        report, failures = tts._run_case(case)
    print(f"\n[tf32 train-step {case}] " + json.dumps(report, default=float))
    assert not failures, "\n".join(failures)


def _run_train_variant(packed, criterion):
    """test_value_range_gpu._run_train on the PackedBags form of the batch (attention scattered back to [B, L]) and / or
    with a criterion (nn.CrossEntropyLoss(): the criterion-options kernels, the same loss as the plain fused one)"""
    def run(w, P, batch, angular=False, inverse_temp=30.0):
        m = tvr._model(w, P, angular=angular, inverse_temp=inverse_temp).train()
        s, p, e, lab = batch
        crit = nn.CrossEntropyLoss() if criterion else None
        if packed:
            keep = s > 0                                # (real contexts have indices >= 1 in these batches)
            off = np.concatenate([[0], np.cumsum(keep.sum(1).cpu().numpy())])
            bags = CF.PackedBags(s[keep], p[keep], e[keep], off, s.shape[1])
            loss, am, mx, cv, att = m.forward_loss(bags, None, None, lab, criterion=crit)
            full = torch.zeros(s.shape, dtype=torch.float32, device=s.device)
            full[keep] = att.detach()
        else:
            loss, am, mx, cv, full = m.forward_loss(s, p, e, lab, criterion=crit)
        return _finish(m, loss, am, mx, cv, full.detach())
    return run


def _finish(m, loss, am, mx, cv, full):
    out = {"loss": loss.detach().clone(), "pred_score": mx.clone(), "am": am.clone(), "cv": cv.detach().clone(), "att": full}
    cv.register_hook(lambda g: out.__setitem__("dcv", g.detach().clone()))
    loss.backward()
    out["grads"] = {n: q.grad.clone() for n, q in m.named_parameters()}
    torch.cuda.synchronize()
    return out


RANGE_CASES = ["tables-2^0", "tables-2^0-packed", "tables-2^0-criterion", "tables-2^-3-packed-criterion", "tables-2^-3",
               "tables-2^4", "tables-2^0-h100", "tables-2^0-h256", "ln-mean-8", "w_in-2^4", "w_out-2^-8", "attention-2^0",
               "tables-2^-9-cfg2", "ln-mean-64-cfg3"]


@pytest.mark.parametrize("case", RANGE_CASES)
def test_tf32_value_range(case, monkeypatch):
    """test_value_range_gpu's case in TF32 mode.  Its 1e-4 parity bar describes the default mode and is not applied."""
    packed, criterion = "-packed" in case, "-criterion" in case
    base = case.replace("-packed", "").replace("-criterion", "")
    monkeypatch.setattr(tvr, "LOOSER", {base: LOOSER_RANGE.get(case, {})})
    monkeypatch.setattr(tvr.Judge, "bar", lambda *a, **k: None)
    if packed or criterion:
        monkeypatch.setattr(tvr, "_run_train", _run_train_variant(packed, criterion))
        shape, modify, in_range, _ = tvr.CASES[base]
        monkeypatch.setitem(tvr.CASES, base, (shape, modify, in_range, ("train",)))
    with tf32():
        J = tvr._run_case(base, monkeypatch)
    print(f"\n[tf32 value-range {case}] " + json.dumps(J.report, default=float))
    assert not J.failures, "\n".join(J.failures)


# ---- the OnePass kernels run -----------------------------------------------------------------------------------------
CONVERTED = ("encode_wgmma_kernel", "backward_dw_tc_kernel", "label_gemm_v2_kernel", "label_dw_tc_kernel",
             "label_dcv_tc_kernel")
# three passes in both modes: dC (bound by its scatter) and the top-k label GEMM (bound by its epilogue)
KEPT = ("backward_dc_tc_kernel", "label_gemm_v2_kernel<false, true")


def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.key for e in prof.key_averages() if "c2v::" in e.key}


def test_one_pass_kernels_run_only_in_tf32_mode():
    opt = tdg._option(5000, 7000, 300, 128, 128, 128)
    m = tdg._model(opt)
    o = ShardedFlatAdam(m.parameters(), lr=0.01)
    b = tdg._batch(opt, 64, 50, seed=3)

    def work():
        ddp_step(m, o, None, *b, None)
        m.eval()
        m.predict_topk(*b[:3], k=10)
        m.train()
    seen = {}
    for on in (True, False, True):
        with tf32(on):
            work()                                   # warm-up: persistent workspaces, module loads
            seen[on] = _kernel_names(work)
    assert not any("c2v::OnePass" in n for n in seen[False]), seen[False]
    for k in CONVERTED + KEPT:
        assert any(k in n for n in seen[False]), f"{k}: not launched in IEEE mode"
    for n in seen[True]:
        if any(k in n for k in KEPT):
            assert "c2v::OnePass" not in n, f"{n}: one pass in TF32 mode"
        elif any(k + "<" in n for k in CONVERTED):
            assert "c2v::OnePass" in n, f"{n}: three passes in TF32 mode"
    for k in CONVERTED:
        assert any(k + "<" in n and "c2v::OnePass" in n for n in seen[True]), f"{k}: no OnePass instantiation in TF32 mode"
    for k in KEPT:
        assert any(k in n for n in seen[True]), f"{k}: not launched in TF32 mode"


# ---- the default mode is unchanged -----------------------------------------------------------------------------------
def _train_and_predict(opt, batch, kw=None):
    m = tdg._model(opt, **(kw or {}))
    torch.manual_seed(5)
    out = tdg._step_plain(m, batch, False)
    if not opt.angular_margin_loss:
        m.eval()
        am, mx, cv, att = m.predict(*batch[:3])
        out.update(pred=am.clone(), score=mx.clone(), pred_cv=cv.clone(), pred_att=att.clone())
    torch.cuda.synchronize()
    return out


def _equal(a, b):
    return a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)


@pytest.mark.parametrize("H", [100, 128, 256])
def test_ieee_tf32_ieee(H):
    opt = tdg._option(5000, 7000, 300, H, H, H)
    batch = tdg._batch(opt, 64 if H < 256 else 32, 50, seed=11)
    runs = []
    with tdg.deterministic():
        for on in (False, True, False):
            with tf32(on):
                runs.append(_train_and_predict(opt, batch))
                assert _lib.load().c2v_get_matmul_precision() == int(on)
    assert _equal(runs[0], runs[2]), [k for k in runs[0] if not torch.equal(runs[0][k], runs[2][k])]
    for k in ("loss", "cv", "pred_cv", "input_linear.weight", "output_linear.weight", "terminal_embedding.weight"):
        assert not torch.equal(runs[0][k], runs[1][k]), f"{k}: TF32 mode gave the IEEE bits"


# ---- what stays fp32 in both modes -----------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["ffma", "angular-ffma"])
def test_cuda_core_paths_are_identical_in_both_modes(case, monkeypatch):
    """algo="ffma" selects the encode forward and the label head; the encode backward's dC and dW run on the tensor cores
    whenever the shape allows (and follow the switch) unless C2V_BACKWARD_DC / _DW = ffma put them on the CUDA cores"""
    monkeypatch.setenv("C2V_BACKWARD_DC", "ffma")
    monkeypatch.setenv("C2V_BACKWARD_DW", "ffma")
    opt, B, L, kw, _ = tdg.CASES[case]
    batch = tdg._batch(opt, B, L, seed=11)
    runs = []
    with tdg.deterministic():
        for on in (False, True):
            with tf32(on):
                runs.append(_train_and_predict(opt, batch, kw))
    assert _equal(runs[0], runs[1]), [k for k in runs[0] if not torch.equal(runs[0][k], runs[1][k])]


def test_knn_is_identical_in_both_modes():
    g = torch.Generator(device=DEV).manual_seed(3)
    vec = torch.randn(20000, 128, generator=g, device=DEV)
    vec[100] = vec[7]                                 # exact ties
    vec[101] = vec[7] * 1.0000001                     # near ties
    q = vec[:300] + 0.01 * torch.randn(300, 128, generator=g, device=DEV)
    res = []
    for on in (False, True):
        with tf32(on):
            idx = CodeVectorIndex(vec)
            s_idx, s_val = idx.search(q, k=10)
            pairs = idx.pairs(0.3, rows=torch.arange(300, device=DEV))
            torch.cuda.synchronize()
            res.append([s_idx, s_val] + [t for t in pairs if isinstance(t, torch.Tensor)])
    assert len(res[0]) == len(res[1]) >= 3
    for a, b in zip(*res):
        assert torch.equal(a, b)


def _session_forward(m, s, p, e, lab):
    o = m.option
    B, L = s.shape
    dims = CF.make_dims(o.terminal_count, o.path_count, o.label_count, o.terminal_embed_size, o.path_embed_size,
                        o.encode_size)
    params = CF.make_params(m.terminal_embedding.weight.data, m.path_embedding.weight.data, m.input_linear.weight.data,
                            m.input_layer_norm.weight.data, m.input_layer_norm.bias.data, m.attention_parameter.data,
                            m.output_linear.weight.data, m.output_linear.bias.data)
    lib = _lib.load()
    sess = ctypes.c_void_p()
    _lib.check(lib.c2v_session_create(0, ctypes.byref(dims), B, L, ctypes.byref(sess)), "session_create")
    try:
        pin = lambda t: t.cpu().contiguous().pin_memory()
        hs, hp, he, hl = pin(s), pin(p), pin(e), pin(lab)
        cv = torch.empty((B, o.encode_size), dtype=torch.float32).pin_memory()
        att = torch.empty((B, L), dtype=torch.float32).pin_memory()
        pred = torch.empty((B,), dtype=torch.int64).pin_memory()
        score = torch.empty((B,), dtype=torch.float32).pin_memory()
        P = lambda t: ctypes.c_void_p(t.data_ptr())
        rc = lib.c2v_forward_host(sess, ctypes.byref(params), P(hs), P(hp), P(he), P(hl), B, None, P(cv), P(att), P(pred),
                                  P(score), _lib.ALGO_AUTO)
        _lib.check(rc, "c2v_forward_host")
        return cv.to(DEV), pred.to(DEV)
    finally:
        lib.c2v_session_destroy(sess)


def test_session_call_follows_the_thread_mode():
    opt = tdg._option(5000, 7000, 300, 128, 128, 128)
    m = tdg._model(opt).eval()
    batch = tdg._batch(opt, 64, 50, seed=4)
    got = {}
    for on in (False, True):
        with tf32(on):
            am, _, cv, _ = m.predict(*batch[:3])            # sets this thread's library mode from the switch
            got[on] = (cv, am, *_session_forward(m, *batch))
    for on in (False, True):
        cv, am, s_cv, s_am = got[on]
        assert torch.equal(s_am, am)
        assert (s_cv - cv).abs().max().item() <= 1e-6 * cv.abs().max().item()
    d_mode = (got[True][0] - got[False][0]).abs().max().item()
    assert d_mode > 0
    assert (got[True][2] - got[True][0]).abs().max().item() < 0.1 * d_mode


# ---- deterministic + TF32, graphs ------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["tc-100", "tc-128", "tc-256", "packed", "angular", "ddp-fused"])
def test_deterministic_tf32_runs_are_bit_identical(case):
    junk = []
    with tf32():
        runs = [tdg._one_run(case, junk) for _ in range(2)]
        assert _lib.load().c2v_get_matmul_precision() == _lib.MATMUL_TF32
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), f"{case}: {k} differs between runs"


def test_graphed_tf32_step_matches_eager():
    with tf32():
        tdg.test_eager_steps_and_graph_replays_agree()


def test_graph_refuses_a_changed_switch():
    opt = tdg._option(5000, 7000, 300, 128, 128, 128)
    B, L = 32, 20
    m = tdg._model(opt)
    m.use_device_rng(seed=5)
    o = ShardedFlatAdam(m.parameters(), lr=0.01, capturable=True)
    step = GraphedTrainStep(m, o, B, L)
    b = tdg._batch(opt, B, L, seed=1)
    with tf32():
        for _ in range(3):                           # warm-up, warm-up, capture
            step(*b)
        step(*b)                                     # a replay in the captured mode
    with pytest.raises(RuntimeError, match="TF32"):
        step(*b)


# ---- training --------------------------------------------------------------------------------------------------------
class _Torch(nn.Module):
    """the same model in plain torch on the GPU (oracle.torch_forward), for torch's own TF32 on / off difference"""

    def __init__(self, params):
        super().__init__()
        self.p = nn.ParameterDict({k.replace(".", "__"): nn.Parameter(v.clone()) for k, v in params.items()})

    def forward(self, s, p, e, lab):
        from oracle import oracle
        P = {k.replace("__", "."): v for k, v in self.p.items()}
        out, _, _ = oracle.torch_forward(P, s, p, e, lab, dropmask=torch.ones((), device=s.device))
        return out


def _loss_curve(params, batches, use_torch, steps):
    if use_torch:
        m = _Torch(params).to(DEV)
    else:
        opt = tdg._option(3000, 2000, 97, 128, 128, 128, dropout=0.0)
        m = Code2Vec(opt)
        m.load_state_dict(params)
        m = m.to(DEV).train()
    o = torch.optim.Adam(m.parameters(), lr=0.01)
    crit = nn.NLLLoss()
    losses = []
    for i in range(steps):
        s, p, e, lab = batches[i % len(batches)]
        o.zero_grad()
        out = m(s, p, e, lab) if use_torch else m(s, p, e, lab)[0]
        loss = crit(torch.log_softmax(out, dim=1), lab)
        loss.backward()
        o.step()
        losses.append(loss.item())
    return np.array(losses)


def test_training_loss_curves():
    """25 Adam steps of the drop-in loop (forward, log_softmax + NLLLoss, backward, torch.optim.Adam) in both modes: at
    every step |library TF32 - library IEEE| <= 4 |torch TF32 - torch IEEE| + 1e-4 (1 + |loss|)"""
    torch.manual_seed(0)
    ref = Code2Vec(tdg._option(3000, 2000, 97, 128, 128, 128, dropout=0.0))
    params = {k: v.detach().to(DEV) for k, v in ref.state_dict().items()}
    opt = tdg._option(3000, 2000, 97, 128, 128, 128)
    batches = [tdg._batch(opt, 128, 40, seed=100 + i) for i in range(5)]
    curves = {}
    for use_torch in (False, True):
        for on in (False, True):
            with tf32(on):
                curves[use_torch, on] = _loss_curve(params, batches, use_torch, 25)
    d_lib = np.abs(curves[False, True] - curves[False, False])
    d_torch = np.abs(curves[True, True] - curves[True, False])
    print(f"\n[tf32 training] library |dloss| max {d_lib.max():.3g}, torch |dloss| max {d_torch.max():.3g}; "
          f"final losses library {curves[False, False][-1]:.5f} / {curves[False, True][-1]:.5f}, "
          f"torch {curves[True, False][-1]:.5f} / {curves[True, True][-1]:.5f}")
    bound = 4.0 * d_torch + 1e-4 * (1.0 + np.abs(curves[False, False]))
    assert (d_lib <= bound).all(), list(zip(d_lib.round(6), bound.round(6)))
    assert curves[False, True][-1] < curves[False, True][0]              # it trains

"""-m gpu: deterministic mode and sparse embedding gradients across the shape envelope, against fp64, element by element.

The case table is tests/mode_envelope.py.  Each training case runs in its modes (det, sparse, det+sparse, and the default
mode where the shape is new), with the helpers of test_shape_envelope_gpu.py and test_wide_encode_gpu.py:

  * fp64 judge: cv, att, loss, pred_score, d cv and every parameter gradient, with the bound the case has in the default
    mode (FACTOR = 8 or its LOOSER entry there).  Sparse gradients are made dense first; their indices must be
    torch.unique of the indices the batch passes (padding row 0 included in the padded layout);
  * dispatch: torch.profiler shows the stage paths of the case and the mode's own instantiations;
  * deterministic modes: two runs, with an allocation between them so that the buffers move, are bit-identical; det+sparse
    equals det bit for bit (the compact rows are the dense gradient's rows: the same keys are summed in the same order, only
    the destination row differs).

Label-head cases: every shape-envelope label case with the switch on (judged as in the default mode, and bit-identical to
it except d cv, which alone changes kernels), and the CUDA-core head where the default mode's sgemm splits K.  A model
switched off, on and off again gives the single-mode results.

Each case prints one JSON line per mode: per tensor the kernel's rho, fp32 torch's rho and their ratio.
"""
import json

import numpy as np
import pytest
import torch

import mode_envelope as ME
import shape_envelope as SE
import test_deterministic_gpu as tdg
import test_shape_envelope_gpu as env
import test_wide_encode_gpu as WE
from code2vec_b200 import functional as CF
from fp64_judge import rho
from test_shape_envelope_gpu import _fp32_without_tf32  # noqa: F401  (autouse: fp32 torch without TF32)

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
TABLES = {"shape": env.LOOSER, "wide": WE.LOOSER}
TABLES_KEYS = ("terminal_embedding.weight", "path_embedding.weight")
# Tensors of a case and mode that need more than the case's default-mode bound: measured on one H100 80GB HBM3 (700 W,
# 132 SMs), the measured ratio in brackets.  Keyed "<case> <mode>".
LOOSER = {}


def _judge(label, mode, c, P, batch, out, mask, monkeypatch):
    """test_wide_encode_gpu._judge with the case's default-mode bound, and this file's entry for the mode on top"""
    key = c["looser"][1] if c["looser"] else label
    bound = dict(TABLES[c["looser"][0]].get(key, {})) if c["looser"] else {}
    bound.update(LOOSER.get(f"{label} {mode}", {}))
    monkeypatch.setattr(env, "LOOSER", {key: bound})
    return WE._judge(key, c, P, batch, out, mask, angular=c["angular"])


def _run(c, P, batch, mode):
    """one training step (forward_loss + backward) in `mode` -> (outputs, dropout mask, kernel names)"""
    with pytest.MonkeyPatch.context() as mp:
        for k, v in c["env"].items():
            mp.setenv(k, v)
        if mode in (ME.SPARSE, ME.DET_SPARSE):
            build = env._model

            def sparse_model(*a):
                m = build(*a)
                m.terminal_embedding.sparse = m.path_embedding.sparse = True
                return m
            mp.setattr(env, "_model", sparse_model)
        with tdg.deterministic(mode in (ME.DET, ME.DET_SPARSE)):
            if c["angular"]:
                return WE._run_head(c, P, batch, DEV, angular=True)
            return env._run_train(c, P, batch, DEV)


def _same(a, b):
    if a.is_sparse:
        return b.is_sparse and torch.equal(a._indices(), b._indices()) and torch.equal(a._values(), b._values())
    return torch.equal(a, b)


def _differences(a, b, what):
    """every output of two runs, bit for bit"""
    out = [f"{what}: {k} differs" for k in ("loss", "am", "pred_score", "cv", "att", "dcv")
           if k in a and not torch.equal(a[k], b[k])]
    return out + [f"{what}: {k} differs" for k, g in a["grads"].items() if not _same(g, b["grads"][k])]


def _sparse_rows(c, batch):
    """the table rows the batch passes to the encode, as torch.unique of its indices"""
    s, p, e, _ = batch
    if c["layout"] == "packed":
        valid = s > 0
        s, p, e = s[valid], p[valid], e[valid]
    return {TABLES_KEYS[0]: torch.unique(torch.cat((s.reshape(-1), e.reshape(-1)))), TABLES_KEYS[1]: torch.unique(p)}


def _sparse_failures(c, batch, out, dense=True):
    """the compact gradients' indices; dense: make them dense for the judge"""
    f = []
    for k, rows in _sparse_rows(c, batch).items():
        g = out["grads"][k]
        if not (g.is_sparse and g.is_coalesced()):
            f.append(f"{k}: not a coalesced sparse gradient")
            g = g.to_sparse().coalesce()
        if not torch.equal(g._indices()[0], rows):
            f.append(f"{k}: indices are not torch.unique of the batch's indices")
        if dense or k != TABLES_KEYS[0]:
            out["grads"][k] = g.to_dense()
    return f


def _dispatch(c, mode, names, rerun):
    want, never = ME.mode_kernels(c, mode)
    # unstashed, backward_rows_kernel also runs next to the tensor-core dC: the dc stage is checked by the mode's dC
    # instantiation in `want` alone
    paths = {k: v for k, v in c["paths"].items() if not (k == "dc" and v == ME.TC and c["env"].get("C2V_NO_STASH") == "1")}

    def check(nm):
        f = env._dispatch_failures(nm, paths)
        f += [f"dispatch {mode}: {k} did not run" for k in want if not any(k in n for n in nm)]
        return f + [f"dispatch {mode}: {k} ran" for k in never if any(k in n for n in nm)]
    return WE._dispatch(names, check, rerun)


def _modes(label, c, P, batch, monkeypatch, compact=False):
    """every mode of a case: runs, dispatch, exact checks, the fp64 judge -> failures"""
    runs, junk, failures = {}, [], []
    for mode in c["modes"]:
        det = mode in (ME.DET, ME.DET_SPARSE)
        res = []
        for _ in range(2 if det else 1):
            junk.append(torch.empty(int(1 + 4096 * np.random.randint(1, 64)), device=DEV))   # move the next allocations
            res.append(_run(c, P, batch, mode))
        runs[mode] = res
    for mode, res in runs.items():
        out, mask, names = res[0]
        f = _dispatch(c, mode, set().union(*(r[2] for r in res)), lambda: _run(c, P, batch, mode)[2])
        if len(res) > 1:
            f += _differences(out, res[1][0], f"{mode}: two runs")
        if mode == ME.DET_SPARSE and ME.DET in runs:
            dense = runs[ME.DET][0][0]
            for k in TABLES_KEYS:
                g = out["grads"][k]
                if not torch.equal(g._values(), dense["grads"][k][g._indices()[0]]):
                    f.append(f"det+sparse: {k} values are not the det gradient's rows")
            f += _differences(dict(out, grads={k: g for k, g in out["grads"].items() if k not in TABLES_KEYS}),
                              dense, "det+sparse against det")
        Pj, bj = P, batch
        if mode in (ME.SPARSE, ME.DET_SPARSE):
            out = dict(out, grads=dict(out["grads"]))
            f += _sparse_failures(c, batch, out, dense=not compact)
        if compact:
            # the judge on the rows the batch touches: the terminal table and batch compacted by _compact_terminals (given
            # a zero [T, 1] stand-in for the gradient: a compact gradient has no other rows), the gradient's values
            g = out["grads"][TABLES_KEYS[0]]
            stand_in = {"grads": {TABLES_KEYS[0]: torch.zeros(c["T"], 1, device=DEV)}}
            Pj, bj, _ = env._compact_terminals(P, batch, stand_in)
            out["grads"][TABLES_KEYS[0]] = g._values()
        J = _judge(label, mode, c, Pj, bj, out, mask, monkeypatch)
        print(f"\n[mode-envelope {label} {mode}] " + json.dumps(J.report, default=float))
        failures += [f"{mode}: {x}" for x in J.failures + f]
    return failures


def _inputs(c):
    P = env._params(c, DEV)
    if c["hot"]:
        batch = tuple(torch.from_numpy(a).to(DEV) for a in ME.hot_batch(c))
    else:
        batch = env._batch(c, DEV)
    if c["angular"]:
        P["output_linear"] = P.pop("output_linear.weight")
        del P["output_linear.bias"]
    return P, batch


@pytest.mark.parametrize("case", list(ME.TRAIN))
def test_training_case(case, monkeypatch):
    c = ME.TRAIN[case]
    P, batch = _inputs(c)
    failures = _modes(case, c, P, batch, monkeypatch)
    assert not failures, "\n".join(failures)


def test_table_past_4gb():
    c = ME.TABLE_4GB
    need = c["T"] * c["Et"] * 4 + (1 << 30)          # the table (its gradient is compact), headroom
    free, _ = torch.cuda.mem_get_info(0)
    if free < need:
        pytest.skip(f"a terminal table past 4 GB needs ~{need / 2 ** 30:.1f} GiB free on the device ({free / 2 ** 30:.1f})")
    P, batch = _inputs(c)
    with pytest.MonkeyPatch.context() as mp:
        failures = _modes("table-past-4GB", c, P, batch, mp, compact=True)
    assert not failures, "\n".join(failures)


def test_mode_switch(monkeypatch):
    """one model stepped with the switch off, on and off: each step equals a fresh model's step in its mode (the
    deterministic one bit for bit, the default one's forward bit for bit and its gradients against fp64), so workspaces
    cached in one mode serve the other"""
    c = ME.TRAIN[ME.MODE_SWITCH]
    P, batch = _inputs(c)
    fresh = {on: _run(c, P, batch, ME.DET if on else ME.DEFAULT)[0] for on in (False, True)}
    m = env._model(c, P, DEV)

    def same_model(*a):
        m.zero_grad(set_to_none=True)
        return m
    monkeypatch.setattr(env, "_model", same_model)
    failures = []
    for i, on in enumerate((False, True, False)):
        out, mask, _ = _run(c, P, batch, ME.DET if on else ME.DEFAULT)
        if on:
            failures += _differences(out, fresh[True], f"step {i} (on)")
        else:
            failures += [f"step {i} (off): {k} differs" for k in ("loss", "am", "pred_score", "cv", "att")
                         if not torch.equal(out[k], fresh[False][k])]
            J = _judge(ME.MODE_SWITCH, "default", c, P, batch, out, mask, monkeypatch)
            failures += [f"step {i} (off): {x}" for x in J.failures]
    assert not failures, "\n".join(failures)


# ---- label head ---------------------------------------------------------------------------------------------------------
class _Deterministic:
    """the functional module with every library call made under torch.use_deterministic_algorithms(True); the torch
    references of the label-head test stay outside (torch raises there for cuBLAS and NLLLoss on CUDA)"""

    def __init__(self, mod):
        self._mod = mod

    def __getattr__(self, name):
        v = getattr(self._mod, name)
        if not callable(v) or isinstance(v, type):
            return v

        def call(*a, **k):
            with tdg.deterministic():
                return v(*a, **k)
        return call


def _label_outputs(dims, params, cv, lab, W, G_in):
    """the outputs of test_shape_envelope_gpu's label-head calls (plain head, its top-k, the angular head), by name"""
    B, C = cv.shape[0], dims.label_count
    o = env._run_plain(dims, params, cv, lab, W, G_in, CF.PrepCache())
    cache = CF.PrepCache()
    for k in SE.topk_ks(C):
        o[f"topk{k} idx"], o[f"topk{k} val"], _ = CF.label_topk(dims, params, cv, k, want_probs=False, cache=cache,
                                                                 weight=W)
    pa, cache = CF.make_params(w_out=W), CF.PrepCache()
    loss, lse, am, mx, inv, _ = CF.angular_loss(dims, pa, cv, lab, env.MARGIN, env.INV_TEMP, cache=cache, weight=W)
    g = CF.angular_dlogits(dims, pa, cv, lab, lse, inv, env.MARGIN, env.INV_TEMP, 1.0 / B, cache=cache, weight=W)
    dcv, dw = CF.angular_backward_ws(dims, pa, cv, g, inv, cache=cache, weight=W, absmax_ready=True)
    o.update({"angular loss": loss, "angular lse": lse, "angular am": am, "angular mx": mx, "angular G": g,
              "angular dw": dw, "angular dcv": dcv})
    for k in SE.topk_ks(C):
        o[f"angular topk{k} idx"], o[f"angular topk{k} val"], _ = CF.angular_topk(
            dims, pa, cv, k, env.INV_TEMP, want_probs=False, cache=cache, weight=W)
    return o


@pytest.mark.parametrize("case", list(SE.LABEL))
def test_label_head_case(case, monkeypatch):
    """test_shape_envelope_gpu's label-head case with the switch on around every library call (its fp64 judge, its
    dispatch and its tile orders); then the mode's own kernels ran, every output but d cv is bit-identical to the default
    mode's (d cv alone changes kernels), and d cv is bit-identical across runs"""
    with monkeypatch.context() as mp:
        mp.setattr(env, "CF", _Deterministic(CF))
        env.test_label_head_case(case, mp)
    c = SE.LABEL[case]
    B, C, H = c["B"], c["C"], c["H"]
    W, bias, cv, lab = env._label_inputs(c, DEV)
    dims = CF.make_dims(10, 10, C, H, H, H)
    params = CF.make_params(w_out=W, b_out=bias)
    G_in = torch.randn(B, C, generator=torch.Generator(device=DEV).manual_seed(4), device=DEV) / B
    base = _label_outputs(dims, params, cv, lab, W, G_in)
    runs, names, junk = [], set(), []
    for _ in range(2):
        junk.append(torch.empty(int(1 + 4096 * np.random.randint(1, 64)), device=DEV))   # move the next allocations
        with tdg.deterministic():
            o, nm = env._kernel_names(lambda: _label_outputs(dims, params, cv, lab, W, G_in))
        runs.append(o)
        names |= nm
    failures = [f"dispatch: {k} did not run" for k in ME.label_det_kernels(H) if not any(k in n for n in names)]
    for k, v in base.items():
        if "dcv" in k:
            if not torch.equal(runs[0][k], runs[1][k]):
                failures.append(f"{k} differs between deterministic runs")
        elif not torch.equal(runs[0][k], v):
            failures.append(f"{k}: the deterministic mode's differs from the default mode's")
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("mode", [ME.DEFAULT, ME.DET])
def test_cuda_core_head(mode):
    """the CUDA-core label head (H = 260): logits, loss / arg-max, d logits and the label backward through sgemm, which
    splits K in the default mode (C >= 1024 over few output tiles) and must not in the deterministic one"""
    c = ME.FFMA_HEAD
    B, C, H = c["B"], c["C"], c["H"]
    W, bias, cv, lab = env._label_inputs(c, DEV)
    dims = CF.make_dims(10, 10, C, H, H, H)
    params = CF.make_params(w_out=W, b_out=bias)

    def run():
        with tdg.deterministic(mode == ME.DET):
            lg = CF.label_logits(dims, params, cv)
            loss, am, mx, G = CF.loss_argmax(lg, lab, want_grad=True)
            dcv, dw, db = CF.label_backward(dims, params, cv, G)
        return {"logits": lg, "loss": loss, "am": am, "mx": mx, "G": G, "dcv": dcv, "dw": dw, "db": db}
    o, names = env._kernel_names(run)
    J = env.Judge(f"ffma-head-{mode}")
    want = ["sgemm_kernel"] + (["loss_sum_kernel"] if mode == ME.DET else [])
    J.failures += [f"dispatch: {k} did not run" for k in want if not any(k in n for n in names)]
    J.failures += [f"dispatch: {n} ran" for n in names if "label_gemm_v2_kernel" in n or "label_dcv_tc_kernel" in n]
    if mode == ME.DET:
        o2 = run()
        J.failures += [f"{k} differs between deterministic runs" for k in o if not torch.equal(o[k], o2[k])]
    r64 = env._plain_ref(cv, W, bias, lab, torch.float64)
    r32 = env._plain_ref(cv, W, bias, lab, torch.float32)
    # S as in test_shape_envelope_gpu.test_label_head_case
    aW, acv = W.double().abs(), cv.double().abs()
    Sl = acv @ aW.t() + bias.double().abs()
    p64 = torch.softmax(r64["logits"], 1)
    pS = (p64 * Sl).sum(1, keepdim=True)
    oh = torch.zeros_like(p64).scatter_(1, lab[:, None], 1.0)
    SG = (p64 * (Sl + pS) + p64 + oh) / B
    S = {"logits": Sl, "loss": (r64["lse"].abs() + r64["logits"].gather(1, lab[:, None])[:, 0].abs()).mean(),
         "G": SG, "dcv": SG @ aW, "dw": SG.t() @ acv, "db": SG.sum(0)}
    J.argmax("argmax", o["am"], o["mx"], r64["logits"], Sl, rho(r32["logits"], r64["logits"], Sl, "", []))
    for k in S:
        J.full(k, o[k], r64[k], r32[k], S[k])
    print(f"\n[mode-envelope ffma-head {mode}] " + json.dumps(J.report, default=float))
    assert not J.failures, "\n".join(J.failures)

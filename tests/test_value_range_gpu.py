"""-m gpu: the kernels across the value ranges of trained weights, against fp64 (tests/fp64_judge.py).

Every GPU parity test builds its parameters at init scale.  A trained model does not stay there, and the tensor-core paths
are fp32-accurate only through the 3-pass fp16 hi/lo split, which keeps ~22 bits of a value only while its lo part is a
normal fp16.  Here one quantity at a time is scaled by a power of two (everything else at init scale) and every path the
case reaches is judged as test_train_step_gpu.py judges the training step:
  * train:    Code2Vec.forward_loss + backward (tensor-core encode with the stashed x, tensor-core dW / dC, fused loss and
              label backward): cv, att, loss, pred_score, d cv and every parameter gradient;
  * train-dc: the same with dC on the CUDA cores (C2V_BACKWARD_DC=ffma);
  * eval-tc / eval-ffma: predict_topk on the tensor cores / the CUDA cores: cv, att and the top-k values.
Per tensor, max rho(kernel) <= max(FACTOR * max rho(fp32 torch), 2^-20), or the case's entry in LOOSER.  Inside the
trained range (the third field of CASES) the forward outputs also meet the README's parity bar, 1e-4 * max(1, |fp64|).  Each case prints
one JSON line: per path and tensor, the kernel's rho, fp32 torch's rho and their ratio.
"""
import json
import math
import types

import pytest
import torch

from code2vec_b200 import functional as CF
from code2vec_b200.model import Code2Vec
from code2vec_b200.similarity import CodeVectorIndex
from fp64_judge import reference, rho, scales

pytestmark = pytest.mark.gpu

FACTOR, FLOOR, BAR = 8.0, 2.0 ** -20, 1e-4
TOPK = 5
BASE = dict(T=8192, P=8192, C=4096, Et=128, Ep=128, H=128, B=128, L=200)
SHAPES = {128: BASE, 100: dict(BASE, Et=100, Ep=100, H=100), 256: dict(BASE, Et=256, Ep=256, H=256, B=64),
          "cfg2": dict(T=360633, P=342846, C=8192, Et=128, Ep=128, H=128, B=1024, L=200),
          "cfg3": dict(T=360633, P=342846, C=195299, Et=100, Ep=100, H=100, B=1024, L=200)}

# Tensors that need more than FACTOR, per case (every path the case runs): measured on one H100 80GB HBM3 (700 W), the
# worst measured ratio max rho(kernel) / max rho(fp32 torch) over the paths in brackets.  Each is a precision deficit of
# the kernels as they are, not a tolerance for a wrong result; INTEGRATION.md, "Value range", lists the operands.
LOOSER = {
    # gathered embedding rows, unscaled fp16 hi/lo split (encode A producers, dW gather): below |v| ~ 2^-3 the lo part
    # falls into the fp16 subnormals and each entry keeps an absolute error of ~2^-25, so x loses relative accuracy as
    # the table RMS drops.  cv, att, the label GEMM (unscaled code vectors) and every gradient downstream inherit it.
    # (The CUDA-core encode's small excess at 2^-16 .. 2^-12 is the tanh term below.)
    "tables-2^-16": {"cv": 8192.0, "att": 256.0, "pred_score": 32.0, "attention_parameter": 512.0,   # [4077, 86, 16, 131]
                     "terminal_embedding.weight": 64.0, "path_embedding.weight": 64.0,               # [23, 28]
                     "input_linear.weight": 4096.0, "input_layer_norm.weight": 4096.0,               # [1211, 1348]
                     "output_linear.weight": 16384.0, "topk": 64.0},                                 # [7129, 18]
    "tables-2^-16-h100": {"cv": 2048.0, "att": 256.0, "topk": 128.0},                                # [653, 94, 33]
    "tables-2^-16-h256": {"cv": 8192.0, "att": 256.0, "topk": 64.0},                                 # [3359, 77, 22]
    "tables-2^-12": {"cv": 1024.0, "att": 256.0, "pred_score": 32.0, "attention_parameter": 512.0,   # [361, 66, 16, 143]
                     "terminal_embedding.weight": 64.0, "path_embedding.weight": 64.0,               # [26, 20]
                     "input_linear.weight": 256.0, "input_layer_norm.weight": 256.0,                 # [94, 124]
                     "output_linear.weight": 1024.0, "topk": 64.0},                                  # [286, 19]
    "tables-2^-12-h100": {"cv": 2048.0, "att": 256.0, "topk": 64.0},                                 # [738, 71, 19]
    "tables-2^-12-h256": {"cv": 1024.0, "att": 256.0, "topk": 64.0},                                 # [302, 73, 18]
    "tables-2^-9": {"cv": 256.0, "att": 64.0, "pred_score": 32.0, "terminal_embedding.weight": 32.0,  # [113, 24, 8.3, 15]
                    "path_embedding.weight": 64.0, "input_linear.weight": 32.0,                      # [23, 10]
                    "attention_parameter": 64.0, "input_layer_norm.weight": 32.0,                    # [30, 16]
                    "output_linear.weight": 32.0, "topk": 32.0},                                     # [16, 8.3]
    "tables-2^-9-h100": {"cv": 128.0, "att": 64.0, "topk": 32.0},                                    # [38, 28, 8.4]
    "tables-2^-9-h256": {"att": 64.0, "topk": 16.0},                                                 # [17, 6.4]
    "tables-2^-9-cfg2": {"cv": 64.0, "att": 64.0, "terminal_embedding.weight": 32.0,                 # [30, 21, 12]
                         "path_embedding.weight": 32.0, "output_linear.weight": 128.0, "topk": 32.0,  # [12, 43, 12]
                         "pred_score": 16.0},                                                        # [7.6]
    "tables-2^-9-cfg3": {"cv": 256.0, "att": 64.0, "output_linear.weight": 128.0, "topk": 32.0,      # [72, 25, 34, 8.3]
                         "pred_score": 16.0, "terminal_embedding.weight": 16.0,                      # [7.4, 7.2]
                         "path_embedding.weight": 16.0},                                             # [7.3]
    **{f"tables-2^{k}-h256": {"cv": 16.0} for k in (-6, -3, 0, 2, 4, 8, 12)},                       # [6.4 - 6.9]
    "tables-2^-6": {"output_linear.weight": 32.0},                                                   # [9.8]
    "tables-2^-6-h100": {"cv": 32.0},                                                                # [8.8]
    "terminal-2^-12": {"input_linear.weight": 512.0, "cv": 16.0},                                    # [133, 7.1]
    # tanh of a small argument: every encode (tensor and CUDA cores alike) evaluates tanh through exp, with an absolute
    # error of ~2^-24 where torch's tanh is accurate relative to its value.  With W_in x 2^-20 or gamma = 2^-10 the LN
    # output is ~2^-10 or below, and cv (and the W_out gradient, G^T cv) lose relative accuracy; |error| stays ~1e-7.
    "w_in-2^-20": {"cv": 2048.0, "output_linear.weight": 256.0, "attention_parameter": 16.0},        # [625, 101, 7.6]
    "gamma-2^-10": {"cv": 256.0, "output_linear.weight": 1024.0},                                    # [66, 307]
    "gamma-2^4": {"cv": 32.0},                                                                       # [13]
    "ln-mean-1-h256": {"cv": 32.0},                                                                  # [8.9]
    # dX fp16 split under ONE scale (backward_dw_tc_kernel / backward_dc_tc_kernel, "dX fp16 split" in
    # test_train_step_gpu.py): a concentrated softmax (attention x 2^3) spreads dX over many octaves within one batch,
    # and embedding rows fed only by low-attention contexts lose nearly all their bits.  At x 2^5 and above those
    # attentions underflow to exact zeros instead.
    "attention-2^3": {"terminal_embedding.weight": 131072.0, "path_embedding.weight": 131072.0},     # [47546, 52104]
    # G fp16 split under ONE scale (label backward, c2v_label_backward_tc.cu): with a wide softmax (large W_out, row norm
    # spread, bias +-16) the W_out rows of labels with tiny probabilities get G entries flushed to zero (rho 1).
    "w_out-rows-2^+-8": {"output_linear.weight": 512.0},                                             # [157]
    "bias-16": {"output_linear.weight": 512.0},                                                      # [154]
    "beta-0": {"output_linear.weight": 32.0},                                                        # [8.2]
    # near FACTOR, from run to run (the gradients accumulate with atomics, in no fixed order; worst over five runs):
    # tensors whose kernel rho sits at the 2^-20 floor while fp32 torch's is below it, and the wide encode's cv (the
    # scores of 256 terms of the forward's fp16-split x, as cfg4 in test_train_step_gpu.py)
    "beta-4": {"output_linear.bias": 16.0},                                                          # [7.0]
    "beta--4": {"output_linear.bias": 16.0, "input_layer_norm.bias": 16.0,                           # [6.4, 5.8]
                "attention_parameter": 64.0},                                                        # [35; 1 - 35 over runs]
    "w_out-2^8": {"dcv": 64.0, "terminal_embedding.weight": 64.0, "path_embedding.weight": 64.0,     # [21, 20, 21]
                  "input_linear.weight": 32.0, "output_linear.weight": 512.0,                        # [9.6, 157]
                  "output_linear.bias": 16.0},                                                       # [7.0]
    # functional label API: code vectors enter the label GEMM and LB1 unscaled (split_rows_kernel with no scale), so
    # below ~2^-3 their lo part is subnormal (logits, d W_out = G^T cv); above, G's single scale (d W_out) as above
    "label-api-2^-12": {"logits": 512.0, "dw": 8192.0},                                              # [186, 3940]
    "label-api-2^-8": {"logits": 32.0, "dw": 1024.0},                                                # [9.5, 266]
    "label-api-2^-4": {"dw": 64.0},                                                                  # [16]
    "label-api-2^4": {"dw": 256.0},                                                                  # [87]
    # angular head, inverse_temp 64: the softmax of s * cos spans ~e^128, G fp16 split as above
    "angular-2^+-0-s64": {"output_linear": 1024.0},                                                  # [361]
}


@pytest.fixture(autouse=True)
def _fp32_without_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved
    torch.cuda.empty_cache()


# ---- parameters and batches ------------------------------------------------------------------------------------------
def _params(w, dev, seed=1):
    """init scale, as bench.synth_params (model.py:18-42), with a small LN jitter and bias so that no term is exactly 0"""
    g = torch.Generator(device=dev).manual_seed(seed)
    D = 2 * w["Et"] + w["Ep"]
    r = lambda *s: torch.randn(*s, generator=g, device=dev)
    u = lambda bound, *s: (torch.rand(*s, generator=g, device=dev) * 2 - 1) * bound
    return {"terminal_embedding.weight": r(w["T"], w["Et"]), "path_embedding.weight": r(w["P"], w["Ep"]),
            "input_linear.weight": u(D ** -0.5, w["H"], D),
            "input_layer_norm.weight": 1.0 + 0.1 * r(w["H"]), "input_layer_norm.bias": 0.1 * r(w["H"]),
            "attention_parameter": r(w["H"]) * (2.0 / (w["H"] + 1)) ** 0.5,
            "output_linear.weight": u(w["H"] ** -0.5, w["C"], w["H"]), "output_linear.bias": 0.05 * r(w["C"])}


def _batch(w, dev, seed=2):
    """ragged bags with a zero-padded suffix (bag 0 full, bag 1 of one context), indices >= 1 (row 0 is the pad row);
    bag 2: one real context among pads; bag 3 alone gathers terminal row T-1 and path row P-1"""
    g = torch.Generator(device=dev).manual_seed(seed)
    B, L = w["B"], w["L"]
    s = torch.randint(1, w["T"] - 1, (B, L), generator=g, device=dev)
    p = torch.randint(1, w["P"] - 1, (B, L), generator=g, device=dev)
    e = torch.randint(1, w["T"] - 1, (B, L), generator=g, device=dev)
    n = torch.randint(1, L + 1, (B,), generator=g, device=dev)
    n[0], n[1] = L, 1
    valid = (torch.arange(L, device=dev)[None, :] < n[:, None]).long()
    s, p, e = s * valid, p * valid, e * valid
    s[2], p[2], e[2] = 0, 0, 0
    s[2, L // 3], p[2, L // 3], e[2, L // 3] = 5, 6, 7
    s[3, 0], p[3, 0] = w["T"] - 1, w["P"] - 1
    lab = torch.randint(0, w["C"], (B,), generator=g, device=dev)
    return s, p, e, lab


def _max_to_last_partial(P, batch):
    """bag 0 (full): move the context of the largest fp64 score to slot L-1, the last 16-row softmax partial of the bag"""
    s, p, e, lab = batch
    taps = {}
    from oracle import oracle
    P64 = {k: v.double() for k, v in P.items()}
    oracle.torch_forward(P64, s[:1], p[:1], e[:1], lab[:1], dropmask=torch.ones((), dtype=torch.float64, device=s.device),
                         taps=taps)
    j = int(taps["z"][0].argmax())
    for t in (s, p, e):
        t[0, j], t[0, -1] = t[0, -1].clone(), t[0, j].clone()


def _scale(key, f):
    def m(P, batch):
        P[key] = P[key] * f
    return m


def _tables(f, which=("terminal_embedding.weight", "path_embedding.weight")):
    def m(P, batch):
        for k in which:
            P[k] = P[k] * f
    return m


def _ln_mean(r):
    """W_h = u + v_h: a common row component u sized so that the LN input's RMS |mean| / std over contexts is r"""
    def m(P, batch):
        W = P["input_linear.weight"]
        g = torch.Generator(device=W.device).manual_seed(7)
        u = (torch.rand(W.shape[1], generator=g, device=W.device) * 2 - 1) * W.shape[1] ** -0.5
        P["input_linear.weight"] = W + r * u[None, :]
    return m


def _ln_affine(gamma=None, beta=None):
    def m(P, batch):
        if gamma is not None:
            P["input_layer_norm.weight"] = torch.full_like(P["input_layer_norm.weight"], gamma)
        if beta is not None:
            P["input_layer_norm.bias"] = torch.full_like(P["input_layer_norm.bias"], beta)
    return m


def _attention(f):
    def m(P, batch):
        P["attention_parameter"] = P["attention_parameter"] * f
        _max_to_last_partial(P, batch)
    return m


def _row_spread(octaves):
    def m(P, batch):
        W = P["output_linear.weight"]
        g = torch.Generator(device=W.device).manual_seed(8)
        P["output_linear.weight"] = W * torch.exp2(torch.randint(-octaves, octaves + 1, (W.shape[0], 1), generator=g,
                                                                 device=W.device).float())
    return m


def _bias(bound):
    def m(P, batch):
        b = P["output_linear.bias"]
        g = torch.Generator(device=b.device).manual_seed(9)
        P["output_linear.bias"] = (torch.rand(b.shape, generator=g, device=b.device) * 2 - 1) * bound
    return m


def _entry(key, value, row=1):
    def m(P, batch):
        P[key] = P[key].clone()
        P[key][row, 3] = value
    return m


def _zero_rows(P, batch):
    """row 0 all zero (the padding_idx habit) and a context of all-zero rows: x = 0, LN variance exactly 0"""
    s, p, e, _ = batch
    for k in ("terminal_embedding.weight", "path_embedding.weight"):
        P[k] = P[k].clone()
        P[k][0] = 0.0
        P[k][9] = 0.0
    s[4, :3] = 9
    p[4, :3] = torch.tensor([9, 0, 9])
    e[4, :3] = torch.tensor([9, 9, 0])


TRAIN = ("train", "train-dc", "eval-tc", "eval-ffma")
EVAL = ("eval-tc", "eval-ffma")
# name: (shape, modifier, inside the trained range, paths)
CASES = {}
for _s in (-16, -12, -9, -6, -3, 0, 2, 4, 8, 12):
    CASES[f"tables-2^{_s}"] = (128, _tables(2.0 ** _s), -9 <= _s <= 4, TRAIN)
    CASES[f"tables-2^{_s}-h100"] = (100, _tables(2.0 ** _s), -9 <= _s <= 4, EVAL)
    CASES[f"tables-2^{_s}-h256"] = (256, _tables(2.0 ** _s), -9 <= _s <= 4, EVAL)
CASES["tables-2^15"] = (128, _tables(2.0 ** 15), False, ("eval-ffma",))       # tensor cores: test_fp16_overflow
for _s in (-12, 4):
    CASES[f"terminal-2^{_s}"] = (128, _tables(2.0 ** _s, ("terminal_embedding.weight",)), True, TRAIN)
CASES["outlier-2^15"] = (128, _entry("terminal_embedding.weight", 2.0 ** 15), False, TRAIN)
CASES["zero-rows"] = (128, _zero_rows, True, TRAIN)
for _s in (-20, -4, 0, 4, 20):
    CASES[f"w_in-2^{_s}"] = (128, _scale("input_linear.weight", 2.0 ** _s), -4 <= _s <= 4, TRAIN)
for _r in (1, 8, 64, 512, 4096):
    CASES[f"ln-mean-{_r}"] = (128, _ln_mean(_r), _r <= 64, TRAIN)
    CASES[f"ln-mean-{_r}-h100"] = (100, _ln_mean(_r), _r <= 64, EVAL)
    CASES[f"ln-mean-{_r}-h256"] = (256, _ln_mean(_r), _r <= 64, EVAL)
for _gm in (-10, -4, 0, 4, 8):
    CASES[f"gamma-2^{_gm}"] = (128, _ln_affine(gamma=2.0 ** _gm), -4 <= _gm <= 4, TRAIN)
for _b in (0.0, 4.0, -4.0, 256.0, -256.0):
    CASES[f"beta-{_b:g}"] = (128, _ln_affine(beta=_b), abs(_b) <= 4, TRAIN)
for _s in (-10, 0, 3, 5, 10):
    CASES[f"attention-2^{_s}"] = (128, _attention(2.0 ** _s), _s <= 5, TRAIN)
for _s in (-20, -8, 0, 8, 20):
    CASES[f"w_out-2^{_s}"] = (128, _scale("output_linear.weight", 2.0 ** _s), -8 <= _s <= 8, TRAIN)
CASES["w_out-rows-2^+-8"] = (128, _row_spread(8), True, TRAIN)
CASES["bias-16"] = (128, _bias(16.0), True, TRAIN)
for _shape in ("cfg2", "cfg3"):
    CASES[f"tables-2^-9-{_shape}"] = (_shape, _tables(2.0 ** -9), True, TRAIN)
    CASES[f"ln-mean-64-{_shape}"] = (_shape, _ln_mean(64), True, TRAIN)


# ---- running the paths -----------------------------------------------------------------------------------------------
def _option(w, angular=False, inverse_temp=30.0):
    return types.SimpleNamespace(terminal_count=w["T"], path_count=w["P"], label_count=w["C"], terminal_embed_size=w["Et"],
                                 path_embed_size=w["Ep"], encode_size=w["H"], dropout_prob=0.0,
                                 angular_margin_loss=angular, angular_margin=0.5, inverse_temp=inverse_temp,
                                 device=torch.device("cuda:0"))


def _model(w, P, algo="auto", angular=False, inverse_temp=30.0):
    m = Code2Vec(_option(w, angular, inverse_temp), algo=algo)
    m.load_state_dict(P)
    return m.cuda()


def _run_train(w, P, batch, angular=False, inverse_temp=30.0):
    m = _model(w, P, angular=angular, inverse_temp=inverse_temp).train()
    s, p, e, lab = batch
    loss, am, mx, cv, att = m.forward_loss(s, p, e, lab)
    out = {"loss": loss.detach().clone(), "pred_score": mx.clone(), "am": am.clone(), "cv": cv.detach().clone(),
           "att": att.detach().clone()}
    cv.register_hook(lambda g: out.__setitem__("dcv", g.detach().clone()))
    loss.backward()
    out["grads"] = {n: q.grad.clone() for n, q in m.named_parameters()}
    torch.cuda.synchronize()
    return out


def _run_eval(w, P, batch, algo, angular=False, inverse_temp=30.0):
    m = _model(w, P, algo=algo, angular=angular, inverse_temp=inverse_temp).eval()
    s, p, e, _ = batch
    idx, val, _, cv, att = m.predict_topk(s, p, e, k=TOPK, probs=False)
    torch.cuda.synchronize()
    return {"cv": cv, "att": att, "topk_idx": idx, "topk": val}


class Judge:
    """collects per (path, tensor) the kernel's and fp32 torch's rho and the failures of one case"""

    def __init__(self, case, in_range):
        self.case, self.in_range = case, in_range
        self.report, self.failures = {}, []

    def note(self, path, name, rk, r32):
        factor = LOOSER.get(self.case, {}).get(name, FACTOR)
        bound = max(factor * r32, FLOOR)
        ratio = rk / r32 if r32 > 0 else (0.0 if rk == 0 else math.inf)
        self.report.setdefault(path, {})[name] = {"rho": rk, "rho32": r32, "ratio": ratio}
        if not rk <= bound:
            self.failures.append(f"{path} {name}: max rho {rk:.3g} > bound {bound:.3g} (fp32 torch {r32:.3g})")

    def bar(self, path, name, a, ref, a32=None):
        """inside the trained range: the README's parity bar, and nothing non-finite where fp64 is finite.  Where fp32
        torch itself misses the bar (a32: its result), FACTOR times its error replaces it"""
        if not self.in_range:
            return
        a, ref = a.double(), ref.double()
        fin = torch.isfinite(ref)
        if bool((~torch.isfinite(a) & fin).any()):
            self.failures.append(f"{path} {name}: non-finite where fp64 is finite")
        err = lambda x: float(((x.double() - ref).abs() / ref.abs().clamp_min(1.0))[fin].max()) if bool(fin.any()) else 0.0
        bar = max(BAR, FACTOR * err(a32)) if a32 is not None else BAR
        if not err(a) <= bar:
            self.failures.append(f"{path} {name}: max |err| / max(1, |fp64|) = {err(a):.3g} > {bar:.3g}")


def _judge_forward(J, path, out, r64, r32, S):
    zv = []
    for name in ("cv", "att"):
        J.note(path, name, rho(out[name], r64[name], S[name], name, zv), rho(r32[name], r64[name], S[name], "", []))
        J.bar(path, name, out[name], r64[name], r32[name])
    J.failures += [f"{path} {v}" for v in zv]


def _judge_topk(J, path, out, r64, r32, S):
    lg = r64["logits"]
    idx = out["topk_idx"]
    ref = lg.gather(1, idx)
    rl32 = rho(r32["logits"], lg, S["logits"], "", [])
    J.note(path, "topk", float(((out["topk"].double() - ref).abs() / S["logits"].gather(1, idx)).max()), rl32)
    J.bar(path, "topk", out["topk"], ref)
    # the first label is an fp64 maximum up to the same bound on both logits
    mx64, am64 = lg.max(1)
    b = torch.arange(lg.shape[0], device=lg.device)
    slack = max(FACTOR * rl32, FLOOR) * (S["logits"][b, idx[:, 0]] + S["logits"][b, am64])
    n_wrong = int((ref[:, 0] < mx64 - slack).sum())
    if n_wrong:
        J.failures.append(f"{path}: {n_wrong} rows whose first label is not an fp64 maximum")


def _judge_train(J, path, out, r64, r32, S):
    _judge_forward(J, path, out, r64, r32, S)
    zv = []
    J.note(path, "loss", rho(out["loss"], r64["loss"], S["loss"], "loss", zv), rho(r32["loss"], r64["loss"], S["loss"], "", []))
    J.bar(path, "loss", out["loss"], r64["loss"])
    lg = r64["logits"]
    mx64 = lg.max(1).values
    b = torch.arange(lg.shape[0], device=lg.device)
    rl32 = rho(r32["logits"], lg, S["logits"], "", [])
    J.note(path, "pred_score", float(((out["pred_score"].double() - mx64).abs() / S["logits"][b, out["am"]]).max()), rl32)
    J.bar(path, "pred_score", out["pred_score"], mx64)
    J.note(path, "dcv", rho(out["dcv"], r64["taps"]["cv"][1], S["dcv"], "dcv", zv),
           rho(r32["taps"]["cv"][1], r64["taps"]["cv"][1], S["dcv"], "", []))
    for name, g in out["grads"].items():
        J.note(path, name, rho(g, r64["grads"][name], S[name], name, zv), rho(r32["grads"][name], r64["grads"][name], S[name], "", []))
    J.failures += [f"{path} {v}" for v in zv]


def _run_case(case, monkeypatch):
    shape, modify, in_range, paths = CASES[case]
    w = SHAPES[shape]
    dev = torch.device("cuda:0")
    P = _params(w, dev)
    batch = _batch(w, dev)
    modify(P, batch)
    mask = torch.ones((), device=dev)
    r32 = reference(P, batch, mask, False, torch.float32)
    r32 = {"loss": r32["loss"], "logits": r32["logits"], "cv": r32["cv"], "att": r32["att"], "grads": r32["grads"],
           "taps": {"cv": r32["taps"]["cv"]}}
    r64 = reference(P, batch, mask, False, torch.float64)
    S = scales(r64, batch, mask, False)
    x = r64["taps"]["x"][0]
    ratio = x.mean(-1).abs() / x.std(-1, unbiased=False).clamp_min(1e-300)
    J = Judge(case, in_range)
    J.report["ln_mean_over_std_rms"] = float(ratio[batch[0] > 0].square().mean().sqrt())
    for path in paths:
        if path in ("train", "train-dc"):
            with monkeypatch.context() as mp:
                if path == "train-dc":
                    mp.setenv("C2V_BACKWARD_DC", "ffma")
                out = _run_train(w, P, batch)
            _judge_train(J, path, out, r64, r32, S)
        else:
            out = _run_eval(w, P, batch, "tcgen05" if path == "eval-tc" else "ffma")
            _judge_forward(J, path, out, r64, r32, S)
            _judge_topk(J, path, out, r64, r32, S)
        del out
        torch.cuda.empty_cache()
    return J


# Out of the trained range and beyond any factor: W_out x 2^20 makes the softmax one-hot, so G is exactly 0 in fp64 for
# the rows whose label wins, while the fused dlogits leaves a residue there (G fp16 split, exp of logits ~2^20 apart).
XFAIL = {"w_out-2^20": "W_out x 2^20: one-hot softmax, nonzero G residue where fp64 G is exactly 0 (G fp16 split)"}


@pytest.mark.parametrize("case", [pytest.param(c, marks=pytest.mark.xfail(strict=True, reason=XFAIL[c])) if c in XFAIL
                                  else c for c in CASES])
def test_value_range(case, monkeypatch):
    J = _run_case(case, monkeypatch)
    print(f"\n[value-range {case}] " + json.dumps(J.report, default=float))
    assert not J.failures, "\n".join(J.failures)


# ---- fp16 overflow of the unscaled gathered operand ------------------------------------------------------------------
# The encode's A producers split the gathered fp32 embedding rows into fp16 hi + lo with no scale.  An entry that rounds
# to +-inf in fp16 (|v| >= 65520) makes hi = inf and lo = NaN: the contexts gathering it get a NaN x and their bags a NaN
# code vector, where fp32 is finite.  65519 still rounds to 65504.  Pinned as strict xfails so that a fix shows up.
@pytest.mark.parametrize("value", [65504.0, 65519.0,
                                   pytest.param(65520.0, marks=pytest.mark.xfail(strict=True, reason="fp16 overflow of the "
                                                "unscaled gathered embedding row on the tensor cores")),
                                   pytest.param(70000.0, marks=pytest.mark.xfail(strict=True, reason="fp16 overflow of the "
                                                "unscaled gathered embedding row on the tensor cores"))])
def test_fp16_overflow_of_gathered_rows(value):
    w = SHAPES[128]
    dev = torch.device("cuda:0")
    P = _params(w, dev)
    batch = _batch(w, dev)
    _entry("terminal_embedding.weight", value, row=w["T"] - 1)(P, batch)     # gathered by bag 3 only
    out = _run_eval(w, P, batch, "tcgen05")
    r64 = reference(P, batch, torch.ones((), device=dev), False, torch.float64)
    assert bool(torch.isfinite(r64["cv"]).all())
    assert bool(torch.isfinite(out["cv"]).all()), f"non-finite code vectors in bags {torch.nonzero(~torch.isfinite(out['cv']).all(1)).view(-1).tolist()}"


# ---- non-finite containment ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("value", [math.inf, math.nan])
@pytest.mark.parametrize("where", ["table", "w_out"])
def test_non_finite_stays_local(where, value):
    """one inf / NaN table row changes only the bags that gather it; one inf / NaN W_out entry only its label's column.
    Everything else meets the criterion: no global scale is poisoned by one value"""
    w = SHAPES[128]
    dev = torch.device("cuda:0")
    P = _params(w, dev)
    batch = _batch(w, dev)
    s, p, e, lab = batch
    B = w["B"]
    keep_b = torch.ones(B, dtype=torch.bool, device=dev)
    keep_c = torch.ones(w["C"], dtype=torch.bool, device=dev)
    if where == "table":
        P["terminal_embedding.weight"] = P["terminal_embedding.weight"].clone()
        P["terminal_embedding.weight"][w["T"] - 1] = value                    # gathered by bag 3 only
        keep_b[3] = False
    else:
        P["output_linear.weight"] = P["output_linear.weight"].clone()
        P["output_linear.weight"][11, 5] = value
        keep_c[11] = False
    Pc = dict(P)                                    # the same parameters with the non-finite value replaced by 0
    key = "terminal_embedding.weight" if where == "table" else "output_linear.weight"
    Pc[key] = torch.nan_to_num(P[key], nan=0.0, posinf=0.0)
    mask = torch.ones((), device=dev)
    # the references of the finite parameters: identical on the kept bags / columns
    r64 = reference(Pc, batch, mask, False, torch.float64)
    r32 = reference(Pc, batch, mask, False, torch.float32)
    S = scales(r64, batch, mask, False)
    J = Judge(f"non-finite-{where}", True)
    for path, algo in (("eval-tc", "tcgen05"), ("eval-ffma", "ffma")):
        m = _model(w, P, algo=algo).eval()
        cv, att, _ = m._encode_eval(s, p, e)
        logits = CF.label_logits(m._dims(), CF.make_params(w_out=m.output_linear.weight, b_out=m.output_linear.bias), cv,
                                 m._label_algo, cache=m._lab_cache, weight=m.output_linear.weight)
        kb, kc = keep_b, keep_c
        for name, a, ref, r_32, Sx in (("cv", cv[kb], r64["cv"][kb], r32["cv"][kb], S["cv"][kb]),
                                       ("att", att[kb], r64["att"][kb], r32["att"][kb], S["att"][kb]),
                                       ("logits", logits[kb][:, kc], r64["logits"][kb][:, kc], r32["logits"][kb][:, kc],
                                        S["logits"][kb][:, kc])):
            J.note(path, name, rho(a, ref, Sx, name, []), rho(r_32, ref, Sx, "", []))
            J.bar(path, name, a, ref)
    print(f"\n[value-range non-finite {where} {value}] " + json.dumps(J.report, default=float))
    assert not J.failures, "\n".join(J.failures)


# ---- the functional label API on code vectors of any magnitude ------------------------------------------------------
@pytest.mark.parametrize("s", [-12, -8, -4, 0, 4])
def test_label_api_code_vector_magnitude(s):
    """label_logits / _argmax, label_loss + label_dlogits + label_backward (absmax_ready or not) and label_topk on code
    vectors with entries ~2^s (the model's own lie within +-1/(1-p))"""
    w = SHAPES[128]
    dev = torch.device("cuda:0")
    B, C, H = w["B"], w["C"], w["H"]
    P = _params(w, dev)
    W, bias = P["output_linear.weight"], P["output_linear.bias"]
    g = torch.Generator(device=dev).manual_seed(3)
    cv = torch.randn(B, H, generator=g, device=dev) * 2.0 ** s
    lab = torch.randint(0, C, (B,), generator=g, device=dev)
    dims = CF.make_dims(w["T"], w["P"], C, w["Et"], w["Ep"], H)
    params = CF.make_params(w_out=W, b_out=bias)

    def ref(dtype):
        c = cv.to(dtype).requires_grad_()
        Wd = W.to(dtype).requires_grad_()
        bd = bias.to(dtype).requires_grad_()
        lg = torch.nn.functional.linear(c, Wd, bd)
        lg.retain_grad()
        loss = torch.nn.functional.cross_entropy(lg, lab)
        loss.backward()
        return {"logits": lg.detach(), "loss": loss.detach(), "dcv": c.grad, "dw": Wd.grad, "db": bd.grad, "G": lg.grad}
    r64, r32 = ref(torch.float64), ref(torch.float32)
    G = r64["G"].abs()
    S = {"logits": cv.double().abs() @ W.double().abs().t() + bias.double().abs(),
         "dcv": G @ W.double().abs(), "dw": G.t() @ cv.double().abs(), "db": G.sum(0)}
    lse = torch.logsumexp(r64["logits"], 1)
    S["loss"] = (lse.abs() + r64["logits"].gather(1, lab[:, None])[:, 0].abs()).mean()
    J = Judge(f"label-api-2^{s}", -8 <= s <= 4)
    b = torch.arange(B, device=dev)
    mx64 = r64["logits"].max(1).values
    rl32 = rho(r32["logits"], r64["logits"], S["logits"], "", [])
    cache = CF.PrepCache()
    lg = CF.label_logits(dims, params, cv, cache=cache, weight=W)
    J.note("logits", "logits", rho(lg, r64["logits"], S["logits"], "logits", []), rl32)
    J.bar("logits", "logits", lg, r64["logits"])
    _, am, mx = CF.label_logits_argmax(dims, params, cv, cache=cache, weight=W, want_logits=False)
    J.note("argmax", "max", float(((mx.double() - mx64).abs() / S["logits"][b, am]).max()), rl32)
    J.bar("argmax", "max", mx, mx64)
    loss, lse_k, am, mx, _ = CF.label_loss(dims, params, cv, lab, cache=cache, weight=W)
    J.note("loss", "loss", rho(loss, r64["loss"], S["loss"], "loss", []), rho(r32["loss"], r64["loss"], S["loss"], "", []))
    J.bar("loss", "loss", loss, r64["loss"])
    for ready in (True, False):
        Gk = CF.label_dlogits(dims, params, cv, lab, lse_k, 1.0 / B, cache=cache, weight=W)
        d_cv, d_w, d_b = CF.label_backward(dims, params, cv, Gk, cache=cache, weight=W, absmax_ready=ready)
        path = "backward-absmax-ready" if ready else "backward"
        for name, a in (("dcv", d_cv), ("dw", d_w), ("db", d_b)):
            J.note(path, name, rho(a, r64[name], S[name], name, []), rho(r32[name], r64[name], S[name], "", []))
    idx, val, _ = CF.label_topk(dims, params, cv, TOPK, want_probs=False, cache=cache, weight=W)
    ref_v = r64["logits"].gather(1, idx)
    J.note("topk", "topk", float(((val.double() - ref_v).abs() / S["logits"].gather(1, idx)).max()), rl32)
    J.bar("topk", "topk", val, ref_v)
    print(f"\n[value-range label-api 2^{s}] " + json.dumps(J.report, default=float))
    assert not J.failures, "\n".join(J.failures)


# ---- the angular head ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("inverse_temp", [30.0, 64.0])
@pytest.mark.parametrize("octaves", [0, pytest.param(20, marks=pytest.mark.xfail(strict=True, reason=(
    "W_out row norms over 2^+-20: the angular head's W_out image takes one power-of-two scale from max |W|, so rows "
    "2^40 below the largest lose every bit, and cos, the loss and all gradients go wrong")))])
def test_angular_head_row_norms(octaves, inverse_temp, monkeypatch):
    """the angular-margin head (fused loss and its backward, predict_topk) with W_out row norms over 2^+-octaves"""
    w = SHAPES[128]
    dev = torch.device("cuda:0")
    P = _params(w, dev)
    P["output_linear"] = P.pop("output_linear.weight")
    del P["output_linear.bias"]
    g = torch.Generator(device=dev).manual_seed(8)
    P["output_linear"] = P["output_linear"] * torch.exp2(
        torch.randint(-octaves, octaves + 1, (w["C"], 1), generator=g, device=dev).float())
    batch = _batch(w, dev)
    mask = torch.ones((), device=dev)
    r32 = reference(P, batch, mask, True, torch.float32, 0.5, inverse_temp)
    r64 = reference(P, batch, mask, True, torch.float64, 0.5, inverse_temp)
    S = scales(r64, batch, mask, True, 0.5, inverse_temp)
    J = Judge(f"angular-2^+-{octaves}-s{inverse_temp:g}", True)
    out = _run_train(w, P, batch, angular=True, inverse_temp=inverse_temp)
    _judge_train(J, "train", out, r64, r32, S)
    print(f"\n[value-range angular 2^+-{octaves} s={inverse_temp:g}] " + json.dumps(J.report, default=float))
    assert not J.failures, "\n".join(J.failures)


# ---- kNN: rows of any finite magnitude -------------------------------------------------------------------------------
def _knn_rows(kind, n, H, g, dev):
    x = torch.randn(n, H, generator=g, device=dev)
    if kind == "2^100":
        return x * 2.0 ** 100
    if kind == "2^-100":
        return x * 2.0 ** -100
    if kind == "subnormal":
        return x * 2.0 ** -140
    if kind == "below-clamp":                      # norm below F.normalize's 1e-12: the clamp decides, cos != 1 for a pair
        return x * (1e-14 / math.sqrt(H))
    if kind == "mixed":
        f = torch.tensor([2.0 ** 100, 2.0 ** -100, 2.0 ** -140, 1e-14 / math.sqrt(H), 1.0], device=dev)
        return x * f[torch.arange(n, device=dev) % 5][:, None]
    return x


@pytest.mark.parametrize("kind", ["init", "2^100", "2^-100", "subnormal", "below-clamp", "mixed"])
def test_knn_row_magnitudes(kind):
    """search() against fp64 cosines with F.normalize's clamp: each returned similarity within 2^-20 of fp64 (|cos| <= 1),
    and the first hit an fp64 maximum up to the same slack"""
    H, N, Q = 128, 3000, 200
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(5)
    bank = _knn_rows(kind, N, H, g, dev).contiguous()
    queries = _knn_rows(kind, Q, H, g, dev).contiguous()

    def cos64(a, b):
        a, b = a.double(), b.double()
        return (a @ b.t()) / (a.norm(dim=1, keepdim=True).clamp_min(1e-12) * b.norm(dim=1).clamp_min(1e-12)[None, :])
    ref = cos64(queries, bank)
    idx, sims = CodeVectorIndex(bank).search(queries, k=TOPK)
    err = float((sims.double() - ref.gather(1, idx)).abs().max())
    first_gap = float((ref.max(1).values - ref.gather(1, idx[:, :1])[:, 0]).max())
    print(f"\n[value-range knn {kind}] " + json.dumps({"max_err": err, "first_gap": first_gap}))
    assert bool(torch.isfinite(sims).all())
    assert err <= FLOOR, f"max |sim - fp64 cos| = {err:.3g}"
    assert first_gap <= 2 * FLOOR, f"first hit {first_gap:.3g} below the fp64 maximum"

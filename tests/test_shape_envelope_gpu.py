"""-m gpu: every kernel path across its shape envelope, against fp64, element by element (tests/fp64_judge.py).

The library picks its kernels by shape (tests/shape_envelope.py lists the rules and the cases).  Each case here names the
kernels it must reach; torch.profiler checks that they ran and that the alternatives did not, so a silent fallback fails
the case instead of making it test nothing.

  * training cases: Code2Vec.forward_loss + backward with dropout 0.25 (the kernels' Philox mask rebuilt with
    philox_ref.dropout_mask), padded and packed batches: cv, att, loss, pred_score, d cv and every parameter gradient;
  * a terminal table past 4 GB, judged on the compacted rows its batch touches;
  * label-head cases (functional API, plain and angular head): loss, lse, arg-max, dlogits, label backward (d cv, dW, db)
    and top-k; the logits, arg-max and loss modes also under C2V_LABEL_ORDER=groups / lanes, bit for bit equal to the
    default order (every output tile is computed by one CTA in a fixed k order, whichever order hands out the tiles).

Per tensor, max rho(kernel) <= max(FACTOR * max rho(fp32 torch), 2^-20), or the case's entry in LOOSER; where S = 0 the
kernel's value must be exactly 0.  Each case prints one JSON line: per tensor the kernel's rho, fp32 torch's rho and
their ratio.
"""
import json
import math
import types

import pytest
import torch
import torch.nn.functional as F

import shape_envelope as SE
from code2vec_b200 import functional as CF
from code2vec_b200.model import Code2Vec
from fp64_judge import reference, rho, scales
from philox_ref import dropout_mask

pytestmark = pytest.mark.gpu

FACTOR, FLOOR = 8.0, 2.0 ** -20
DROPOUT, MARGIN, INV_TEMP = 0.25, 0.5, 30.0

# Tensors that need more than FACTOR, per case: measured on one H100 80GB HBM3 (700 W, 132 SMs), the measured ratio
# max rho(kernel) / max rho(fp32 torch) in brackets.  Each is a precision deficit of the kernels as they are, not a
# tolerance for a wrong result.
#  * cv where |h| is small: every encode (tensor and CUDA cores alike) evaluates tanh through exp, with an absolute error of
#    ~2^-24 where torch's tanh is accurate relative to its value, and the tensor-core encode's x comes from fp16 hi/lo
#    splits (~22 bits).  S_cv = sum att |h| is small where h is near 0 in every context of a short bag, so cv's rho is
#    large there for fp32 torch too (up to ~2e-4) and the ratio spreads.  Worst in one-context bags ("cv one-context",
#    cv = h; as cfg2-zipf in test_train_step_gpu.py), and in ragged bags of a few contexts ("cv").  The bags whose cv is a
#    softmax-weighted sum over many partials are judged at FACTOR.
#  * one context (B = L = 1): no gradient is a sum, so fp32 torch rounds each element once or twice, while the kernels
#    carry their intermediates' errors: dW on the tensor cores takes dX and the gathered rows as fp16 hi/lo splits, and d W_out
#    = G^T cv inherits cv's error above.
#  * near FACTOR from run to run (gradients accumulate with atomics, in no fixed order): listed at 16.
#  * label head: d W_out = G^T cv takes G = d loss / d logits as an fp16 hi/lo split under ONE scale
#    (c2v_label_backward_tc.cu), so the W_out rows of labels whose G entries are small next to max |G| lose relative
#    accuracy (as "label-api" in test_value_range_gpu.py).  The angular head's d W_out takes its G the same way.
LOOSER = {
    "e4-4-h100-b1x1": {"input_linear.weight": 32.0},                                         # [15]
    "e124-124-h128-b1x1": {"input_layer_norm.weight": 16.0},                                 # [8.0]
    "e124-124-h128-b129x33": {"cv": 64.0},                                                  # [24]
    "e124-124-h128-b129x33-packed": {"cv": 64.0},                                           # [24]
    "e124-124-h128-b7x333": {"cv one-context": 64.0},                                       # [33]
    "e132-132-h256-b7x333": {"cv one-context": 16.0},                                       # [7.3]
    "e256-256-h256-b1x1": {"cv one-context": 256.0, "input_linear.weight": 64.0,            # [90, 29]
                           "output_linear.weight": 256.0},                                  # [88]
    "e256-256-h256-b129x33": {"cv one-context": 16.0},                                      # [9.6]
    "e256-256-h256-b7x333": {"cv one-context": 32.0, "att": 16.0,                           # [16, 7.0]
                             "input_layer_norm.weight": 16.0, "output_linear.weight": 16.0},  # [7.5, 7.0]
    "e128-128-h4-b1x1": {"input_linear.weight": 128.0, "input_layer_norm.bias": 16.0},      # [76, 9.1]
    "e256-256-h252-b1x1": {"input_linear.weight": 32.0},                                    # [13]
    "e256-256-h252-b129x33": {"cv": 16.0},                                                  # [9.2]
    "e128-96-h128-b1x1": {"input_layer_norm.bias": 16.0},                                   # [8.7]
    "e128-128-h260-b129x33": {"cv": 16.0},                                                  # [10]
    "e128-128-h128-b85x200": {"cv": 16.0},                                                  # [10]
    "b1-c16897-h256": {"dw": 32.0, "dw_g": 64.0, "angular dw": 128.0},                      # [14, 33, 81]
    "b129-c195299-h100": {"dw": 16.0, "dw_g": 128.0},                                       # [10, 45]
    "b1793-c129-h100": {"dw": 64.0, "dw_g": 64.0, "angular dw": 32.0},                      # [34, 36, 15]
    "b1920-c1023-h4": {"dw": 64.0, "dw_g": 64.0, "angular dw": 32.0},                       # [32, 25, 12]
    "b1920-c128-h256": {"dw_g": 64.0, "angular dw": 32.0},                                  # [29, 17]
}
# One label (C = 1): the angular head's softmax is constant, so d cv and d W_out are exactly 0 in fp64 and fp32 torch, and
# S = 0 everywhere.  The kernels leave a rounding residue there (their G = exp(logit - lse) - 1 is not exactly 0, where
# the plain head's is).  There the residue must be finite and within 2^-20 of the scale the gradient
# would have with |G| = 1 / B: inverse_temp |wn| / (B |cv|) for d cv, inverse_temp sum_b |cvn_b| / (B |w|) for d W_out.
C1_RESIDUE = ("angular dcv", "angular dw")


@pytest.fixture(autouse=True)
def _fp32_without_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved
    torch.cuda.empty_cache()


def _kernel_names(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        res = fn()
        torch.cuda.synchronize()
    return res, {e.key for e in prof.key_averages() if "c2v::" in e.key}


def _dispatch_failures(names, paths):
    """each stage launched the kernels of its expected path and none of the other path's"""
    out = []
    for stage, path in paths.items():
        other = SE.FFMA if path == SE.TC else SE.TC
        for k in SE.KERNELS[stage][path]:
            if not any(k in n for n in names):
                out.append(f"dispatch {stage}: {k} did not run ({path} expected)")
        for k in SE.KERNELS[stage][other]:
            if any(k in n for n in names):
                out.append(f"dispatch {stage}: {k} ran ({path} expected)")
    return out


def _mode_dispatch(names, mode, want):
    """a label-head mode launched its tensor-core kernels (the instantiation named by its template prefix) and no
    CUDA-core GEMM"""
    out = [f"dispatch {mode}: {k} did not run" for k in want if not any(k in n for n in names)]
    if any("sgemm_kernel" in n for n in names):
        out.append(f"dispatch {mode}: sgemm_kernel ran")
    return out


class Judge:
    """per tensor: the kernel's and fp32 torch's rho, and the failures of one case"""

    def __init__(self, case):
        self.case, self.report, self.failures = case, {}, []

    def note(self, name, rk, r32):
        factor = LOOSER.get(self.case, {}).get(name, FACTOR)
        bound = max(factor * r32, FLOOR)
        ratio = rk / r32 if r32 > 0 else (0.0 if rk == 0 else math.inf)
        self.report[name] = {"rho": rk, "rho32": r32, "ratio": ratio}
        if not rk <= bound:
            self.failures.append(f"{name}: max rho {rk:.3g} > bound {bound:.3g} (fp32 torch {r32:.3g})")

    def full(self, name, a, ref, r32, S):
        zv = []
        self.note(name, rho(a, ref, S, name, zv), rho(r32, ref, S, "", []))
        self.failures += zv

    def residue(self, name, a, S1):
        """where S = 0 by symmetry: finite, and |a| <= 2^-20 S1"""
        if not bool(torch.isfinite(a).all()):
            self.failures.append(f"{name}: non-finite")
        r = float((a.double().abs() / S1).max())
        self.report[name] = {"residue": r}
        if not r <= FLOOR:
            self.failures.append(f"{name}: residue {r:.3g} x the |G| = 1/B scale > 2^-20")

    def argmax(self, name, am, mx, lg64, S, rl32):
        """mx: the rho rule on the row's maximum; am: an fp64 maximum up to the same bound on both logits"""
        mx64, am64 = lg64.max(1)
        b = torch.arange(lg64.shape[0], device=lg64.device)
        self.note(name, float(((mx.double() - mx64).abs() / S[b, am64]).max()), rl32)
        slack = max(FACTOR * rl32, FLOOR) * (S[b, am] + S[b, am64])
        n_wrong = int((lg64[b, am] < mx64 - slack).sum())
        if n_wrong:
            self.failures.append(f"{name}: {n_wrong} rows whose arg-max is not an fp64 maximum")

    def topk(self, name, idx, val, lg64, S, rl32):
        """values by the rho rule at their labels; k distinct labels, in descending order, each within the bound of the
        fp64 k-th largest"""
        k = idx.shape[1]
        ref = lg64.gather(1, idx)
        Sk = S.gather(1, idx)
        self.note(name, float(((val.double() - ref).abs() / Sk).max()), rl32)
        if k > 1:
            if bool((idx.sort(1).values.diff(dim=1) == 0).any()):
                self.failures.append(f"{name}: repeated labels in a row")
            if bool((val.diff(dim=1) > 0).any()):
                self.failures.append(f"{name}: values not in descending order")
        kth64 = lg64.topk(k, dim=1).values[:, -1:]
        slack = max(FACTOR * rl32, FLOOR) * 2 * S.max(1, keepdim=True).values
        n_wrong = int((ref < kth64 - slack).sum())
        if n_wrong:
            self.failures.append(f"{name}: {n_wrong} labels outside the fp64 top {k}")


# ---- training cases ----------------------------------------------------------------------------------------------------
def _params(c, dev, seed=1):
    """init scale, as bench.synth_params, with a small LN jitter and bias so that no term is exactly 0"""
    g = torch.Generator(device=dev).manual_seed(seed)
    D = 2 * c["Et"] + c["Ep"]
    r = lambda *s: torch.randn(*s, generator=g, device=dev)
    u = lambda bound, *s: (torch.rand(*s, generator=g, device=dev) * 2 - 1) * bound
    return {"terminal_embedding.weight": r(c["T"], c["Et"]), "path_embedding.weight": r(c["P"], c["Ep"]),
            "input_linear.weight": u(D ** -0.5, c["H"], D),
            "input_layer_norm.weight": 1.0 + 0.1 * r(c["H"]), "input_layer_norm.bias": 0.1 * r(c["H"]),
            "attention_parameter": r(c["H"]) * (2.0 / (c["H"] + 1)) ** 0.5,
            "output_linear.weight": u(c["H"] ** -0.5, c["C"], c["H"]), "output_linear.bias": 0.05 * r(c["C"])}


def _batch(c, dev, seed=2):
    """bags with a zero-padded suffix (bag 0 full, bag 1 of one context, the rest ragged), indices >= 1; the last rows
    of both tables are gathered (terminal row T - 1 as a start and as an end)"""
    g = torch.Generator(device=dev).manual_seed(seed)
    B, L, T, P = c["B"], c["L"], c["T"], c["P"]
    s = torch.randint(1, T - 1, (B, L), generator=g, device=dev)
    p = torch.randint(1, P - 1, (B, L), generator=g, device=dev)
    e = torch.randint(1, T - 1, (B, L), generator=g, device=dev)
    n = torch.randint(1, L + 1, (B,), generator=g, device=dev)
    n[0] = L
    if B > 1:
        n[1] = 1
    s[0, L - 1], p[0, L - 1], e[B - 1, 0] = T - 1, P - 1, T - 1
    valid = torch.arange(L, device=dev)[None, :] < n[:, None]
    s, p, e = s * valid, p * valid, e * valid
    lab = torch.randint(0, c["C"], (B,), generator=g, device=dev)
    return s, p, e, lab


def _model(c, P, dev):
    """Code2Vec holding the parameters P (built with 2-row tables, which are then replaced, so that a table past 4 GB
    is never initialised on the host)"""
    o = types.SimpleNamespace(terminal_count=2, path_count=2, label_count=c["C"], terminal_embed_size=c["Et"],
                              path_embed_size=c["Ep"], encode_size=c["H"], dropout_prob=DROPOUT,
                              angular_margin_loss=False, angular_margin=MARGIN, inverse_temp=INV_TEMP, device=dev)
    m = Code2Vec(o).to(dev)
    o.terminal_count, o.path_count = c["T"], c["P"]
    m.terminal_embedding.weight = torch.nn.Parameter(P["terminal_embedding.weight"])
    m.path_embedding.weight = torch.nn.Parameter(P["path_embedding.weight"])
    with torch.no_grad():
        for n, q in m.named_parameters():
            if "embedding" not in n:
                q.copy_(P[n])
    return m.train()


def _packed(s, p, e):
    valid = s > 0
    n = valid.sum(1)
    offsets = torch.zeros(s.shape[0] + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(n.cpu(), 0)
    return CF.PackedBags(s[valid].contiguous(), p[valid].contiguous(), e[valid].contiguous(), offsets, s.shape[1])


def _run_train(c, P, batch, dev):
    """-> (outputs in the padded layout, dropout mask [B, L, H], the c2v:: kernels launched)"""
    m = _model(c, P, dev)
    torch.manual_seed(0)                        # Code2Vec draws its dropout key from torch's CPU generator
    seeds = []
    next_seed = m._next_seed
    m._next_seed = lambda: seeds.append(next_seed()) or seeds[-1]
    s, p, e, lab = batch
    packed = c["layout"] == "packed"
    x = (_packed(s, p, e), None, None) if packed else (s, p, e)
    out = {}

    def work():
        loss, am, mx, cv, att = m.forward_loss(*x, lab)
        out.update(loss=loss.detach().clone(), am=am.clone(), pred_score=mx.clone(), cv=cv.detach().clone(),
                   att=att.detach().clone())
        if "dw" in c["paths"]:
            cv.register_hook(lambda g_: out.__setitem__("dcv", g_.detach().clone()))
            loss.backward()
    _, names = _kernel_names(work)
    if packed:
        valid = s > 0
        att = torch.zeros(s.shape, device=dev)
        att[valid] = out["att"]
        out["att"] = att
    out["grads"] = {n: q.grad for n, q in m.named_parameters()}
    B, L = s.shape
    mask = torch.from_numpy(dropout_mask(seeds[-1], B * L, c["H"], DROPOUT).reshape(B, L, c["H"])).to(dev)
    return out, mask, names


def _compact_terminals(P, batch, out):
    """the terminal rows the batch touches (row 0 first) -> the parameters and batch on those rows, the kernel's
    gradient on them; failures if any other row of the kernel's gradient is nonzero"""
    s, p, e, lab = batch
    dev = s.device
    rows = torch.unique(torch.cat((torch.zeros(1, dtype=torch.int64, device=dev), s.reshape(-1), e.reshape(-1))))
    g = out["grads"]["terminal_embedding.weight"]
    hit = torch.zeros(g.shape[0], dtype=torch.bool, device=dev)
    hit[rows] = True
    n_stray = int((g.ne(0).any(1) & ~hit).sum())
    out["grads"]["terminal_embedding.weight"] = g[rows]
    del g
    Pc = dict(P, **{"terminal_embedding.weight": P["terminal_embedding.weight"][rows]})
    bc = (torch.searchsorted(rows, s), p, torch.searchsorted(rows, e), lab)
    return Pc, bc, ([f"terminal_embedding.weight: {n_stray} untouched rows with a nonzero gradient"] if n_stray else [])


def _judge_train(J, out, r64, r32, S, starts):
    # cv of a one-context bag is h itself: judged apart, so that the bags whose cv is a softmax-weighted sum over
    # partials (the finalize) keep their own bound
    one = (starts > 0).sum(1) <= 1
    for name, sel in (("cv", ~one), ("cv one-context", one)):
        if bool(sel.any()):
            J.full(name, out["cv"][sel], r64["cv"][sel], r32["cv"][sel], S["cv"][sel])
    J.full("att", out["att"], r64["att"], r32["att"], S["att"])
    J.full("loss", out["loss"], r64["loss"], r32["loss"], S["loss"])
    rl32 = rho(r32["logits"], r64["logits"], S["logits"], "", [])
    J.argmax("pred_score", out["am"], out["pred_score"], r64["logits"], S["logits"], rl32)
    if "dcv" not in out:
        return
    J.full("dcv", out["dcv"], r64["taps"]["cv"][1], r32["taps"]["cv"][1], S["dcv"])
    for name, g in out["grads"].items():
        J.full(name, g, r64["grads"][name], r32["grads"][name], S[name])


def _train_case(case):
    c = SE.TRAIN[case]
    dev = torch.device("cuda:0")
    P = _params(c, dev)
    batch = _batch(c, dev)
    out, mask, names = _run_train(c, P, batch, dev)
    J = Judge(case)
    J.failures += _dispatch_failures(names, c["paths"])
    if c["T"] * c["Et"] * 4 >= 2 ** 32:
        P, batch, stray = _compact_terminals(P, batch, out)
        J.failures += stray
        torch.cuda.empty_cache()
    r32 = reference(P, batch, mask, False, torch.float32)
    r32 = {"loss": r32["loss"], "logits": r32["logits"], "cv": r32["cv"], "att": r32["att"], "grads": r32["grads"],
           "taps": {"cv": r32["taps"]["cv"]}}
    r64 = reference(P, batch, mask, False, torch.float64)
    S = scales(r64, batch, mask, False)
    _judge_train(J, out, r64, r32, S, batch[0])
    return J


@pytest.mark.parametrize("case", [c for c in SE.TRAIN if c != "table-past-4GB"])
def test_training_case(case):
    J = _train_case(case)
    print(f"\n[shape-envelope {case}] " + json.dumps(J.report, default=float))
    assert not J.failures, "\n".join(J.failures)


def test_table_past_4gb():
    c = SE.TRAIN["table-past-4GB"]
    need = 3 * c["T"] * c["Et"] * 4 + (2 << 30)          # table, gradient, one transient of the compaction, headroom
    free, _ = torch.cuda.mem_get_info(0)
    if free < need:
        pytest.skip(f"a terminal table past 4 GB needs ~{need / 2 ** 30:.1f} GiB free on the device ({free / 2 ** 30:.1f})")
    J = _train_case("table-past-4GB")
    print("\n[shape-envelope table-past-4GB] " + json.dumps(J.report, default=float))
    assert not J.failures, "\n".join(J.failures)


# ---- label-head cases ----------------------------------------------------------------------------------------------------
def _label_inputs(c, dev, seed=3):
    g = torch.Generator(device=dev).manual_seed(seed)
    B, C, H = c["B"], c["C"], c["H"]
    W = (torch.rand(C, H, generator=g, device=dev) * 2 - 1) * H ** -0.5
    bias = 0.05 * torch.randn(C, generator=g, device=dev)
    cv = torch.tanh(torch.randn(B, H, generator=g, device=dev))
    lab = torch.randint(0, C, (B,), generator=g, device=dev)
    return W, bias, cv, lab


def _plain_ref(cv, W, bias, lab, dtype):
    c = cv.detach().to(dtype, copy=True).requires_grad_()
    Wd = W.detach().to(dtype, copy=True).requires_grad_()
    bd = bias.detach().to(dtype, copy=True).requires_grad_()
    lg = F.linear(c, Wd, bd)
    lg.retain_grad()
    loss = F.cross_entropy(lg, lab)
    loss.backward()
    return {"logits": lg.detach(), "lse": torch.logsumexp(lg.detach(), 1), "loss": loss.detach(), "G": lg.grad,
            "dcv": c.grad, "dw": Wd.grad, "db": bd.grad}


def _angular_ref(cv, W, lab, dtype):
    c = cv.detach().to(dtype, copy=True).requires_grad_()
    Wd = W.detach().to(dtype, copy=True).requires_grad_()
    cos = F.linear(F.normalize(c), F.normalize(Wd))
    cos.retain_grad()
    sin = torch.sqrt(1.0 - cos * cos)
    phi = torch.where(cos > 0, cos * math.cos(MARGIN) - sin * math.sin(MARGIN), cos)
    oh = torch.zeros_like(cos).scatter_(1, lab[:, None], 1)
    lg = (oh * phi + (1.0 - oh) * cos) * INV_TEMP
    loss = F.cross_entropy(lg, lab)
    loss.backward()
    return {"logits": lg.detach(), "lse": torch.logsumexp(lg.detach(), 1), "loss": loss.detach(), "Gc": cos.grad,
            "cos": cos.detach(), "topk_logits": INV_TEMP * cos.detach(), "dcv": c.grad, "dw": Wd.grad}


def _run_plain(dims, params, cv, lab, W, G_in, cache):
    B = cv.shape[0]
    o = {"logits": CF.label_logits(dims, params, cv, cache=cache, weight=W)}
    _, o["am_only"], o["mx_only"] = CF.label_logits_argmax(dims, params, cv, cache=cache, weight=W, want_logits=False)
    o["loss"], o["lse"], o["am"], o["mx"], _ = CF.label_loss(dims, params, cv, lab, cache=cache, weight=W)
    o["G"] = CF.label_dlogits(dims, params, cv, lab, o["lse"], 1.0 / B, cache=cache, weight=W)
    o["dcv"], o["dw"], o["db"] = CF.label_backward(dims, params, cv, o["G"], cache=cache, weight=W, absmax_ready=True)
    o["dcv_g"], o["dw_g"], o["db_g"] = CF.label_backward(dims, params, cv, G_in, cache=cache, weight=W)
    return o


ORDER_KEYS = ("logits", "am_only", "mx_only", "loss", "lse", "am", "mx")


@pytest.mark.parametrize("case", list(SE.LABEL))
def test_label_head_case(case, monkeypatch):
    c = SE.LABEL[case]
    dev = torch.device("cuda:0")
    B, C, H = c["B"], c["C"], c["H"]
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    if case in SE.LABEL_GROUPS_CASES:
        assert SE.default_label_order(B, C, sms) == "groups", f"{sms} SMs: this batch takes lane order by default"
    W, bias, cv, lab = _label_inputs(c, dev)
    dims = CF.make_dims(10, 10, C, H, H, H)
    params = CF.make_params(w_out=W, b_out=bias)
    J = Judge(case)
    r64 = _plain_ref(cv, W, bias, lab, torch.float64)
    r32 = _plain_ref(cv, W, bias, lab, torch.float32)
    G_in = r64["G"].float()                     # the label backward on a given G: fp64's, rounded to fp32
    cache = CF.PrepCache()
    o, names = _kernel_names(lambda: _run_plain(dims, params, cv, lab, W, G_in, cache))
    J.failures += _dispatch_failures(names, {"label": SE.TC})
    J.failures += _mode_dispatch(names, "plain", ("label_gemm_v2_kernel<false, false",))
    # the same calls in each tile order: bit for bit the default order's results
    for order in ("groups", "lanes"):
        with monkeypatch.context() as mp:
            mp.setenv("C2V_LABEL_ORDER", order)
            oo = _run_plain(dims, params, cv, lab, W, G_in, CF.PrepCache())
        for k in ORDER_KEYS:
            if not torch.equal(oo[k], o[k]):
                J.failures.append(f"C2V_LABEL_ORDER={order}: {k} differs from the default order's")
        del oo
    # S: the last sum that produces each quantity, on absolute values
    aW, acv = W.double().abs(), cv.double().abs()
    Sl = acv @ aW.t() + bias.double().abs()
    p64 = torch.softmax(r64["logits"], 1)
    pS = (p64 * Sl).sum(1, keepdim=True)
    oh = torch.zeros_like(p64).scatter_(1, lab[:, None], 1.0)
    SG = (p64 * (Sl + pS) + p64 + oh) / B
    S = {"logits": Sl, "lse": r64["lse"].abs() + pS[:, 0],
         "loss": (r64["lse"].abs() + r64["logits"].gather(1, lab[:, None])[:, 0].abs()).mean(),
         "G": SG, "dcv": SG @ aW, "dw": SG.t() @ acv, "db": SG.sum(0)}
    rl32 = rho(r32["logits"], r64["logits"], Sl, "", [])
    J.full("logits", o["logits"], r64["logits"], r32["logits"], Sl)
    J.argmax("argmax", o["am_only"], o["mx_only"], r64["logits"], Sl, rl32)
    J.argmax("loss-argmax", o["am"], o["mx"], r64["logits"], Sl, rl32)
    for k in ("loss", "lse", "G", "dcv", "dw", "db"):
        J.full(k, o[k], r64[k], r32[k], S[k])
    # the backward on the given G: against its fp64 contractions, fp32 torch's on the same G
    Gd, aG = G_in.double(), G_in.double().abs()
    ref_g = {"dcv_g": (Gd @ W.double(), G_in @ W, aG @ aW), "dw_g": (Gd.t() @ cv.double(), G_in.t() @ cv, aG.t() @ acv),
             "db_g": (Gd.sum(0), G_in.sum(0), aG.sum(0))}
    for k, (ref, a32, Sx) in ref_g.items():
        J.full(k, o[k], ref, a32, Sx)
    del o
    for k in SE.topk_ks(C):
        (idx, val, _), names = _kernel_names(lambda: CF.label_topk(dims, params, cv, k, want_probs=False, cache=cache,
                                                                    weight=W))
        J.failures += _mode_dispatch(names, f"topk{k}", ("label_gemm_v2_kernel<false, true",))
        J.topk(f"topk{k}", idx, val, r64["logits"], Sl, rl32)
    del r64, r32, S, SG, Sl, p64
    torch.cuda.empty_cache()
    _angular_case(J, c, dims, W, cv, lab)
    print(f"\n[shape-envelope label {case}] " + json.dumps(J.report, default=float))
    assert not J.failures, "\n".join(J.failures)


def _angular_case(J, c, dims, W, cv, lab):
    """the angular head: fused loss (loss, lse, arg-max), its backward (d cv, dW) and top-k"""
    B = c["B"]
    params = CF.make_params(w_out=W)
    cache = CF.PrepCache()
    r64 = _angular_ref(cv, W, lab, torch.float64)
    r32 = _angular_ref(cv, W, lab, torch.float32)

    def run():
        loss, lse, am, mx, inv, _ = CF.angular_loss(dims, params, cv, lab, MARGIN, INV_TEMP, cache=cache, weight=W)
        g = CF.angular_dlogits(dims, params, cv, lab, lse, inv, MARGIN, INV_TEMP, 1.0 / B, cache=cache, weight=W)
        return (loss, lse, am, mx) + CF.angular_backward_ws(dims, params, cv, g, inv, cache=cache, weight=W,
                                                               absmax_ready=True)
    (loss, lse, am, mx, dcv, dw), names = _kernel_names(run)
    J.failures += _mode_dispatch(names, "angular", ("label_gemm_v2_kernel<true, false", "label_dw_tc_kernel",
                                                    "label_dcv_tc_kernel"))
    # S as fp64_judge.scales for the angular head
    Wd, cvd = W.double(), cv.double()
    wnorm = Wd.norm(dim=1, keepdim=True).clamp_min(1e-12)
    wn, cvn = Wd / wnorm, F.normalize(cvd)
    Gc = r64["Gc"].abs()
    Ac = Gc.t() @ cvn.abs()
    Sdw = (Ac + wn.abs() * (Ac * wn.abs()).sum(1, keepdim=True)) / wnorm
    Ad = Gc @ wn.abs()
    Sdcv = (Ad + cvn.abs() * (Ad * cvn.abs()).sum(1, keepdim=True)) / cvd.norm(dim=1, keepdim=True).clamp_min(1e-12)
    St = INV_TEMP * (cvn.abs() @ wn.abs().t())                  # inverse_temp * cos, no margin: top-k
    Sl = St.clone()
    cl = r64["cos"].gather(1, lab[:, None])
    sin = torch.sqrt((1.0 - cl * cl).clamp_min(1e-12))
    amp = torch.where(cl > 0, math.cos(MARGIN) + math.sin(MARGIN) * cl.abs() / sin, torch.ones_like(cl))
    Sl.scatter_(1, lab[:, None], Sl.gather(1, lab[:, None]) * amp)
    p64 = torch.softmax(r64["logits"], 1)
    Slse = r64["lse"].abs() + (p64 * Sl).sum(1)
    Sloss = (r64["lse"].abs() + r64["logits"].gather(1, lab[:, None])[:, 0].abs()).mean()
    rl32 = rho(r32["logits"], r64["logits"], Sl, "", [])
    J.full("angular loss", loss, r64["loss"], r32["loss"], Sloss)
    J.full("angular lse", lse, r64["lse"], r32["lse"], Slse)
    J.argmax("angular argmax", am, mx, r64["logits"], Sl, rl32)
    if c["C"] == 1:
        Ga = torch.full_like(Gc, INV_TEMP / B)
        Ad, Ac = Ga @ wn.abs(), Ga.t() @ cvn.abs()
        J.residue("angular dcv", dcv, (Ad + cvn.abs() * (Ad * cvn.abs()).sum(1, keepdim=True))
                  / cvd.norm(dim=1, keepdim=True).clamp_min(1e-12))
        J.residue("angular dw", dw, (Ac + wn.abs() * (Ac * wn.abs()).sum(1, keepdim=True)) / wnorm)
    else:
        J.full("angular dcv", dcv, r64["dcv"], r32["dcv"], Sdcv)
        J.full("angular dw", dw, r64["dw"], r32["dw"], Sdw)
    rt32 = rho(r32["topk_logits"], r64["topk_logits"], St, "", [])
    for k in SE.topk_ks(c["C"]):
        (idx, val, _), names = _kernel_names(lambda: CF.angular_topk(dims, params, cv, k, INV_TEMP, want_probs=False,
                                                                      cache=cache, weight=W))
        J.failures += _mode_dispatch(names, f"angular topk{k}", ("label_gemm_v2_kernel<true, true",))
        J.topk(f"angular topk{k}", idx, val, r64["topk_logits"], St, rt32)

"""-m gpu: the benchmarked training step -- bench.py's training leg, `ddp_step(model, ShardedFlatAdam, ...)` with dropout
0.25 at the benchmark's own shapes -- against an fp64 restatement, three consecutive steps per case.

At every step the references are recomputed from the parameters the CUDA model holds at that moment (no shadow model:
Adam would turn rounding differences into O(lr) moves): oracle.torch_forward + mean NLL with torch autograd on the GPU,
in fp64 (the judge) and in fp32 with TF32 off (the plain-precision baseline), on the dropout mask the kernels drew
(tests/philox_ref.py, seed recorded from Code2Vec._next_seed).

Scale-free criterion.  For every checked element i, rho_i = |g_i - g64_i| / S_i, where S_i is the last sum or contraction
that produces the quantity, evaluated in fp64 on absolute values (e.g. |dX|^T |C| for input_linear, the scatter of
|dX| |W| for the embedding tables).  Per tensor, max rho(kernel) <= max(8 * max rho(fp32 torch), 2^-20); where S_i = 0 (an
embedding row the batch does not touch, PAD row 0 when no bag is all-pad, the attention of a padded slot) the kernel's
value must be exactly 0.  One wrong row fails even when it is small next to the tensor's maximum.

Adam: fp64 Adam from the (p, g, m, v, t) the kernel read, with the hyperparameters as the fp32 values the kernel receives,
within 2 ulp of p plus lr * 2^-20; afterwards the gradient bucket, padding included, is exactly zero.
"""
import json
import math
import time
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from bench import WORKLOADS, synth_params, synth_pool
from code2vec_b200.distributed import ShardedFlatAdam, ddp_step
from code2vec_b200.model import Code2Vec
from oracle import oracle
from philox_ref import dropout_mask

pytestmark = pytest.mark.gpu

DROPOUT, LR, BETAS, EPS = 0.25, 0.01, (0.9, 0.999), 1e-8
MARGIN, INV_TEMP = 0.5, 30.0
N_STEPS = 3
FACTOR, FLOOR = 8.0, 2.0 ** -20
F32_EPS = 2.0 ** -24

# Tensors that need more than FACTOR, per case: the factor replaces FACTOR for that tensor and case only.  Measured on one
# H100 80GB HBM3 (700 W): the worst ratio max rho(kernel) / max rho(fp32 torch) over the three steps is in brackets.
# Each is a precision deficit of the kernels as they are, not a tolerance for a wrong result; a tighter kernel lowers it.
# The test prints the measured spread (log2 of the largest over the smallest nonzero per-context max |dX|, and of
# max |G| over the smallest nonzero |G|) next to the ratios.
#  * dX fp16 split: the dC and dW tensor-core GEMMs take dX as a 3-pass fp16 hi/lo split under ONE power-of-two scale
#    for the whole [B*L, H] dX (max |dX| lifted just below 2^14).  A context whose dX is 2^-k of the batch's maximum keeps
#    about 38 - k bits (its lo part falls into the fp16 subnormals), so embedding rows and input_linear entries fed only
#    by such contexts lose relative accuracy.  Zipf batches with ragged bags (att = 1 in one-context bags, att ~ 1/200
#    in full ones) spread dX over the widest range.
#  * G fp16 split: likewise the label-head backward splits G = d loss / d logits under one scale.  With the angular
#    head's logits s * cos (s = 30) the softmax spans ~e^60, and the W_out rows of labels with tiny probabilities lose
#    relative accuracy.
#  * d cv common part (cfg3, plain head, from the second step on; listed as (factor, first step)): the first Adam step
#    moves every one of the 195,299 W_out rows by about lr in the same direction, so d cv = G W_out gains a large part
#    that is nearly the same in every bag.  The label-head backward forms it from the fp16 hi/lo splits of G and of the
#    forward's W_out image (no lo*lo term: about 22 bits), so its rounding error is nearly the same in every bag as well.
#    The encode-parameter gradients sum over all 1,024 bags: that shared error adds up linearly, where fp32 torch's
#    independent errors partly cancel.  The per-element error of d cv itself stays within 5x of fp32 torch.  The three
#    encode-backward implementations give the same ratios: stashed x, x recomputed in fp32, and CUDA-core dC / dW.  The
#    softmax-backward bag sum taken from the backward's own h instead of d cv . code_vector gives the same ratios too.
LOOSER = {
    "cfg3": {"attention_parameter": (256.0, 1),         # [114] d cv common part
             "input_layer_norm.weight": (256.0, 1),     # [115]
             "input_layer_norm.bias": (256.0, 1),       # [77]
             "input_linear.weight": (128.0, 1),         # [59]  d cv common part + dX fp16 split
             "terminal_embedding.weight": (32.0, 1),    # [12]
             "path_embedding.weight": (32.0, 1)},       # [12]
    "cfg4": {"att": 16.0,                               # [7.7] scores of 256 terms of the forward's fp16-split x
             "terminal_embedding.weight": 32.0,         # [13]  dX fp16 split (encode 256: two h blocks)
             "path_embedding.weight": 32.0,             # [16]
             "input_linear.weight": 64.0},              # [23]
    "cfg2-zipf": {"cv": 16.0,                           # [10; 3.4 - 10 over runs] one-context bags: cv = h of the
                                                        #       forward's fp16-split x, fp32 torch's h is exact there
                  "terminal_embedding.weight": 1024.0,  # [313] dX fp16 split
                  "path_embedding.weight": 128.0,       # [33]
                  "input_linear.weight": 32.0,          # [16]
                  "input_layer_norm.weight": 64.0,      # [25]
                  "input_layer_norm.bias": 32.0},       # [12]
    "cfg3-angular": {"output_linear": 1024.0,           # [297] G fp16 split
                     "input_linear.weight": 32.0,       # [15]  dX fp16 split
                     "input_layer_norm.weight": 16.0},  # [9]
}

# case: (workload, data, fused loss, angular head)
CASES = {
    "cfg2": ("cfg2", "uniform", True, False),
    "cfg3": ("cfg3", "uniform", True, False),
    "cfg4": ("cfg4", "uniform", True, False),
    "cfg2-unfused": ("cfg2", "uniform", False, False),
    "cfg2-zipf": ("cfg2", "zipf", True, False),
    "cfg3-angular": ("cfg3", "uniform", True, True),
}
ALL_PAD_BAGS = (0, 1, 63, 64, 127, 128, 511, 1023)          # bags of the Zipf batches that hold no context at all


@pytest.fixture(autouse=True)
def _fp32_without_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved
    torch.cuda.empty_cache()


# ---- the model and the data, as bench.py's training leg builds them --------------------------------------------------
def _model(w, dev, angular):
    o = types.SimpleNamespace(terminal_count=w["T"], path_count=w["P"], label_count=w["C"], terminal_embed_size=w["Et"],
                              path_embed_size=w["Ep"], encode_size=w["H"], dropout_prob=DROPOUT,
                              angular_margin_loss=angular, angular_margin=MARGIN, inverse_temp=INV_TEMP, device=dev)
    p = synth_params(w, dev)
    if angular:
        p["output_linear"] = p.pop("output_linear.weight")
        del p["output_linear.bias"]
    m = Code2Vec(o)
    m.load_state_dict(p)
    return m.to(dev).train()


def _zipf(n, shape, g, dev):
    """indices 0 .. n-1 with P(i) proportional to 1 / (i + 1)"""
    cdf = torch.cumsum(1.0 / torch.arange(1, n + 1, dtype=torch.float64, device=dev), 0)
    cdf /= cdf[-1].clone()
    u = torch.rand(shape, generator=g, device=dev, dtype=torch.float64)
    return torch.searchsorted(cdf, u).clamp_(max=n - 1)


def _batches(w, data, dev):
    B, L = w["B"], w["L"]
    if data == "uniform":
        s, p, e, lab = synth_pool(w, N_STEPS, dev, 1234)
        return [(s[i * B:(i + 1) * B], p[i * B:(i + 1) * B], e[i * B:(i + 1) * B], lab[i * B:(i + 1) * B])
                for i in range(N_STEPS)]
    # Zipf-like batches: a few terminals / paths in a large share of the contexts (index 1 takes ~7 % of the terminal
    # draws: ~29 K scatter-adds into one row per step), ragged bags with a zero-padded suffix, some all-pad bags
    g = torch.Generator(device=dev).manual_seed(4321)
    out = []
    for _ in range(N_STEPS):
        s = 1 + _zipf(w["T"] - 1, (B, L), g, dev)
        p = 1 + _zipf(w["P"] - 1, (B, L), g, dev)
        e = 1 + _zipf(w["T"] - 1, (B, L), g, dev)
        lab = _zipf(w["C"], (B,), g, dev)
        n = torch.randint(1, L + 1, (B,), generator=g, device=dev)
        n[list(ALL_PAD_BAGS)] = 0
        valid = (torch.arange(L, device=dev)[None, :] < n[:, None]).long()
        out.append((s * valid, p * valid, e * valid, lab))
    return out


# ---- the references ----------------------------------------------------------------------------------------------------
def _reference(params, batch, mask, angular, dtype):
    """oracle.torch_forward + mean NLL in `dtype` with autograd -> dict of everything the checks read"""
    s, pth, e, lab = batch
    p = {k: v.detach().to(dtype).requires_grad_() for k, v in params.items()}
    taps = {}
    ang = {"margin": MARGIN, "inverse_temp": INV_TEMP} if angular else None
    out, cv, att = oracle.torch_forward(p, s, pth, e, lab, angular=ang, dropmask=mask.to(dtype), taps=taps)
    for t in taps.values():
        t.retain_grad()
    loss = F.nll_loss(F.log_softmax(out, dim=1), lab)
    loss.backward()
    r = {"loss": loss.detach(), "logits": out.detach(), "cv": cv.detach(), "att": att.detach(),
         "grads": {k: v.grad for k, v in p.items()}, "taps": {k: (v.detach(), v.grad) for k, v in taps.items()},
         "params": {k: v.detach() for k, v in p.items()}}
    del out, cv, att, loss, p, taps
    return r


def _scales(r, batch, mask, angular):
    """S for every checked quantity: its last sum / contraction in fp64 on absolute values"""
    s, pth, e, lab = batch
    P = r["params"]
    B, L = s.shape
    x, dX = r["taps"]["x"]
    ln, dY = r["taps"]["ln"]
    _, dz = r["taps"]["z"]
    H = x.shape[-1]
    N = B * L
    Wi = P["input_linear.weight"]
    Et, Ep = P["terminal_embedding.weight"].shape[1], P["path_embedding.weight"].shape[1]
    S = {}
    adX = dX.reshape(N, H).abs()
    # input_linear: dW = dX^T C
    aC = torch.cat((P["terminal_embedding.weight"][s.reshape(-1)].abs(), P["path_embedding.weight"][pth.reshape(-1)].abs(),
                    P["terminal_embedding.weight"][e.reshape(-1)].abs()), dim=1)
    S["input_linear.weight"] = adX.t() @ aC
    del aC
    # embedding tables: the scatter of dC = dX W by (starts, paths, ends)
    A = adX @ Wi.abs()
    S["terminal_embedding.weight"] = torch.zeros_like(P["terminal_embedding.weight"]).index_add_(
        0, s.reshape(-1), A[:, :Et]).index_add_(0, e.reshape(-1), A[:, Et + Ep:])
    S["path_embedding.weight"] = torch.zeros_like(P["path_embedding.weight"]).index_add_(0, pth.reshape(-1), A[:, Et:Et + Ep])
    del A, adX
    # LayerNorm affine: d gamma = sum dy * y_hat, d beta = sum dy
    xv = x.reshape(N, H)
    y_hat = (xv - xv.mean(1, keepdim=True)) / torch.sqrt(xv.var(1, unbiased=False, keepdim=True) + 1e-5)
    S["input_layer_norm.weight"] = (dY.reshape(N, H) * y_hat).abs().sum(0)
    S["input_layer_norm.bias"] = dY.reshape(N, H).abs().sum(0)
    del y_hat
    # attention: d a = sum over contexts of (dz * mask) h;  code vector: sum_l att h;  attention: the softmax normaliser
    h = torch.tanh(ln) * mask.double()
    valid = (s > 0).double()
    S["attention_parameter"] = torch.einsum("bl,blh->h", (dz * valid).abs(), h.abs())
    S["cv"] = torch.einsum("bl,blh->bh", r["att"], h.abs())
    S["att"] = r["att"].clone()
    del h
    cv, logits = r["cv"], r["logits"]
    if angular:
        W = P["output_linear"]
        wnorm = W.norm(dim=1, keepdim=True).clamp_min(1e-12)
        wn = W / wnorm
        cvn = F.normalize(cv)
        cos, Gc = r["taps"]["cos"]
        # cos = cvn . wn^T;  dW = (dwn - (dwn . wn) wn) / |w| with dwn = Gc^T cvn
        Ac = Gc.abs().t() @ cvn.abs()
        S["output_linear"] = (Ac + wn.abs() * (Ac * wn.abs()).sum(1, keepdim=True)) / wnorm
        # d cv = (dcvn - (dcvn . cvn) cvn) / |cv| with dcvn = Gc wn
        Ad = Gc.abs() @ wn.abs()
        S["dcv"] = (Ad + cvn.abs() * (Ad * cvn.abs()).sum(1, keepdim=True)) / cv.norm(dim=1, keepdim=True).clamp_min(1e-12)
        del Ac, Ad
        Sl = INV_TEMP * (cvn.abs() @ wn.abs().t())
        # at the label column (cos > 0) the logit is s * phi(cos): phi' = cos m + sin m * cos / sin
        c = cos.gather(1, lab[:, None])
        sin = torch.sqrt((1.0 - c * c).clamp_min(1e-12))
        amp = torch.where(c > 0, math.cos(MARGIN) + math.sin(MARGIN) * c.abs() / sin, torch.ones_like(c))
        Sl.scatter_(1, lab[:, None], Sl.gather(1, lab[:, None]) * amp)
    else:
        G = r["taps"]["logits"][1]
        S["output_linear.weight"] = G.abs().t() @ cv.abs()
        S["output_linear.bias"] = G.abs().sum(0)
        S["dcv"] = G.abs() @ P["output_linear.weight"].abs()
        Sl = cv.abs() @ P["output_linear.weight"].abs().t() + P["output_linear.bias"].abs()
    S["logits"] = Sl
    lse = torch.logsumexp(logits, 1)
    S["loss"] = (lse.abs() + logits.gather(1, lab[:, None])[:, 0].abs()).mean()
    return S


def _rho(a, ref, S, name, zero_violations):
    """max |a - ref| / S over S > 0; where S == 0, `a` must be exactly 0 (recorded in zero_violations)"""
    a = a.double()
    nz = S > 0
    d = (a - ref).abs()
    if not bool(nz.all()):
        bad = int(((a != 0) & ~nz).sum())
        if bad:
            zero_violations.append(f"{name}: {bad} elements nonzero where S = 0")
    if not bool(nz.any()):
        return 0.0
    return float((d[nz] / S[nz]).max())


# ---- the case ----------------------------------------------------------------------------------------------------------
def _ulp32(x):
    _, ex = torch.frexp(x.float())
    return torch.ldexp(torch.ones_like(x, dtype=torch.float64), (ex - 24).double())


def _check_adam(snap, new_p, new_m, new_v, step_t):
    """fp64 Adam (torch.optim.Adam's update, main.py:138) from what the kernel read; the hyperparameters are the fp32
    values the kernel receives"""
    b1, b2 = float(np.float32(BETAS[0])), float(np.float32(BETAS[1]))
    lr, eps = float(np.float32(LR)), float(np.float32(EPS))
    g, p, m, v = (snap[k].double() for k in ("g", "p", "m", "v"))
    m64 = m + (g - m) * (1.0 - b1)
    v64 = v * b2 + (1.0 - b2) * g * g
    bc1, bc2 = 1.0 - b1 ** step_t, 1.0 - b2 ** step_t
    p64 = p - (lr / bc1) * m64 / (torch.sqrt(v64) / math.sqrt(bc2) + eps)
    msgs = {}
    ep = (new_p.double() - p64).abs() - (2.0 * _ulp32(p64) + lr * FLOOR)
    em = (new_m.double() - m64).abs() - (4.0 * F32_EPS * (m.abs() + g.abs()) + 2.0 ** -146)
    ev = (new_v.double() - v64).abs() - (4.0 * F32_EPS * (v * b2 + (1.0 - b2) * g * g) + 2.0 ** -146)
    for name, ex in (("param", ep), ("exp_avg", em), ("exp_avg_sq", ev)):
        n_bad = int((ex > 0).sum())
        if n_bad:
            i = int(ex.argmax())
            msgs[name] = f"{n_bad} elements off, worst at flat index {i}"
    return msgs


def _run_case(case):
    wname, data, fused, angular = CASES[case]
    w = dict(WORKLOADS[wname])
    dev = torch.device("cuda:0")
    t0 = time.perf_counter()
    torch.manual_seed(0)
    m = _model(w, dev, angular)
    opt = ShardedFlatAdam(m.parameters(), lr=LR, betas=BETAS)
    assert opt.world == 1
    names = [n for n, _ in m.named_parameters()]
    assert [id(p) for p in opt.params] == [id(p) for p in m.parameters()]
    offs, o = {}, 0
    for n, p in m.named_parameters():
        offs[n] = (o, p.shape)
        o += p.numel()
    numel = o

    seeds, captured, snap = [], {}, {}
    next_seed = m._next_seed

    def record_seed():
        sd = next_seed()
        seeds.append(sd)
        return sd
    m._next_seed = record_seed
    if fused:
        forward_loss = m.forward_loss

        def capture_fl(*a):
            res = forward_loss(*a)
            captured.update(loss=res[0].detach().clone(), am=res[1].clone(), mx=res[2].clone(),
                            cv=res[3].detach().clone(), att=res[4].detach().clone())
            res[3].register_hook(lambda g: captured.__setitem__("dcv", g.detach().clone()))   # the label head's d cv
            return res
        m.forward_loss = capture_fl
        loss_fn = None
    else:
        forward = m.forward

        def capture_fw(*a):
            res = forward(*a)
            captured.update(logits=res[0].detach().clone(), cv=res[1].detach().clone(), att=res[2].detach().clone())
            res[1].register_hook(lambda g: captured.__setitem__("dcv", g.detach().clone()))
            return res
        m.forward = capture_fw

        def loss_fn(o_, l_):                                # bench.py --train-unfused-loss
            return F.nll_loss(F.log_softmax(o_, dim=1), l_)
    opt_step = opt.step

    def snap_step():
        snap.update(g=opt.bucket.clone(), p=opt.flat_param.clone(), m=opt.exp_avg.clone(), v=opt.exp_avg_sq.clone(),
                    t=opt.t + 1, bucket=opt.bucket)
        opt_step()
    opt.step = snap_step

    report, failures = {}, []

    def note(step, name, rk, r32):
        factor = LOOSER.get(case, {}).get(name, FACTOR)
        if isinstance(factor, tuple):
            factor = factor[0] if step >= factor[1] else FACTOR
        bound = max(factor * r32, FLOOR)
        prev = report.get(name)
        ratio = rk / r32 if r32 > 0 else (0.0 if rk == 0 else math.inf)
        if prev is None or ratio > prev["ratio"]:
            report[name] = {"ratio": ratio, "rho": rk, "rho32": r32, "step": step}
        if not rk <= bound:
            failures.append(f"step {step} {name}: max rho {rk:.3g} > bound {bound:.3g} (fp32 torch {r32:.3g})")

    for step, batch in enumerate(_batches(w, data, dev)):
        s, pth, e, lab = batch
        B, L = s.shape
        H = w["H"]
        loss_k = ddp_step(m, opt, None, s, pth, e, lab, loss_fn).detach().clone()
        torch.cuda.synchronize()
        assert len(seeds) == step + 1
        mask = torch.from_numpy(dropout_mask(seeds[-1], B * L, H, DROPOUT).reshape(B, L, H)).to(dev)
        params = {n: snap["p"][o:o + math.prod(sh)].view(sh) for n, (o, sh) in offs.items()}
        g_k = {n: snap["g"][o:o + math.prod(sh)].view(sh) for n, (o, sh) in offs.items()}
        # the gradient never lands in the padding; the step leaves the whole bucket zeroed
        assert bool((snap["g"][numel:] == 0).all())
        bucket = snap.pop("bucket")
        if not bool((bucket == 0).all()):
            failures.append(f"step {step}: {int((bucket != 0).sum())} gradient elements not zeroed by the Adam step")
        for k, msg in _check_adam(snap, opt.flat_param, opt.exp_avg, opt.exp_avg_sq, snap["t"]).items():
            failures.append(f"step {step} Adam {k}: {msg}")

        r32 = _reference(params, batch, mask, angular, torch.float32)
        r32 = {"loss": r32["loss"], "logits": r32["logits"], "cv": r32["cv"], "att": r32["att"], "grads": r32["grads"],
               "dcv": r32["taps"]["cv"][1]}
        torch.cuda.empty_cache()
        r64 = _reference(params, batch, mask, angular, torch.float64)
        S = _scales(r64, batch, mask, angular)
        dxm = r64["taps"]["x"][1].abs().amax(-1).reshape(-1)
        G = (r64["taps"]["cos"] if angular else r64["taps"]["logits"])[1].abs()
        spread = {"dx_range_log2": math.log2(float(dxm.max() / dxm[dxm > 0].min())),
                  "g_range_log2": math.log2(float(G.max() / G[G > 0].min()))}
        for k, v in spread.items():
            report[k] = max(report.get(k, 0.0), v)
        zv = []
        # stage by stage: code vector and attention, the logits / loss / prediction, then the gradients
        for name in ("cv", "att"):
            note(step, name, _rho(captured[name], r64[name], S[name], name, zv),
                 _rho(r32[name], r64[name], S[name], name + " (fp32 torch)", []))
        rl32 = _rho(r32["logits"], r64["logits"], S["logits"], "logits (fp32 torch)", [])
        if fused:
            note(step, "loss", _rho(captured["loss"], r64["loss"], S["loss"], "loss", zv),
                 _rho(r32["loss"], r64["loss"], S["loss"], "", []))
            lg = r64["logits"]
            mx64, am64 = lg.max(1)
            am = captured["am"]
            b = torch.arange(B, device=dev)
            Sk, S64 = S["logits"][b, am], S["logits"][b, am64]
            # pred_score: the rho rule on the row's maximum; pred_label: an fp64 maximum up to the same bound on both logits
            note(step, "pred_score", float(((captured["mx"].double() - mx64).abs() / S64).max()), rl32)
            slack = max(FACTOR * rl32, FLOOR) * (Sk + S64)
            n_wrong = int((lg[b, am] < mx64 - slack).sum())
            if n_wrong:
                failures.append(f"step {step}: {n_wrong} rows whose pred_label is not an fp64 maximum")
        else:
            note(step, "logits", _rho(captured["logits"], r64["logits"], S["logits"], "logits", zv), rl32)
            note(step, "loss", _rho(loss_k, r64["loss"], S["loss"], "loss", zv),
                 _rho(r32["loss"], r64["loss"], S["loss"], "", []))
        note(step, "dcv", _rho(captured["dcv"], r64["taps"]["cv"][1], S["dcv"], "dcv", zv),
             _rho(r32["dcv"], r64["taps"]["cv"][1], S["dcv"], "", []))
        for name in names:
            note(step, name, _rho(g_k[name], r64["grads"][name], S[name], name, zv),
                 _rho(r32["grads"][name], r64["grads"][name], S[name], "", []))
        failures += [f"step {step} {v}" for v in zv]
        del r32, r64, S, mask, params, g_k
        snap.clear()
        captured.clear()
        torch.cuda.empty_cache()
    report["_wall_s"] = time.perf_counter() - t0
    del m, opt
    torch.cuda.empty_cache()
    return report, failures


@pytest.mark.parametrize("case", list(CASES))
def test_training_step_matches_fp64_reference(case):
    report, failures = _run_case(case)
    # per tensor: the worst ratio max rho(kernel) / max rho(fp32 torch) over the steps
    print(f"\n[train-step {case}] " + json.dumps(report, default=float))
    assert not failures, "\n".join(failures)

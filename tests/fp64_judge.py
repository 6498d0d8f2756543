"""The fp64 judge of the -m gpu parity tests: a scale-free per-element error measure against an fp64 restatement.

reference(): oracle.torch_forward + mean NLL with torch autograd, in the dtype asked for (fp64: the judge; fp32 with TF32
off: the plain-precision baseline), on a given dropout mask.  scales(): for every checked quantity S, the last sum or
contraction that produces it, evaluated in fp64 on absolute values (e.g. |dX|^T |C| for input_linear, the scatter of
|dX| |W| for the embedding tables).  rho(): max |g - g64| / S over S > 0, and exact zeros where S = 0.
"""
import math

import torch
import torch.nn.functional as F

from oracle import oracle


def reference(params, batch, mask, angular, dtype, margin=0.5, inverse_temp=30.0):
    """oracle.torch_forward + mean NLL in `dtype` with autograd -> dict of everything the checks read"""
    s, pth, e, lab = batch
    p = {k: v.detach().to(dtype).requires_grad_() for k, v in params.items()}
    taps = {}
    ang = {"margin": margin, "inverse_temp": inverse_temp} if angular else None
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


def scales(r, batch, mask, angular, margin=0.5, inverse_temp=30.0):
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
        Sl = inverse_temp * (cvn.abs() @ wn.abs().t())
        # at the label column (cos > 0) the logit is s * phi(cos): phi' = cos m + sin m * cos / sin
        c = cos.gather(1, lab[:, None])
        sin = torch.sqrt((1.0 - c * c).clamp_min(1e-12))
        amp = torch.where(c > 0, math.cos(margin) + math.sin(margin) * c.abs() / sin, torch.ones_like(c))
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


def rho(a, ref, S, name, zero_violations):
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

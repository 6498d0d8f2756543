"""-m gpu: the fused loss with a criterion (class weights, ignore_index, label smoothing, reduction) against fp64 torch
on the same logits: F.cross_entropy, or F.nll_loss(F.log_softmax) for NLLLoss.  Both heads, the tensor-core kernels
(c2v_*_opts), the CUDA-core fallback (c2v_loss_argmax_opts), PackedBags, ddp_step and GraphedTrainStep."""
import contextlib
import math

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from fp64_judge import rho
from gpu_util import cuda, option_from, random_batch, random_params
from code2vec_b200 import _lib
from code2vec_b200 import functional as CF
from code2vec_b200.distributed import ShardedFlatAdam, ddp_step
from code2vec_b200.graphs import GraphedTrainStep
from code2vec_b200.model import Code2Vec, _LabelLossFn, _LabelLossOptsFn, _LossArgmaxOptsFn

pytestmark = pytest.mark.gpu

MARGIN, S = 0.5, 30.0
FACTOR, FLOOR = 8.0, 2.0 ** -20


@contextlib.contextmanager
def _no_tf32():
    saved = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = saved


def _case(rng, B, C, H, scale=1.0):
    cv = (rng.standard_normal((B, H)) * 0.5).astype(np.float32)
    W = (rng.uniform(-1, 1, (C, H)) / np.sqrt(H) * scale).astype(np.float32)
    b = (0.05 * rng.standard_normal(C)).astype(np.float32)
    lab = rng.integers(0, C, B).astype(np.int64)
    return cuda(cv), cuda(W), cuda(b), cuda(lab)


def _weight(kind, C, rng):
    if kind == "none":
        return None
    w = rng.uniform(0.25, 2.0, C).astype(np.float32)
    if kind == "zeros":
        w[rng.random(C) < 0.3] = 0.0
        w[0] = 0.0
    return cuda(w)


def _criterion(cls, weight, ii, eps, reduction):
    if cls is nn.NLLLoss:
        return nn.NLLLoss(weight=weight, ignore_index=ii, reduction=reduction)
    return nn.CrossEntropyLoss(weight=weight, ignore_index=ii, reduction=reduction, label_smoothing=eps)


def logits(cv, W, b, lab, angular, taps=None):
    """the head's logits in cv's dtype: cv . W^T + b, or the angular-margin logits (model.py:71-80; no margin at a label
    outside [0, C))"""
    if not angular:
        return cv @ W.t() + b
    cos = F.normalize(cv) @ F.normalize(W).t()
    if taps is not None:
        cos.retain_grad()
        taps["cos"] = cos
    ok = (lab >= 0) & (lab < W.shape[0])
    li = torch.where(ok, lab, torch.zeros_like(lab))
    c = cos.gather(1, li[:, None])
    phi = torch.where(c > 0, c * math.cos(MARGIN) - torch.sqrt((1.0 - c * c).clamp_min(0.0)) * math.sin(MARGIN), c)
    hit = F.one_hot(li, W.shape[0]).bool() & ok[:, None]
    return S * torch.where(hit, phi.expand_as(cos), cos)


def criterion_loss(crit, z, lab):
    """the criterion on logits z, with its weight in z's dtype"""
    c = type(crit)(**{k: getattr(crit, k) for k in ("ignore_index", "reduction")},
                   **({"label_smoothing": crit.label_smoothing} if isinstance(crit, nn.CrossEntropyLoss) else {}),
                   weight=None if crit.weight is None else crit.weight.to(z.dtype))
    return c(F.log_softmax(z, dim=1) if type(crit) is nn.NLLLoss else z, lab)


def _den(crit, lab, C):
    ok = lab != crit.ignore_index
    w = crit.weight.double() if crit.weight is not None else torch.ones(C, dtype=torch.float64, device=lab.device)
    return float(w[lab[ok]].sum())


def _fused(cv, W, b, lab, crit, angular):
    """the fused loss with autograd (the module's _LabelLossOptsFn) -> (loss, argmax, maxval)"""
    C, H = W.shape
    dims = CF.make_dims(10, 10, C, H, H, H)
    c = CF.LossCriterion(crit, C, cv.device)
    cache = CF.PrepCache()
    return _LabelLossOptsFn.apply(cv, W, None if angular else b, lab, dims, _lib.ALGO_AUTO, cache,
                                  (MARGIN, S) if angular else None, c)


def _upstream(crit, loss, lab, C):
    """unit scale: d loss = 1 for the mean, 1 / den (of every row, for none) for sum and none"""
    if crit.reduction == "mean":
        return torch.ones_like(loss)
    den = _den(crit, lab, C)
    return torch.full_like(loss, 1.0 / den if den > 0 else 1.0)


def check(cv, W, b, lab, crit, angular, grad_tol=1e-7, looser=None):
    """loss and d loss / d logits of the fused path against fp64 torch on the same logits, and the gradients of
    code_vector / W_out / b against fp64 autograd with fp64_judge's criterion (looser: {tensor: factor} instead of
    FACTOR)"""
    C = W.shape[0]
    cv_, W_, b_ = (t.detach().clone().requires_grad_() for t in (cv, W, b))
    loss, am, mx = _fused(cv_, W_, b_, lab, crit, angular)
    r = {k: t.detach().double().requires_grad_() for k, t in (("cv", cv), ("W", W), ("b", b))}
    taps = {}
    z64 = logits(r["cv"], r["W"], r["b"], lab, angular, taps)
    z64.retain_grad()
    ref = criterion_loss(crit, z64, lab)
    up = _upstream(crit, loss, lab, C)
    ref.backward(up.double())
    got, want = loss.detach().double().cpu(), ref.detach().cpu()
    assert got.shape == want.shape
    if got.numel() == 1 and torch.isnan(want):
        assert torch.isnan(got)
    else:
        assert ((got - want).abs() <= 2e-5 * want.abs().clamp_min(1.0)).all(), (got, want)
    # fp32 torch on the same inputs: the precision baseline of the parameter gradients
    r32 = {k: t.detach().clone().requires_grad_() for k, t in (("cv", cv), ("W", W), ("b", b))}
    with _no_tf32():
        criterion_loss(crit, logits(r32["cv"], r32["W"], r32["b"], lab, angular), lab).backward(up)
    loss.backward(up)
    # d loss / d logits: what the dlogits kernel wrote, recomputed here through the same call (plain head)
    G = z64.grad
    if not angular:
        dims = CF.make_dims(10, 10, C, W.shape[1], W.shape[1], W.shape[1])
        params = CF.make_params(w_out=W, b_out=b)
        c = CF.LossCriterion(crit, C, cv.device)
        _, lse, _, _, coef, _ = CF.label_loss_opts(dims, params, cv, lab, c)
        g = CF.label_dlogits_opts(dims, params, cv, lab, lse, coef, c, up)
        assert (g.double() - G).abs().max().item() <= grad_tol, (g.double() - G).abs().max().item()
    aG, acv = G.abs(), r["cv"].detach().abs()
    if angular:                                                      # fp64_judge.scales, through F.normalize
        Gc, cv64, W64 = taps["cos"].grad.abs(), r["cv"].detach(), r["W"].detach()
        cvn, wn = F.normalize(cv64).abs(), F.normalize(W64).abs()
        Ad, Ac = Gc @ wn, Gc.t() @ cvn
        S_cv = (Ad + cvn * (Ad * cvn).sum(1, keepdim=True)) / cv64.norm(dim=1, keepdim=True).clamp_min(1e-12)
        S_W = (Ac + wn * (Ac * wn).sum(1, keepdim=True)) / W64.norm(dim=1, keepdim=True).clamp_min(1e-12)
        pairs = (("cv", cv_.grad, S_cv), ("W", W_.grad, S_W))
    else:
        pairs = (("cv", cv_.grad, aG @ r["W"].detach().abs()), ("W", W_.grad, aG.t() @ acv), ("b", b_.grad, aG.sum(0)))
    zv = []
    for k, g, Sk in pairs:
        rk = rho(g, r[k].grad, Sk, k, zv)
        r32k = rho(r32[k].grad, r[k].grad, Sk, "", [])
        assert rk <= max((looser or {}).get(k, FACTOR) * r32k, FLOOR), (k, rk, r32k)
    assert not zv, zv


REDUCTIONS = ["mean", "sum", "none"]


@pytest.mark.parametrize("angular", [False, True])
@pytest.mark.parametrize("wkind", ["none", "positive", "zeros"])
@pytest.mark.parametrize("ii", ["-100", "class"])
@pytest.mark.parametrize("eps", [0.0, 0.1, 1.0])
@pytest.mark.parametrize("reduction", REDUCTIONS)
def test_criterion_grid(angular, wkind, ii, eps, reduction):
    rng = np.random.default_rng([int(angular), ["none", "positive", "zeros"].index(wkind), int(ii == "class"), int(eps * 10),
                                 REDUCTIONS.index(reduction)])
    B, C, H = 130, 1000, 128
    cv, W, b, lab = _case(rng, B, C, H, 4.0)
    lab[3] = C - 1
    w = _weight(wkind, C, rng)
    if ii == "-100":
        lab[::7] = -100
        ignore = -100
    else:
        ignore = int(lab[5])                                     # a valid class, present in the labels
    check(cv, W, b, lab, _criterion(nn.CrossEntropyLoss, w, ignore, eps, reduction), angular)
    if eps == 0.0:
        check(cv, W, b, lab, _criterion(nn.NLLLoss, w, ignore, eps, reduction), angular)


@pytest.mark.parametrize("B,C,H,scale", [(7, 11, 128, 1.0), (64, 4097, 100, 4.0), (33, 260, 256, 2.0),
                                          (1024, 8192, 128, 6.0), (5, 3, 4, 1.0)])
@pytest.mark.parametrize("angular", [False, True])
@pytest.mark.parametrize("reduction", REDUCTIONS)
def test_shapes(B, C, H, scale, angular, reduction):
    rng = np.random.default_rng(B * 31 + C)
    cv, W, b, lab = _case(rng, B, C, H, scale)
    lab[0] = -100
    # angular head at H = 4, C = 3: d code_vector measured at 18x fp32 torch's rho on one H100 80GB HBM3 (700 W), the
    # same for every reduction; the cause is not isolated here
    looser = {"cv": 32.0} if angular and H == 4 else None
    check(cv, W, b, lab, _criterion(nn.CrossEntropyLoss, _weight("positive", C, rng), -100, 0.1, reduction), angular,
          looser=looser)


@pytest.mark.parametrize("angular", [False, True])
def test_top11_label_count(angular):
    """C = 195,299 (top11_dataset's label vocabulary) at H = 100.  The W_out gradient needs more than FACTOR: the smoothing
    term puts ~eps / (C den) into every d logit, ~2^-21 of max |G|, and in the label backward's fp16 hi / lo split of G
    (one power-of-two scale for the whole matrix) the lo part of such an entry is an fp16 subnormal -- the deficit
    test_value_range_gpu.py lists for small operands.  Measured on one H100 80GB HBM3 (700 W): 24x fp32 torch's rho."""
    rng = np.random.default_rng(11)
    cv, W, b, lab = _case(rng, 200, 195299, 100, 5.0)
    lab[::9] = -100
    check(cv, W, b, lab, _criterion(nn.CrossEntropyLoss, _weight("zeros", 195299, rng), -100, 0.1, "mean"), angular,
          looser={"W": 32.0})


@pytest.mark.parametrize("angular", [False, True])
def test_every_row_ignored(angular):
    rng = np.random.default_rng(3)
    cv, W, b, lab = _case(rng, 40, 300, 128)
    lab[:] = -100
    for reduction, want in (("mean", math.nan), ("sum", 0.0)):
        cv_, W_, b_ = (t.clone().requires_grad_() for t in (cv, W, b))
        crit = nn.CrossEntropyLoss(weight=_weight("positive", 300, rng), reduction=reduction, label_smoothing=0.1)
        loss = _fused(cv_, W_, b_, lab, crit, angular)[0]
        assert (math.isnan(loss.item()) if math.isnan(want) else loss.item() == want), (reduction, loss.item())
        loss.backward()
        for g in (cv_.grad, W_.grad) + (() if angular else (b_.grad,)):
            assert g is not None and not g.any(), reduction


def test_a_bias_offset_keeps_the_smoothing_term_accurate():
    """logits sharing an offset of 2^10: the smoothing term sum_j w_j (lse - z_j) (eps = 1 isolates it) stays within 8x of
    fp32 torch's error against fp64 -- W lse - sum_j w_j z_j would lose most of its bits"""
    rng = np.random.default_rng(5)
    B, C, H = 256, 20000, 128
    cv, W, b, lab = _case(rng, B, C, H, 4.0)
    b = b + 2.0 ** 10
    for eps in (1.0, 0.1):
        crit = nn.CrossEntropyLoss(weight=_weight("positive", C, rng), label_smoothing=eps)
        with torch.no_grad():
            got = _fused(cv, W, b, lab, crit, False)[0].double().item()
            ref = criterion_loss(crit, logits(cv.double(), W.double(), b.double(), lab, False), lab).item()
            with _no_tf32():
                r32 = criterion_loss(crit, logits(cv, W, b, lab, False), lab).double().item()
        err, err32 = abs(got - ref), abs(r32 - ref)
        assert err <= max(FACTOR * err32, FLOOR * abs(ref)), (eps, err, err32)


@pytest.mark.parametrize("angular", [False, True])
def test_a_default_criterion_gives_the_bits_of_no_criterion(angular):
    rng = np.random.default_rng(9)
    B, C, H = 300, 5000, 128
    cv, W, b, lab = _case(rng, B, C, H, 4.0)
    dims = CF.make_dims(10, 10, C, H, H, H)
    for det in (False, True):
        torch.use_deterministic_algorithms(det, warn_only=True)
        try:
            res = []
            for crit in (None, nn.CrossEntropyLoss(), nn.NLLLoss()):
                cv_, W_, b_ = (t.clone().requires_grad_() for t in (cv, W, b))
                args = (cv_, W_, None if angular else b_, lab, dims, _lib.ALGO_AUTO, CF.PrepCache(),
                        (MARGIN, S) if angular else None)
                if crit is None:
                    loss, am, mx = _LabelLossFn.apply(*args)
                else:
                    loss, am, mx = _LabelLossOptsFn.apply(*args, CF.LossCriterion(crit, C, cv.device))
                loss.backward()
                res.append((loss.detach(), am, mx, cv_.grad, W_.grad) + (() if angular else (b_.grad,)))
            for other in res[1:]:
                for i, (x, y) in enumerate(zip(res[0], other)):
                    if i == 3 and not det:           # d code_vector: a split-K sum through atomics outside deterministic mode
                        torch.testing.assert_close(x, y, rtol=1e-5, atol=1e-7)
                    else:
                        assert torch.equal(x, y), (det, i)
        finally:
            torch.use_deterministic_algorithms(False)


def test_cuda_core_path_against_fp64():
    """c2v_loss_argmax_opts (forward_loss's fallback under torch.use_deterministic_algorithms) on materialised logits"""
    rng = np.random.default_rng(12)
    B, C = 96, 3001
    z = cuda((rng.standard_normal((B, C)) * 3).astype(np.float32))
    lab = cuda(rng.integers(0, C, B).astype(np.int64))
    lab[::5] = 7
    for reduction in REDUCTIONS:
        for eps in (0.0, 0.1, 1.0):
            for cls in (nn.CrossEntropyLoss, nn.NLLLoss):
                crit = _criterion(cls, _weight("zeros", C, rng), 7, eps, reduction)
                z_ = z.clone().requires_grad_()
                loss = _LossArgmaxOptsFn.apply(z_, lab, CF.LossCriterion(crit, C, z.device))[0]
                z64 = z.double().requires_grad_()
                ref = criterion_loss(crit, z64, lab)
                up = _upstream(crit, loss, lab, C)
                loss.backward(up)
                ref.backward(up.double())
                assert ((loss.double() - ref).abs() <= 2e-5 * ref.abs().clamp_min(1.0)).all()
                assert (z_.grad.double() - z64.grad).abs().max().item() <= 1e-7


def _model(angular=False, algo="auto", C=57, H=128, seed=0):
    o = {"T": 300, "P": 200, "C": C, "Et": H, "Ep": H, "H": H, "angular": int(angular)}
    m = Code2Vec(option_from(o), algo=algo)
    params = random_params(np.random.default_rng(seed), 300, 200, C, H, H, H)
    if angular:
        params.pop("output_linear.bias")
        params["output_linear"] = params.pop("output_linear.weight")
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    return m.to("cuda:0").eval()


@pytest.mark.parametrize("algo", ["ffma", "auto"])
@pytest.mark.parametrize("angular", [False, True])
def test_fallbacks_and_deterministic_mode(algo, angular):
    """forward_loss with a criterion on the CUDA-core head (algo="ffma": the criterion itself; deterministic: the library)
    and on the fused path, against fp64 on forward()'s logits; in deterministic mode two runs give identical bits"""
    C = 57
    m = _model(angular, algo, C)
    s, p, e, lab = (cuda(a) for a in random_batch(np.random.default_rng(2), 48, 20, 300, 200, C))
    lab[::6] = 4
    crit = nn.CrossEntropyLoss(weight=_weight("zeros", C, np.random.default_rng(4)), ignore_index=4, label_smoothing=0.1,
                               reduction="sum")
    with torch.no_grad():
        z = m(s, p, e, lab)[0]
    ref = criterion_loss(crit, z.double(), lab).item()
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        runs = []
        for _ in range(2):
            m.zero_grad(set_to_none=True)
            loss = m.forward_loss(s, p, e, lab, criterion=crit)[0]
            loss.backward()
            runs.append([loss.detach()] + [q.grad.clone() for q in m.parameters()])
        for x, y in zip(*runs):
            assert torch.equal(x, y)
    finally:
        torch.use_deterministic_algorithms(False)
    assert abs(runs[0][0].item() - ref) <= 2e-5 * max(1.0, abs(ref))
    loss = m.forward_loss(s, p, e, lab, criterion=crit)[0]
    assert abs(loss.item() - ref) <= 2e-5 * max(1.0, abs(ref))


def test_packed_bags():
    C, L = 57, 20
    m = _model(False, "auto", C)
    s, p, e, lab = (cuda(a) for a in random_batch(np.random.default_rng(6), 40, L, 300, 200, C))
    lab[::4] = -100
    n = (s > 0).sum(1).clamp(min=1).cpu().numpy()
    off = np.concatenate([[0], np.cumsum(n)])
    keep = torch.arange(L, device="cuda:0")[None, :] < torch.from_numpy(n).to("cuda:0")[:, None]
    bags = CF.PackedBags(s[keep], p[keep], e[keep], off, L)
    crit = nn.CrossEntropyLoss(weight=_weight("positive", C, np.random.default_rng(1)), label_smoothing=0.1)
    lp = m.forward_loss(bags, None, None, lab, criterion=crit)[0]
    ld = m.forward_loss(s, p, e, lab, criterion=crit)[0]
    with torch.no_grad():
        ref = criterion_loss(crit, m(s, p, e, lab)[0].double(), lab).item()
    assert abs(lp.item() - ref) <= 2e-5 * max(1.0, abs(ref)) and abs(ld.item() - ref) <= 2e-5 * max(1.0, abs(ref))


def test_ddp_step_sharded_adam_against_torch_adam():
    C, L = 57, 20
    crit = nn.CrossEntropyLoss(weight=_weight("positive", C, np.random.default_rng(8)), label_smoothing=0.1)
    m, ref = _model(False, "auto", C).train(), _model(False, "auto", C).train()
    opt = ShardedFlatAdam(m.parameters(), lr=1e-3)
    ref_opt = torch.optim.Adam(ref.parameters(), lr=1e-3)
    rng = np.random.default_rng(9)
    for _ in range(3):
        s, p, e, lab = (cuda(a) for a in random_batch(rng, 32, L, 300, 200, C))
        loss = ddp_step(m, opt, None, s, p, e, lab, None, criterion=crit)
        ref_opt.zero_grad()
        rl = crit(ref(s, p, e, lab)[0], lab)
        rl.backward()
        ref_opt.step()
        assert abs(loss.item() - rl.item()) <= 1e-4 * max(1.0, abs(rl.item())), (loss.item(), rl.item())
    for (k, a), b in zip(m.named_parameters(), ref.parameters()):
        close = ((a - b).abs() <= 1e-5 + 1e-4 * b.abs()).float().mean().item()
        assert close >= 0.999, (k, close)


@pytest.mark.parametrize("angular", [False, True])
def test_graphed_train_step_with_a_criterion(angular):
    """test_graphs_gpu's reference loop (25 steps, batch 32, ragged last batch) with a weighted, smoothed criterion"""
    from oracle import oracle
    from test_graphs_gpu import _items, _model as graphs_model
    E = H = 128
    T, P, C, L, n, bs = 300, 200, 17, 40, 150, 32
    rng = np.random.default_rng(E)
    data = _items(rng, n, L, T, P, C)
    m, params = graphs_model(dict(Et=E, Ep=E, H=H), T, P, C, angular=angular)
    m.train()
    w = torch.from_numpy(np.random.default_rng(2).uniform(0.5, 2.0, C).astype(np.float32))
    crit = nn.CrossEntropyLoss(weight=w.to("cuda:0"), label_smoothing=0.1)
    ref_crit = nn.CrossEntropyLoss(weight=w, label_smoothing=0.1)
    opt = torch.optim.Adam(m.parameters(), lr=0.01, capturable=True)
    step = GraphedTrainStep(m, opt, bs, L, criterion=crit)
    ang = {"margin": 0.5, "inverse_temp": 30.0} if angular else None
    ref = {k: torch.from_numpy(v).clone().requires_grad_(True) for k, v in params.items()}
    ref_opt = torch.optim.Adam(list(ref.values()), lr=0.01)
    losses, ref_losses = [], []
    for epoch in range(5):
        perm = torch.randperm(n, generator=torch.Generator().manual_seed(epoch))
        for i in range(0, n, bs):
            batch = [t[perm[i:i + bs]] for t in data]
            losses.append(step(*(t.to("cuda:0") for t in batch)))
            ref_opt.zero_grad()
            rl = ref_crit(oracle.torch_forward(ref, *batch, angular=ang)[0], batch[3])
            rl.backward()
            ref_opt.step()
            ref_losses.append(rl.item())
    losses = [float(x) for x in losses]
    assert len(losses) == 25 and step.graph is not None
    assert np.abs(np.array(losses[:5]) - np.array(ref_losses[:5])).max() <= 2e-4, (losses[:5], ref_losses[:5])
    assert np.abs(np.array(losses) - np.array(ref_losses)).max() <= 2e-2, (losses, ref_losses)

"""-m gpu: the angular-margin head (model.py:71-80) fused into the tensor-core label GEMM -- c2v_angular_loss_argmax /
c2v_angular_dlogits / c2v_angular_backward_ws and Code2Vec.forward_loss on an angular model -- against fp64 torch
restatements, the reference's own gradients (tests/golden/angular_grad*.npz) and the CUDA-core angular path."""
import math
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import load_golden
from gpu_util import cuda, model_from_golden, random_batch, random_params
from code2vec_b200 import functional as CF
from code2vec_b200.model import Code2Vec

pytestmark = pytest.mark.gpu

MARGIN, S = 0.5, 30.0


def _case(rng, B, C, H, scale=1.0):
    """cv, W, label with the first and last columns as targets; a third of the rows point towards their target
    (cos > 0: phi's margin branch), a third away from it (cos <= 0: phi(c) = c)"""
    W = (rng.uniform(-1, 1, (C, H)) / np.sqrt(H) * scale).astype(np.float32)
    cv = rng.standard_normal((B, H)) * 0.5
    lab = rng.integers(0, C, B).astype(np.int64)
    lab[0] = C - 1; lab[-1] = 0
    for b in range(B):
        w = W[lab[b]].astype(np.float64)
        w = w / max(np.linalg.norm(w), 1e-12)
        if b % 3 == 0:
            cv[b] = 0.3 * cv[b] + 1.5 * w
        elif b % 3 == 1:
            cv[b] = 0.3 * cv[b] - 1.5 * w
    return cv.astype(np.float32), W, lab


def _ref_logits(cv, W, lab, margin=MARGIN, s=S):
    """oracle.torch_forward's angular branch in fp64 (on the device: C reaches 195,299)"""
    cos = F.linear(F.normalize(cv), F.normalize(W))
    sin = torch.sqrt(1.0 - cos * cos)
    phi = torch.where(cos > 0, cos * math.cos(margin) - sin * math.sin(margin), cos)
    oh = torch.zeros_like(cos).scatter_(1, lab.view(-1, 1), 1)
    return (oh * phi + (1.0 - oh) * cos) * s, cos


def _d64(a):
    return cuda(a).double()


def _dims(C, H):
    return CF.make_dims(10, 10, C, H, H, H)


def _params(W):
    return CF.make_params(None, None, None, None, None, None, W, None)


GRID = [(7, 11, 128, 1.0), (130, 1000, 128, 8.0), (64, 4097, 100, 4.0), (33, 260, 256, 2.0), (1024, 8192, 128, 6.0),
        (5, 3, 4, 1.0)]


@pytest.mark.parametrize("B,C,H,scale", GRID)
@pytest.mark.parametrize("want_logits", [False, True])
def test_angular_loss_matches_fp64(B, C, H, scale, want_logits):
    rng = np.random.default_rng(B * 31 + C)
    cv, W, lab = _case(rng, B, C, H, scale)
    dims, w_t = _dims(C, H), cuda(W)
    params = _params(w_t)
    assert CF.label_loss_supported(dims, B)
    loss, lse, am, mx, inv, out = CF.angular_loss(dims, params, cuda(cv), cuda(lab), MARGIN, S, want_logits=want_logits)
    ref_out, ref_cos = _ref_logits(_d64(cv), _d64(W), cuda(lab))
    tcos = ref_cos.gather(1, cuda(lab).view(-1, 1)).view(-1)
    assert bool((tcos > 0).any()) and bool((tcos <= 0).any())            # both branches of phi
    ref_loss = F.nll_loss(F.log_softmax(ref_out, 1), cuda(lab)).item()
    ref_lse = torch.logsumexp(ref_out, 1)
    ref_mx = ref_out.max(1).values
    assert abs(loss.item() - ref_loss) <= 2e-5 * max(1.0, abs(ref_loss)), (loss.item(), ref_loss)
    assert (lse.double() - ref_lse).abs().max().item() <= 2e-5 * max(1.0, ref_lse.abs().max().item())
    assert (mx.double() - ref_mx).abs().max().item() <= 1e-4
    picked = ref_out.gather(1, am.view(-1, 1)).view(-1)                 # ties / near-ties: the pick must be a maximum
    assert bool((picked >= ref_mx - 1e-4).all())
    ref_inv = 1.0 / torch.cat((_d64(cv).norm(dim=1), _d64(W).norm(dim=1))).clamp_min(1e-12)
    assert ((inv.double() - ref_inv).abs() / ref_inv).max().item() <= 1e-6
    if want_logits:
        lab_d = cuda(lab)
        cc = CF.angular_logits(dims, params, cuda(cv), lab_d, MARGIN, S)            # the CUDA-core head, same inputs
        assert (out - cc).abs().max().item() <= 3e-6 * max(1.0, cc.abs().max().item())
        assert (out.double() - ref_out).abs().max().item() <= 3e-6 * max(1.0, ref_out.abs().max().item())
    else:
        assert out is None


def _ref_dot_grad(cv64, W64, lab, B):
    """fp64 autograd d(mean NLL)/d(cv . W^T) through the angular head"""
    dot = (cv64 @ W64.T).requires_grad_(True)
    icv = 1.0 / cv64.norm(dim=1).clamp_min(1e-12)
    iw = 1.0 / W64.norm(dim=1).clamp_min(1e-12)
    cos = dot * icv[:, None] * iw[None, :]
    sin = torch.sqrt(1.0 - cos * cos)
    phi = torch.where(cos > 0, cos * math.cos(MARGIN) - sin * math.sin(MARGIN), cos)
    oh = torch.zeros_like(cos).scatter_(1, lab.view(-1, 1), 1)
    out = (oh * phi + (1.0 - oh) * cos) * S
    loss = F.nll_loss(F.log_softmax(out, 1), lab)
    loss.backward()
    return loss.item(), out.detach(), dot.grad


def test_angular_loss_at_the_top11_label_count():
    """C = 195,299 (top11_dataset's label vocabulary): 153 MB of logits at B = 200 that are never written"""
    rng = np.random.default_rng(7)
    B, C, H = 200, 195299, 100
    cv, W, lab = _case(rng, B, C, H, 5.0)
    dims, w_t, lab_d, cv_d = _dims(C, H), cuda(W), cuda(lab), cuda(cv)
    params = _params(w_t)
    loss, lse, am, mx, inv, out = CF.angular_loss(dims, params, cv_d, lab_d, MARGIN, S)
    ref_loss, ref_out, ref_g = _ref_dot_grad(_d64(cv), _d64(W), lab_d, B)
    assert out is None
    assert abs(loss.item() - ref_loss) <= 2e-5 * abs(ref_loss), (loss.item(), ref_loss)
    assert (mx.double() - ref_out.max(1).values).abs().max().item() <= 1e-4
    assert (am == ref_out.argmax(1)).double().mean().item() >= 0.99
    G = CF.angular_dlogits(dims, params, cv_d, lab_d, lse, inv, MARGIN, S, 1.0 / B)
    rows = list(range(8)) + list(range(B - 8, B))
    assert (G[rows].double() - ref_g[rows]).abs().max().item() <= 2e-5 * ref_g[rows].abs().max().item()


BGRID = [(7, 11, 128), (130, 1000, 128), (64, 4097, 100), (33, 260, 256), (1024, 8192, 128), (5, 3, 4)]


@pytest.mark.parametrize("B,C,H", BGRID)
def test_angular_backward_matches_fp64_autograd_and_the_cuda_core_backward(B, C, H):
    rng = np.random.default_rng(B * 7 + C)
    cv, W, lab = _case(rng, B, C, H, 3.0)
    dims, w_t, lab_d, cv_d = _dims(C, H), cuda(W), cuda(lab), cuda(cv)
    params = _params(w_t)
    cache = CF.PrepCache()
    loss, lse, am, mx, inv, _ = CF.angular_loss(dims, params, cv_d, lab_d, MARGIN, S, cache=cache, weight=w_t)
    G = CF.angular_dlogits(dims, params, cv_d, lab_d, lse, inv, MARGIN, S, 1.0 / B, cache=cache, weight=w_t)
    d_cv, d_w = CF.angular_backward_ws(dims, params, cv_d, G, inv, cache=cache, weight=w_t, absmax_ready=True)
    # fp64 autograd through F.normalize (oracle.torch_forward's angular branch)
    cv64, W64 = _d64(cv).requires_grad_(True), _d64(W).requires_grad_(True)
    ref_out, _ = _ref_logits(cv64, W64, lab_d)
    F.nll_loss(F.log_softmax(ref_out, 1), lab_d).backward()
    for got, ref, name in ((d_cv, cv64.grad, "d_cv"), (d_w, W64.grad, "d_w")):
        assert (got.double() - ref).abs().max().item() <= 2e-5 * ref.abs().max().item(), name
    # the existing CUDA-core angular backward on the same inputs
    out, cos, inv2 = CF.angular_forward_train(dims, params, cv_d, lab_d, MARGIN, S)
    _, _, _, d_out = CF.loss_argmax(out, lab_d, want_grad=True)
    d_cv2, d_w2 = CF.angular_backward(dims, params, cv_d, lab_d, MARGIN, S, cos, inv2, d_out)
    for got, ref, name in ((d_cv, d_cv2, "d_cv"), (d_w, d_w2, "d_w")):
        assert (got - ref).abs().max().item() <= 2e-5 * ref.abs().max().item(), name


def _tol(ref):
    return 2e-5 * max(1.0, float(np.abs(ref).max()))


@pytest.mark.parametrize("name", ["angular_grad", "angular_grad128"])
def test_forward_loss_reproduces_the_reference_angular_gradients(name):
    rec = load_golden(name)
    m = model_from_golden(rec).train()
    s, p, e, lab = (cuda(rec[k]) for k in ("starts", "paths", "ends", "label"))
    loss, am, mx, cv, att = m.forward_loss(s, p, e, lab)
    assert abs(loss.item() - float(rec["loss"])) <= 1e-5 * max(1.0, abs(float(rec["loss"])))
    assert np.abs(mx.cpu().numpy() - rec["outputs"].max(1)).max() <= 1e-4
    loss.backward()
    for k, prm in m.named_parameters():
        ref = rec["grads"][k]
        assert np.abs(prm.grad.cpu().numpy() - ref).max() <= _tol(ref), k


def _angular_model(rng, T, P, C, E, H, dropout=0.0, algo="auto"):
    opt = types.SimpleNamespace(terminal_count=T, path_count=P, label_count=C, terminal_embed_size=E, path_embed_size=E,
                                encode_size=H, dropout_prob=dropout, angular_margin_loss=True, angular_margin=MARGIN,
                                inverse_temp=S, device=torch.device("cuda:0"))
    prm = random_params(rng, T, P, C, E, E, H)
    prm["output_linear"] = prm.pop("output_linear.weight")
    del prm["output_linear.bias"]
    m = Code2Vec(opt, algo=algo)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in prm.items()}, strict=True)
    return m.to("cuda:0")


def _both_ways(m, batch, seed=11):
    """forward_loss vs forward + calculate_loss (main.py:251-264) + torch.max on the same batch and dropout seed"""
    s, p, e, lab = (cuda(x) for x in batch)
    res = []
    for fused in (True, False):
        m.zero_grad(set_to_none=True)
        torch.manual_seed(seed)
        if fused:
            loss, am, mx, _, _ = m.forward_loss(s, p, e, lab)
        else:
            out, _, _ = m.forward(s, p, e, lab)
            loss = F.nll_loss(F.log_softmax(out, dim=1), lab)
            mx, am = torch.max(out.detach(), dim=1)
        loss.backward()
        res.append((loss.item(), am.cpu().numpy(), mx.cpu().numpy(),
                    {k: v.grad.cpu().numpy().copy() for k, v in m.named_parameters()}))
    return res


def _assert_same(res, am_frac=1.0):
    (l1, am1, mx1, g1), (l2, am2, mx2, g2) = res
    assert abs(l1 - l2) <= 1e-5 * max(1.0, abs(l2)), (l1, l2)
    assert np.abs(mx1 - mx2).max() <= 1e-4
    assert (am1 == am2).mean() >= am_frac
    for k in g2:
        assert np.abs(g1[k] - g2[k]).max() <= _tol(g2[k]), k


def test_forward_loss_at_a_real_size_matches_forward_plus_calculate_loss():
    rng = np.random.default_rng(5)
    T, P, C, E, H, B, L = 5000, 4000, 8192, 128, 128, 1024, 50
    m = _angular_model(rng, T, P, C, E, H, dropout=0.25).train()
    _assert_same(_both_ways(m, random_batch(rng, B, L, T, P, C)), am_frac=0.99)


@pytest.mark.parametrize("case", ["odd_encode", "big_batch", "ffma"])
def test_forward_loss_fallbacks_match_the_eager_path(case):
    rng = np.random.default_rng(9)
    T, P, C, L = 300, 200, 500, 20
    E, H, B, algo = {"odd_encode": (30, 30, 64, "auto"), "big_batch": (128, 128, 2100, "auto"),
                     "ffma": (128, 128, 64, "ffma")}[case]
    m = _angular_model(rng, T, P, C, E, H, algo=algo).train()
    dims = m._dims()
    if case != "ffma":
        assert not CF.label_loss_supported(dims, B)
    _assert_same(_both_ways(m, random_batch(rng, B, L, T, P, C)))


def test_an_out_of_range_label_makes_the_angular_loss_nan():
    rng = np.random.default_rng(1)
    cv, W, lab = _case(rng, 6, 40, 128)
    lab[2] = 40                                                   # the reference's NLLLoss raises "Target out of bounds"
    dims = _dims(40, 128)
    loss = CF.angular_loss(dims, _params(cuda(W)), cuda(cv), cuda(lab), MARGIN, S)[0]
    assert np.isnan(loss.item())


def test_ddp_step_trains_an_angular_model_with_sharded_adam():
    """distributed.ddp_step(..., loss_fn=None) runs forward_loss: the fused multi-GPU step, here at world size 1"""
    from code2vec_b200.distributed import ShardedFlatAdam, ddp_step
    rng = np.random.default_rng(3)
    T, P, C, E, H, B, L = 2000, 1500, 1000, 128, 128, 256, 30
    m = _angular_model(rng, T, P, C, E, H).train()
    opt = ShardedFlatAdam(m.parameters(), lr=1e-2)
    s, p, e, lab = (cuda(x) for x in random_batch(rng, B, L, T, P, C))
    losses = [ddp_step(m, opt, None, s, p, e, lab, None).item() for _ in range(6)]
    assert all(np.isfinite(losses))
    assert losses[-1] < losses[0], losses

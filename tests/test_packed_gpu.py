"""-m gpu: packed (CSR) batches against the [B, L] batches they come from.

Every packed result is checked against the padded result of the same batch: bag b of the packed batch is row b of the
padded one without its zero suffix.  Eval encode, a training step with dropout (the same Philox mask in both layouts), the
builder, the module entry points, ddp_step and the memory of a training step.

Eval tolerance.  Both layouts compute every context row's h and score bit for bit alike (the per-row GEMM, LayerNorm and
tanh do not depend on where the row sits in a tile); they differ only in how the online softmax groups the rows into
partials.  That changes the exp(z - m) weights by the relative error of __expf (< 2^-21) and reorders fp32 sums of at most
16 terms per partial and 14 partials per bag (< 30 * 2^-24 relative): 2^-21 + 30 * 2^-24 < 2^-19.  With |h| <= 1 in eval the
code vectors then agree to 2^-19 absolute and the attention weights to 2^-19 relative; the tests allow 8x that, 2^-16.
"""
import ctypes
import math
import types

import numpy as np
import pytest
import torch

from code2vec_b200 import _lib
from code2vec_b200 import functional as CF
from code2vec_b200.batch_builder import DeviceCorpus, packed_offsets
from code2vec_b200.distributed import ShardedFlatAdam, ddp_step
from code2vec_b200.model import Code2Vec
from gpu_util import random_params
from oracle import oracle
from philox_ref import dropout_mask
from fp64_judge import reference as _reference, rho as _rho, scales as _scales

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
EVAL_TOL = 2.0 ** -16
DROPOUT = 0.25

# (Et, Ep, H, algo): the three tensor-core shapes and one odd shape on the CUDA cores
SHAPES = {"h100": (100, 100, 100, "tcgen05"), "h128": (128, 128, 128, "tcgen05"), "h256": (256, 256, 256, "tcgen05"),
          "odd-ffma": (50, 50, 70, "ffma")}
ALGO = {"tcgen05": _lib.ALGO_TCGEN05, "ffma": _lib.ALGO_FFMA}


def _lengths(rng, B, L, empty=True):
    """bag lengths with 1, L and L-1, a run of 40 one-context bags (16 bags in one 16-row slice), and an empty item (0)"""
    n = rng.integers(1, L + 1, B)
    n[:3] = (1, L, L - 1)
    n[10:50] = 1
    if empty:
        n[5] = 0
    return n


def _batch(rng, B, L, T, P, n, zipf=False):
    """-> (padded (s, p, e) int64 [B, L] numpy, PackedBags, lengths).  Bag 3 starts with a masked context (starts == 0);
    an empty item (n == 0) is an all-pad row padded and one pad context packed."""
    if zipf:
        def draw(hi, shape):
            w = 1.0 / np.arange(1, hi)
            return 1 + rng.choice(hi - 1, size=shape, p=w / w.sum())
    else:
        def draw(hi, shape):
            return rng.integers(1, hi, shape)
    s, p, e = draw(T, (B, L)), draw(P, (B, L)), draw(T, (B, L))
    valid = np.arange(L)[None, :] < n[:, None]
    s, p, e = s * valid, p * valid, e * valid
    s[3, 0] = 0
    lens = np.maximum(n, 1)
    keep = np.arange(L)[None, :] < lens[:, None]
    off = np.zeros(B + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    cu = [torch.from_numpy(np.ascontiguousarray(a[keep]).astype(np.int64)).to(DEV) for a in (s, p, e)]
    return (s.astype(np.int64), p.astype(np.int64), e.astype(np.int64)), CF.PackedBags(*cu, off, L), lens


def _padded_positions(bags):
    """flat [B * L] index of every packed context"""
    n = bags.lengths()
    rows = np.repeat(np.arange(bags.B), n)
    return torch.from_numpy(rows * bags.L + np.arange(bags.N) - np.repeat(bags.offsets_host[:-1], n)).to(DEV)


@pytest.mark.parametrize("shape", list(SHAPES))
def test_eval_encode_matches_padded(shape):
    Et, Ep, H, algo = SHAPES[shape]
    rng = np.random.default_rng(7)
    T, P, C, B, L = 3000, 2000, 50, 300, 200
    prm = random_params(rng, T, P, C, Et, Ep, H)
    dims = CF.make_dims(T, P, C, Et, Ep, H)
    t = {k: torch.from_numpy(v).to(DEV) for k, v in prm.items()}
    params = CF.make_params(t["terminal_embedding.weight"], t["path_embedding.weight"], t["input_linear.weight"],
                            t["input_layer_norm.weight"], t["input_layer_norm.bias"], t["attention_parameter"])
    n = _lengths(rng, B, L)
    (s, p, e), bags, lens = _batch(rng, B, L, T, P, n)
    cv_pad, att_pad = CF.encode_forward(dims, params, *(torch.from_numpy(a).to(DEV) for a in (s, p, e)), algo=ALGO[algo])
    cv_pk, att_pk = CF.encode_forward_packed(dims, params, bags, algo=ALGO[algo], check_indices=True)
    torch.cuda.synchronize()
    assert att_pk.shape == (bags.N,) and cv_pk.shape == (B, H)
    full = n > 0
    d_cv = (cv_pk - cv_pad).abs()
    assert float(d_cv[torch.from_numpy(full).to(DEV)].max()) <= EVAL_TOL
    pos = _padded_positions(bags)
    a_pad = att_pad.reshape(-1)[pos]
    real = torch.from_numpy(np.repeat(full, lens)).to(DEV)
    assert float(((att_pk - a_pad).abs() / a_pad.abs().clamp_min(1e-30))[real & (a_pad > 0)].max()) <= EVAL_TOL
    assert bool((att_pk[real & (a_pad == 0)] == 0).all())
    # the empty item: h(0, 0, 0) in both layouts, attention 1.0 on its one context packed, 1/L on each of L padded
    eb = int(np.flatnonzero(~full)[0])
    assert float(d_cv[eb].max()) <= EVAL_TOL
    assert float(att_pk[int(bags.offsets_host[eb])]) == 1.0
    assert torch.allclose(att_pad[eb], torch.full((L,), 1.0 / L, device=DEV), rtol=1e-6, atol=0)
    # both layouts pass the parity bar against the oracle (on the padded inputs)
    _, ref_cv, ref_att = oracle.forward(prm, s, p, e)
    assert float(np.abs(cv_pad.cpu().numpy() - ref_cv).max()) <= 1e-4
    assert float(np.abs(cv_pk.cpu().numpy() - ref_cv).max()) <= 1e-4
    d_att = np.abs(att_pk.cpu().numpy() - ref_att.reshape(-1)[pos.cpu().numpy()])
    assert float(d_att[real.cpu().numpy()].max()) <= 1e-4                 # the empty item follows its own rule (above)


# ---- training step --------------------------------------------------------------------------------------------------
def _option(T, P, C, Et, Ep, H, angular=False):
    return types.SimpleNamespace(terminal_count=T, path_count=P, label_count=C, terminal_embed_size=Et, path_embed_size=Ep,
                                 encode_size=H, dropout_prob=DROPOUT, angular_margin_loss=angular, angular_margin=0.5,
                                 inverse_temp=30.0, device=DEV)


def _model(rng, T, P, C, Et, Ep, H, angular=False, algo="auto"):
    prm = random_params(rng, T, P, C, Et, Ep, H)
    if angular:
        prm["output_linear"] = prm.pop("output_linear.weight")
        del prm["output_linear.bias"]
    m = Code2Vec(_option(T, P, C, Et, Ep, H, angular), algo=algo)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in prm.items()})
    return m.to(DEV)


def _step(m, inputs, label, seed):
    """forward_loss + backward at a fixed dropout seed -> (loss, cv, att, {name: grad}, seed used)"""
    m.zero_grad(set_to_none=True)
    used = []
    m._next_seed = lambda: used.append(seed) or seed
    loss, _, _, cv, att = m.forward_loss(*inputs, label)
    loss.backward()
    torch.cuda.synchronize()
    return loss.detach(), cv.detach(), att.detach(), {k: p.grad.detach().clone() for k, p in m.named_parameters()}, used


@pytest.mark.parametrize("shape,data", [("h128", "uniform"), ("h256", "uniform"), ("h100", "zipf"), ("odd-ffma", "uniform")])
def test_training_step_matches_padded(shape, data):
    Et, Ep, H, algo = SHAPES[shape]
    rng = np.random.default_rng(11)
    T, P, C, B, L = 3000, 2000, 300, 256, 200
    m = _model(rng, T, P, C, Et, Ep, H, algo="auto" if algo == "tcgen05" else "ffma").train()
    n = _lengths(rng, B, L, empty=False)                       # no empty item: provably the same mask in both layouts
    (s, p, e), bags, _ = _batch(rng, B, L, T, P, n, zipf=data == "zipf")
    label = torch.from_numpy(rng.integers(0, C, B)).to(DEV)
    pad = tuple(torch.from_numpy(a).to(DEV) for a in (s, p, e))
    seed = 0x5EED1234
    l_pd, cv_pd, att_pd, g_pd, _ = _step(m, (*pad, ), label, seed)
    l_pk, cv_pk, att_pk, g_pk, used = _step(m, (bags, None, None), label, seed)
    assert used == [seed] and att_pk.shape == (bags.N,)
    # the judge: the fp64 restatement on the shared mask (padded row b * L + j of packed context j of bag b)
    mask = torch.from_numpy(dropout_mask(seed, B * L, H, DROPOUT).reshape(B, L, H)).to(DEV)
    params = {k: v.detach() for k, v in m.state_dict().items()}
    r64 = _reference(params, (*pad, label), mask, False, torch.float64)
    S = _scales(r64, (*pad, label), mask, False)
    pos = _padded_positions(bags)
    att_pk_pad = torch.zeros(B * L, device=DEV).index_put_((pos,), att_pk).view(B, L)
    failures = []
    checks = [("loss", l_pd, l_pk, r64["loss"], S["loss"]), ("cv", cv_pd, cv_pk, r64["cv"], S["cv"]),
              ("att", att_pd, att_pk_pad, r64["att"], S["att"])]
    checks += [(k, g_pd[k], g_pk[k], r64["grads"][k], S[k]) for k in g_pd]
    # Scale-free: rho = |g - g64| / S with S the last sum that produces the quantity, in fp64 on absolute values (see
    # test_train_step_gpu.py).  The packed step must be as accurate as the padded one: max rho(packed) <= max(4 rho(padded),
    # 2^-20), and exactly 0 where S = 0.
    for name, a_pd, a_pk, ref, Sx in checks:
        zv = []
        r_pd = _rho(a_pd, ref, Sx, name + " padded", [])
        r_pk = _rho(a_pk, ref, Sx, name, zv)
        if r_pk > max(4.0 * r_pd, 2.0 ** -20) or zv:
            failures.append(f"{name}: rho packed {r_pk:.3g} padded {r_pd:.3g} {zv}")
    assert not failures, failures


# ---- builder ----------------------------------------------------------------------------------------------------------
def _corpus(rng, n_items=400):
    ns = rng.integers(0, 500, n_items)
    ns[:4] = (0, 1, 200, 201)
    off = np.zeros(n_items + 1, np.int64)
    np.cumsum(ns, out=off[1:])
    ctx = rng.integers(1, 900, (int(off[-1]), 3)).astype(np.int32)
    ctx[rng.random(len(ctx)) < 0.05, 0] = 2                   # @method_0 -> @question
    return DeviceCorpus(off, ctx, np.arange(n_items) % 37, 2, 1, DEV), ns


def test_build_packed_equals_build_without_suffix():
    rng = np.random.default_rng(3)
    c, ns = _corpus(rng)
    L = 200
    ids = np.concatenate([[0, 1, 2, 3, -5, 10_000], rng.integers(0, len(ns), 250)])
    s, p, e, lab = c.build(torch.from_numpy(ids).to(DEV), L, seed=99)
    bags, lab_pk = c.build_packed(ids, L, seed=99)
    assert np.array_equal(bags.offsets_host, packed_offsets(ns, ids, L))
    assert torch.equal(lab_pk, lab)
    ps, pp, pe = bags.padded()
    assert torch.equal(ps, s) and torch.equal(pp, p) and torch.equal(pe, e)
    assert int(bags.lengths()[4]) == 1 and int(bags.starts[bags.offsets_host[4]]) == 0     # unknown id: one pad context


def test_build_packed_takes_device_ids():
    rng = np.random.default_rng(3)
    c, _ = _corpus(rng)
    ids = rng.integers(-2, 420, 100)
    a, la = c.build_packed(ids, 120, seed=7)
    b, lb = c.build_packed(torch.from_numpy(ids).to(DEV), 120, seed=7)
    assert np.array_equal(a.offsets_host, b.offsets_host) and torch.equal(a.offsets, b.offsets)
    assert torch.equal(la, lb) and all(torch.equal(x, y) for x, y in zip(a.padded(), b.padded()))


@pytest.mark.parametrize("rank,world", [(0, 1), (1, 2)])
def test_epoch_packed_visits_the_same_items_in_the_same_order(rank, world):
    rng = np.random.default_rng(4)
    c, _ = _corpus(rng, 300)
    pd = list(c.epoch(64, 50, seed=5, rank=rank, world=world))
    pk = list(c.epoch_packed(64, 50, seed=5, rank=rank, world=world))
    assert len(pd) == len(pk)
    for (s, p, e, lab), (bags, lab_pk) in zip(pd, pk):
        assert torch.equal(lab, lab_pk)
        assert torch.equal(bags.offsets.cpu(), torch.from_numpy(bags.offsets_host))
        assert all(torch.equal(a, b) for a, b in zip((s, p, e), bags.padded()))


# ---- module ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("angular", [False, True])
def test_predict_and_topk_on_packed_input(angular):
    rng = np.random.default_rng(5)
    T, P, C, Et, H, B, L = 3000, 2000, 500, 128, 128, 200, 200
    m = _model(rng, T, P, C, Et, Et, H, angular=angular).eval()
    (s, p, e), bags, _ = _batch(rng, B, L, T, P, _lengths(rng, B, L))
    w_out, b_out = m._head()
    params = CF.make_params(w_out=w_out, b_out=b_out)
    dims = m._dims()
    idx, val, prob, cv, att = m.predict_topk(bags, None, None, k=5)
    assert att.shape == (bags.N,)
    if angular:
        ref = CF.angular_topk(dims, params, cv, 5, m.option.inverse_temp)
    else:
        ref = CF.label_topk(dims, params, cv, 5)
        am, mx, cv2, _ = m.predict(bags, None, None)
        _, am_ref, mx_ref = CF.label_logits_argmax(dims, params, cv2, want_logits=False)
        assert torch.equal(am, am_ref) and torch.equal(mx, mx_ref)
        assert torch.equal(cv2, cv)
    assert torch.equal(idx, ref[0]) and torch.equal(val, ref[1]) and torch.equal(prob, ref[2])
    # the code vectors are those of the padded batch
    cv_pad = m.predict_topk(*(torch.from_numpy(a).to(DEV) for a in (s, p, e)), k=5)[3]
    assert float((cv - cv_pad).abs().max()) <= EVAL_TOL


def test_packed_out_of_range_index_raises_later():
    rng = np.random.default_rng(6)
    T, P, C, Et, H, B, L = 1000, 800, 50, 128, 128, 32, 20
    m = _model(rng, T, P, C, Et, Et, H).eval()
    (s, p, e), bags, _ = _batch(rng, B, L, T, P, _lengths(rng, B, L))
    bags.paths[7] = P + 3
    m.predict(bags, None, None)                                # clamped to row 0 and counted; no synchronisation
    with pytest.raises(IndexError):
        m.check_indices()
    m.predict(bags, None, None)
    torch.cuda.synchronize()
    with pytest.raises(IndexError):                            # the deferred error of the previous call
        m.predict(bags, None, None)


def test_ddp_step_packed_matches_padded():
    T, P, C, Et, H, B, L = 3000, 2000, 300, 128, 128, 256, 200
    losses = {}
    for layout in ("padded", "packed"):
        rng = np.random.default_rng(8)
        torch.manual_seed(0)
        m = _model(rng, T, P, C, Et, Et, H).train()
        opt = ShardedFlatAdam(m.parameters(), lr=0.01)
        out = []
        for step in range(3):
            (s, p, e), bags, _ = _batch(rng, B, L, T, P, _lengths(rng, B, L, empty=False))
            label = torch.from_numpy(rng.integers(0, C, B)).to(DEV)
            inputs = (bags, None, None) if layout == "packed" else tuple(torch.from_numpy(a).to(DEV) for a in (s, p, e))
            out.append(float(ddp_step(m, opt, None, *inputs, label, None).detach()))
        losses[layout] = out
    # the same mask and parameters in both runs; Adam turns last-bit differences into lr-sized moves only where a gradient
    # element is ~0, which moves the loss far less than this
    assert np.allclose(losses["packed"], losses["padded"], rtol=1e-4, atol=0), losses


def test_packed_training_step_needs_less_memory_at_a_third_full():
    rng = np.random.default_rng(9)
    T, P, C, Et, H, B, L = 20000, 20000, 1000, 128, 128, 1024, 200
    m = _model(rng, T, P, C, Et, Et, H).train()
    n = np.clip(rng.geometric(1.0 / 68, B), 1, L)             # ~34 % mean fill
    (s, p, e), bags, _ = _batch(rng, B, L, T, P, n)
    label = torch.from_numpy(rng.integers(0, C, B)).to(DEV)
    pad = tuple(torch.from_numpy(a).to(DEV) for a in (s, p, e))
    peak = {}
    for name, inputs in (("padded", pad), ("packed", (bags, None, None))):
        _step(m, inputs, label, 1)                             # warm: workspaces and gradients exist
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(DEV)
        base = torch.cuda.memory_allocated(DEV)
        _step(m, inputs, label, 1)
        peak[name] = torch.cuda.max_memory_allocated(DEV) - base
    fill = bags.N / (B * L)
    assert 0.25 < fill < 0.45
    # the x stash alone is N x H fp32: the packed step saves at least (B L - N) H 4 bytes of it
    assert peak["packed"] + 0.9 * (B * L - bags.N) * H * 4 <= peak["padded"], (peak, fill)

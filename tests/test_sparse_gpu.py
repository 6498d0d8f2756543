"""-m gpu: sparse embedding gradients (Code2Vec.terminal_embedding.sparse / path_embedding.sparse): the row maps of
c2v_sparse_rows, the compact gradients of the encode backward against the dense path and an fp64 reference, the fused
SparseAdam step against torch.optim.SparseAdam bit for bit, and a training loop against the torch-CPU restatement with
nn.Embedding(sparse=True) semantics."""
import contextlib
import functools

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F
from torch.utils.data import DataLoader

from gpu_util import option_from, random_params
from philox_ref import dropout_mask
from code2vec_b200 import functional as CF
from code2vec_b200.distributed import FusedSparseAdam
from code2vec_b200.model import Code2Vec

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@contextlib.contextmanager
def _sparse_embedding():
    """oracle.torch_forward with F.embedding(..., sparse=True): the reference module with nn.Embedding(sparse=True)"""
    orig = F.embedding
    F.embedding = functools.partial(orig, sparse=True)
    try:
        yield
    finally:
        F.embedding = orig


# ---- 1. row maps ---------------------------------------------------------------------------------------------------
def _zipf(rng, n, vocab):
    return np.minimum(rng.zipf(1.2, n), vocab - 1).astype(np.int64)


ROW_CASES = {
    "uniform": lambda rng: ([rng.integers(0, 50000, 4096), rng.integers(0, 50000, 3000)], 50000),
    "zipf": lambda rng: ([_zipf(rng, 8192, 300000)], 300000),
    "out_of_range": lambda rng: ([np.array([5, -3, 7, 10**9, 5, 9], np.int64), np.array([12, 11], np.int64)], 12),
    "n=0": lambda rng: ([np.zeros(0, np.int64)], 1000),
    "vocab=1": lambda rng: ([np.array([0, 0, 3, -1], np.int64)], 1),
    "padded": lambda rng: ([np.concatenate([rng.integers(1, 9000, 700), np.zeros(300, np.int64)]),
                            np.zeros(50, np.int64)], 9000),
    "chunks": lambda rng: ([rng.integers(0, 3 * 8192 + 17, 20000)], 3 * 8192 + 17),
}


@pytest.mark.parametrize("case", list(ROW_CASES))
def test_row_maps(case):
    rng = np.random.default_rng(len(case))
    lists, vocab = ROW_CASES[case](rng)
    idx = [torch.from_numpy(a).to(DEV) for a in lists]
    slot, rows, count = CF.sparse_rows(idx, vocab)
    flat = torch.cat(idx) if idx else torch.zeros(0, dtype=torch.int64, device=DEV)
    clamped = torch.where((flat < 0) | (flat >= vocab), torch.zeros_like(flat), flat)
    ref = torch.unique(clamped)
    U = int(count.item())
    assert U == ref.numel()
    assert rows.numel() == min(vocab, flat.numel())
    assert torch.equal(rows[:U], ref)
    assert torch.equal(slot[rows[:U]].long(), torch.arange(U, device=DEV))
    untouched = torch.ones(vocab, dtype=torch.bool, device=DEV)
    untouched[ref] = False
    assert bool((slot[untouched] == -1).all())


# ---- 2. gradients --------------------------------------------------------------------------------------------------
T, P, C, B, L, SEED = 600, 500, 11, 8, 16, 12345
# (Et, Ep, H, dC on the CUDA cores).  Et == Ep <= 256 with Et and H multiples of 4 scatter on the tensor cores
# (backward_dc_tc_kernel); the others -- and C2V_BACKWARD_DC=ffma -- in backward_rows_kernel, with 16-byte vector adds
# when Et and Ep are multiples of 4 (VEC) and scalar ones otherwise.
SHAPES = [(128, 128, 128, False), (100, 100, 100, False), (256, 256, 256, False), (12, 12, 20, False),
          (20, 36, 24, False), (10, 7, 9, False), (128, 128, 128, True), (12, 12, 20, True)]


def _model(params, dims, dropout, sparse):
    Et, Ep, H = dims
    m = Code2Vec(option_from({"T": T, "P": P, "C": C, "Et": Et, "Ep": Ep, "H": H}, dropout=dropout))
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    m = m.to(DEV).train()
    m._next_seed = lambda: SEED                       # the same dropout mask on both models (and in the reference)
    m.terminal_embedding.sparse, m.path_embedding.sparse = sparse
    return m


def _batch(rng, unique):
    if unique:                                        # no row repeats: every value is one dC row, added once
        t = rng.permutation(np.arange(1, T))[:2 * B * L]
        s, e = t[:B * L].reshape(B, L), t[B * L:].reshape(B, L)
        p = rng.permutation(np.arange(1, P))[:B * L].reshape(B, L)
        n = np.full(B, L)
    else:
        s, p, e = rng.integers(1, 40, (B, L)), rng.integers(1, 30, (B, L)), rng.integers(1, T, (B, L))
        n = rng.integers(1, L + 1, B)
        for b in range(B):
            s[b, n[b]:] = 0; p[b, n[b]:] = 0; e[b, n[b]:] = 0
    lab = rng.integers(0, C, B)
    return [torch.from_numpy(np.ascontiguousarray(a, np.int64)) for a in (s, p, e, lab)] + [n]


def _inputs(batch, packed):
    s, p, e, lab, n = batch
    if not packed:
        return (s.to(DEV), p.to(DEV), e.to(DEV)), lab.to(DEV)
    keep = torch.from_numpy(np.arange(L)[None, :] < n[:, None])
    off = np.concatenate([[0], np.cumsum(n)])
    bags = CF.PackedBags(s[keep].to(DEV), p[keep].to(DEV), e[keep].to(DEV), off, L)
    return (bags, None, None), lab.to(DEV)


def _step(model, inputs, lab):
    out, _, _ = model.forward(*inputs, lab)
    F.nll_loss(F.log_softmax(out, dim=1), lab).backward()
    return model.terminal_embedding.weight.grad, model.path_embedding.weight.grad


def _fp64(params, batch, H, dropout):
    """fp64 gradients of the two tables and their scale S (test_train_step_gpu.py's scale-free criterion)"""
    from oracle import oracle
    s, pth, e, lab, _ = batch
    p = {k: torch.from_numpy(v).double().requires_grad_() for k, v in params.items()}
    mask = torch.from_numpy(dropout_mask(SEED, B * L, H, dropout)).view(B, L, H).double() if dropout else None
    taps = {}
    out, _, _ = oracle.torch_forward(p, s, pth, e, lab, dropmask=mask, taps=taps)
    taps["x"].retain_grad()
    F.nll_loss(F.log_softmax(out, dim=1), lab).backward()
    Et, Ep = p["terminal_embedding.weight"].shape[1], p["path_embedding.weight"].shape[1]
    A = taps["x"].grad.reshape(B * L, H).abs() @ p["input_linear.weight"].detach().abs()
    St = torch.zeros(T, Et, dtype=torch.float64).index_add_(0, s.reshape(-1), A[:, :Et]).index_add_(0, e.reshape(-1),
                                                                                                    A[:, Et + Ep:])
    Sp = torch.zeros(P, Ep, dtype=torch.float64).index_add_(0, pth.reshape(-1), A[:, Et:Et + Ep])
    return (p["terminal_embedding.weight"].grad, St), (p["path_embedding.weight"].grad, Sp)


def _rho(a, ref, S):
    nz = S > 0
    assert not bool(((a.double() != 0) & ~nz).any())
    return float(((a.double() - ref).abs()[nz] / S[nz]).max()) if bool(nz.any()) else 0.0


@pytest.mark.parametrize("dropout", [0.0, 0.3])
@pytest.mark.parametrize("stash", [True, False])
@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("Et,Ep,H,dc_ffma", SHAPES)
def test_sparse_gradients(Et, Ep, H, dc_ffma, packed, stash, dropout, monkeypatch):
    if not stash:
        monkeypatch.setenv("C2V_NO_STASH", "1")
    if dc_ffma:
        monkeypatch.setenv("C2V_BACKWARD_DC", "ffma")
    rng = np.random.default_rng(Et * 7 + Ep * 3 + H)
    params = random_params(rng, T, P, C, Et, Ep, H)
    dims = (Et, Ep, H)
    for unique in (True, False):
        batch = _batch(rng, unique)
        inputs, lab = _inputs(batch, packed)
        dense = _step(_model(params, dims, dropout, (False, False)), inputs, lab)
        sparse = _step(_model(params, dims, dropout, (True, True)), inputs, lab)
        s, pth, e = batch[:3]
        if packed:                                    # the rows the packed contexts index (no padding rows)
            ref_idx = [torch.unique(torch.cat([inputs[0].starts, inputs[0].ends])), torch.unique(inputs[0].paths)]
        else:
            from oracle import oracle
            p = {k: torch.from_numpy(v).requires_grad_() for k, v in params.items()}
            with _sparse_embedding():
                out, _, _ = oracle.torch_forward(p, s, pth, e)
            out.sum().backward()
            ks = ("terminal_embedding.weight", "path_embedding.weight")
            assert all(p[k].grad.is_sparse for k in ks)    # the reference really ran with sparse embeddings
            ref_idx = [p[k].grad.coalesce().indices()[0] for k in ks]
        ref64 = _fp64(params, batch, H, dropout) if not unique else None
        for i, (gs, gd) in enumerate(zip(sparse, dense)):
            assert gs.is_sparse and not gd.is_sparse
            assert gs.is_coalesced()                  # one backward into an empty .grad
            assert gs.shape == gd.shape
            rows = gs.indices()[0]
            assert torch.equal(rows.cpu(), ref_idx[i].cpu())
            if unique:
                assert torch.equal(gs.values(), gd[rows])
                assert bool((gd[rows].abs().sum(1) > 0).all())
            else:
                g64, S = ref64[i]
                full = torch.zeros_like(gd).index_put_((rows,), gs.values()).cpu()
                r_s, r_d = _rho(full, g64, S), _rho(gd.cpu(), g64, S)
                assert r_s <= max(2 * r_d, 2.0 ** -20), (i, r_s, r_d)


def test_one_table_sparse_the_other_dense():
    rng = np.random.default_rng(5)
    params = random_params(rng, T, P, C, 128, 128, 128)
    batch = _batch(rng, False)
    inputs, lab = _inputs(batch, False)
    dense = _step(_model(params, (128, 128, 128), 0.0, (False, False)), inputs, lab)
    for which in (0, 1):
        flags = (which == 0, which == 1)
        g = _step(_model(params, (128, 128, 128), 0.0, flags), inputs, lab)
        assert g[which].is_sparse and not g[1 - which].is_sparse
        # (rows repeat: the atomics may add them in another order than the dense run did)
        assert _close(g[1 - which], dense[1 - which]) and _close(g[which].to_dense(), dense[which])


def _close(a, b):
    return torch.allclose(a, b, rtol=1e-5, atol=1e-6)


def test_accumulation_and_coalesced_flag():
    rng = np.random.default_rng(6)
    params = random_params(rng, T, P, C, 128, 128, 128)
    m = _model(params, (128, 128, 128), 0.0, (True, True))
    b1, b2 = _batch(rng, False), _batch(rng, False)
    i1, l1 = _inputs(b1, False)
    i2, l2 = _inputs(b2, False)
    g1 = [g.clone() for g in _step(m, i1, l1)]
    assert all(g.is_coalesced() for g in g1)
    g2 = _step(m, i2, l2)                               # accumulates: still sparse, the sum of both batches
    m.zero_grad()
    g_only2 = _step(m, i2, l2)
    for a, b, c in zip(g1, g2, g_only2):
        assert b.is_sparse
        assert _close(b.to_dense(), a.to_dense() + c.to_dense())


def test_second_backward_through_a_retained_graph_stays_sparse():
    rng = np.random.default_rng(8)
    params = random_params(rng, T, P, C, 128, 128, 128)
    m = _model(params, (128, 128, 128), 0.0, (True, True))
    inputs, lab = _inputs(_batch(rng, False), False)
    out, _, _ = m.forward(*inputs, lab)
    loss = F.nll_loss(F.log_softmax(out, dim=1), lab)
    loss.backward(retain_graph=True)
    first = [m.terminal_embedding.weight.grad.clone(), m.path_embedding.weight.grad.clone()]
    loss.backward()
    for a, b in zip(first, (m.terminal_embedding.weight.grad, m.path_embedding.weight.grad)):
        assert a.is_sparse and b.is_sparse
        assert _close(b.to_dense(), 2 * a.to_dense())


def test_model_off_the_current_device():
    """the row maps, the copy of U and its event follow the batch's device, not the current one"""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    rng = np.random.default_rng(9)
    params = random_params(rng, T, P, C, 128, 128, 128)
    inputs, lab = _inputs(_batch(rng, False), False)
    ref = _step(_model(params, (128, 128, 128), 0.0, (True, True)), inputs, lab)
    dev1 = torch.device("cuda:1")
    m = _model(params, (128, 128, 128), 0.0, (True, True)).to(dev1)
    with torch.cuda.device(0):
        g = _step(m, tuple(t.to(dev1) for t in inputs), lab.to(dev1))
    for a, b in zip(ref, g):
        assert torch.equal(a.indices().cpu(), b.indices().cpu()) and _close(a.values().cpu(), b.values().cpu())


def test_out_of_range_index_raises_at_backward():
    rng = np.random.default_rng(7)
    params = random_params(rng, T, P, C, 128, 128, 128)
    m = _model(params, (128, 128, 128), 0.0, (True, True))
    (s, p, e), lab = _inputs(_batch(rng, False), False)
    s = s.clone(); s[1, 0] = T + 3                       # read as row 0 and counted
    out, _, _ = m.forward(s, p, e, lab)
    torch.cuda.synchronize()
    with pytest.raises(IndexError):
        out.sum().backward()


# ---- 3. optimizer --------------------------------------------------------------------------------------------------
def _grads(rng, n, E):
    """4 gradients: rows missing in some steps, an empty one, an uncoalesced one with duplicate rows (pairs: their sum
    does not depend on the order coalesce adds them in)"""
    def sp(rows, vals):
        return torch.sparse_coo_tensor(torch.tensor(rows, dtype=torch.int64)[None], torch.from_numpy(vals), (n, E))
    r1 = np.sort(rng.choice(n, n // 2, replace=False))
    r3 = rng.choice(n, 10, replace=False)
    r4 = np.sort(rng.choice(n, n // 3, replace=False))
    f = lambda k: rng.standard_normal((k, E)).astype(np.float32)
    return [sp(r1, f(len(r1))).coalesce(), sp(np.zeros(0, np.int64), f(0)),
            sp(np.concatenate([r3, r3[:6]]), f(16)), sp(r4, f(len(r4))).coalesce()]


@pytest.mark.parametrize("E", [12, 100, 128])
def test_fused_sparse_adam_matches_torch_bitwise(E):
    rng = np.random.default_rng(E)
    n = 257
    w0 = torch.from_numpy(rng.standard_normal((n, E)).astype(np.float32)).to(DEV)
    # torch's SparseAdam on the same device: CUDA's sqrt is correctly rounded, as the kernel's is (torch's CPU sqrt may
    # not be, depending on the vector unit)
    ref_p = nn.Parameter(w0.clone())
    p = nn.Parameter(w0.clone())
    kw = dict(lr=0.0123, betas=(0.85, 0.995), eps=1e-6)
    ref, fused = torch.optim.SparseAdam([ref_p], **kw), FusedSparseAdam([p], **kw)
    for g in _grads(rng, n, E):
        ref_p.grad, p.grad = g.clone().to(DEV), g.clone().to(DEV)
        ref.step(); fused.step()
        rs, fs = ref.state[ref_p], fused.state[p]
        assert fs["step"] == rs["step"]
        assert torch.equal(p.detach(), ref_p.detach())
        assert torch.equal(fs["exp_avg"], rs["exp_avg"]) and torch.equal(fs["exp_avg_sq"], rs["exp_avg_sq"])
    assert fused.state[p]["step"] == 4                  # the empty gradient counted


# ---- 4. training loop ----------------------------------------------------------------------------------------------
def test_training_loop_with_sparse_tables():
    from oracle import oracle
    from test_dropin_loop_gpu import _dataset
    E = H = 128
    rng = np.random.default_rng(E)
    T_, P_, C_, L_, n, bs = 300, 200, 17, 40, 150, 32
    ds = _dataset(rng, n, L_, T_, P_, C_)
    params = random_params(rng, T_, P_, C_, E, E, H)
    model = Code2Vec(option_from({"T": T_, "P": P_, "C": C_, "Et": E, "Ep": E, "H": H}))
    model.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    model = model.to(DEV)
    model.terminal_embedding.sparse = model.path_embedding.sparse = True
    tables = [model.terminal_embedding.weight, model.path_embedding.weight]
    rest = [q for q in model.parameters() if all(q is not t for t in tables)]
    sparse_opt = FusedSparseAdam(tables, lr=0.01)
    dense_opt = torch.optim.Adam(rest, lr=0.01, betas=(0.9, 0.999), weight_decay=0.0)
    ref = {k: torch.from_numpy(v).clone().requires_grad_(True) for k, v in params.items()}
    tk = ("terminal_embedding.weight", "path_embedding.weight")
    ref_sparse = torch.optim.SparseAdam([ref[k] for k in tk], lr=0.01)
    ref_dense = torch.optim.Adam([v for k, v in ref.items() if k not in tk], lr=0.01, betas=(0.9, 0.999), weight_decay=0.0)
    criterion = nn.NLLLoss(weight=torch.ones(C_)).to(DEV)
    ref_crit = nn.NLLLoss(weight=torch.ones(C_))
    losses, ref_losses = [], []
    for epoch in range(5):
        loader = DataLoader(ds, batch_size=bs, shuffle=True, generator=torch.Generator().manual_seed(epoch), num_workers=0)
        model.train()
        for sb in loader:
            starts, paths, ends, label = (sb[k].to(DEV) for k in ("starts", "paths", "ends", "label"))
            preds, _, _ = model.forward(starts, paths, ends, label)
            loss = criterion(F.log_softmax(preds, dim=1), label)
            loss.backward()
            dense_opt.step(); sparse_opt.step()
            dense_opt.zero_grad(); sparse_opt.zero_grad()
            losses.append(loss.item())
            with _sparse_embedding():
                rp, _, _ = oracle.torch_forward(ref, sb["starts"], sb["paths"], sb["ends"], sb["label"])
            rl = ref_crit(F.log_softmax(rp, dim=1), sb["label"])
            rl.backward()
            assert ref[tk[0]].grad.is_sparse
            ref_dense.step(); ref_sparse.step()
            ref_dense.zero_grad(); ref_sparse.zero_grad()
            ref_losses.append(rl.item())
    assert len(losses) == 25
    assert np.abs(np.array(losses[:5]) - np.array(ref_losses[:5])).max() <= 2e-4, (losses[:5], ref_losses[:5])
    assert np.abs(np.array(losses) - np.array(ref_losses)).max() <= 2e-2, (losses, ref_losses)
    assert losses[-1] < losses[0]

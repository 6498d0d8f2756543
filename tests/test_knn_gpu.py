"""-m gpu: similarity search over code vectors (c2v_knn_topk / c2v_knn_pairs through code2vec_b200.similarity) against
fp64 cosines on the GPU (F.normalize(x.double()) products).  The bars follow test_topk_gpu._check_angular: returned
similarities within 3e-6 of the fp64 cosine at their index, every returned row at least the fp64 k-th best non-excluded
value - 1e-5, lists sorted by returned value with ties by index."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from code2vec_b200 import _lib
from code2vec_b200.functional import _ptr, _stream
from code2vec_b200.similarity import CodeVectorIndex

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _rand(n, H, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(n, H, generator=g, device=DEV)


def _cos64(q, b):
    return F.normalize(q.double(), dim=1) @ F.normalize(b.double(), dim=1).T


def _check(idx, sims, ref, k, exclude=None):
    """ref: fp64 cosines [Q, N]; exclude: int64 [Q, X] or None"""
    Q, N = ref.shape
    assert idx.shape == (Q, k) and sims.shape == (Q, k) and idx.dtype == torch.int64 and sims.dtype == torch.float32
    ref = ref.clone()
    if exclude is not None:
        r, c = ((exclude >= 0) & (exclude < N)).nonzero(as_tuple=True)
        ref[r, exclude[r, c]] = -float("inf")
    assert bool(((idx >= 0) & (idx < N)).all())
    got = ref.gather(1, idx)
    assert bool(torch.isfinite(got).all()), "an excluded row was returned"
    assert (sims.double() - got).abs().max().item() <= 3e-6
    kth = torch.sort(ref, dim=1, descending=True).values[:, k - 1:k]
    assert bool((got >= kth - 1e-5).all())
    assert all(len(set(r)) == k for r in idx.tolist())
    if k > 1:
        d = sims[:, :-1] - sims[:, 1:]
        assert bool((d >= 0).all())
        assert bool(((d > 0) | (idx[:, :-1] < idx[:, 1:])).all())


def _ks(n):
    return sorted({min(k, n) for k in (1, 5, 10, _lib.TOPK_MAX)})


@pytest.mark.parametrize("N", [1, 5, 127, 128, 129, 4097, 195299])
@pytest.mark.parametrize("H", [4, 36, 100, 128, 256])
def test_knn_matches_fp64_cosines(N, H):
    bank = _rand(N, H, N * 7 + H)
    index = CodeVectorIndex(bank)
    assert index.fused
    for Q in (1, 37, 2048):
        if Q * N > 2048 * 4097:
            continue                                           # keeps the fp64 judge small; Q = 37 covers the large N
        q = _rand(Q, H, Q + N)
        ref = _cos64(q, bank)
        for k in _ks(N):
            idx, sims = index.search(q, k)
            _check(idx, sims, ref, k)
    assert index.prep_builds == 1


def test_knn_cuts_large_query_sets_into_chunks():
    bank, q = _rand(4097, 128, 1), _rand(2049, 128, 2)
    index = CodeVectorIndex(bank)
    idx, sims = index.search(q, 10)
    _check(idx, sims, _cos64(q, bank), 10)
    i2, s2 = index.search(q[2048:], 10)
    assert torch.equal(idx[2048:], i2) and torch.equal(sims[2048:], s2)
    assert index.prep_builds == 1


def test_exact_duplicates_tie_lowest_index_first():
    bank = _rand(1000, 128, 3)
    for r in (10, 50, 999):
        bank[r] = bank[3]
    index = CodeVectorIndex(bank)
    idx, sims = index.search(bank[3:4].clone(), 5)
    assert idx[0, :4].tolist() == [3, 10, 50, 999]
    assert len(set(sims[0, :4].tolist())) == 1 and abs(sims[0, 0].item() - 1.0) <= 3e-6
    _check(idx, sims, _cos64(bank[3:4], bank), 5)


def test_self_exclusion_with_a_clone_present():
    bank = _rand(5000, 100, 4)
    bank[4321] = bank[17]
    index = CodeVectorIndex(bank)
    idx, sims = index.neighbours([17, 4321], k=10)
    assert idx[0, 0].item() == 4321 and idx[1, 0].item() == 17
    assert (sims[:, 0] - 1.0).abs().max().item() <= 3e-6
    assert 17 not in idx[0].tolist() and 4321 not in idx[1].tolist()
    rows = torch.tensor([17, 4321], device=DEV)
    _check(idx, sims, _cos64(bank[rows], bank), 10, rows[:, None])


def test_zero_vectors_score_zero():
    bank = _rand(300, 64, 5)
    bank[[0, 7, 299]] = 0.0
    index = CodeVectorIndex(bank)
    q = _rand(4, 64, 6)
    q[1] = 0.0
    idx, sims = index.search(q, 16)
    assert idx[1].tolist() == list(range(16)) and bool((sims[1] == 0).all())       # everything ties at 0: row order
    _check(idx, sims, F.normalize(q.double(), dim=1) @ F.normalize(bank.double(), dim=1).T, 16)
    full, fs = index.search(q, 16)
    assert torch.equal(full, idx) and torch.equal(fs, sims)


def test_exclusion_width_four_with_duplicates_and_negatives():
    bank, q = _rand(4097, 128, 7), _rand(37, 128, 8)
    ref = _cos64(q, bank)
    top = torch.sort(ref, dim=1, descending=True, stable=True).indices
    ex = torch.stack([top[:, 0], top[:, 0], torch.full_like(top[:, 0], -1), top[:, 2]], 1)   # best twice, none, third
    ex[5] = torch.tensor([-7, top[5, 1].item(), 5000, top[5, 0].item()], device=DEV)        # beyond N is ignored too
    index = CodeVectorIndex(bank)
    idx, sims = index.search(q, _lib.TOPK_MAX, exclude=ex)
    _check(idx, sims, ref, _lib.TOPK_MAX, ex)
    assert idx[0, 0].item() == top[0, 1].item() and idx[0, 1].item() == top[0, 3].item()


def _pairs_ref(bank, thr, band=1e-5):
    c = _cos64(bank, bank)
    upper = torch.triu(torch.ones_like(c, dtype=torch.bool), diagonal=1)
    sure = upper & (c >= thr + band)
    maybe = upper & ((c - thr).abs() <= band)
    return c, sure, maybe


def test_pairs_self_join_matches_fp64_outside_the_band():
    bank = _rand(3000, 128, 9)
    bank[1000:1100] = bank[:100] + 0.1 * _rand(100, 128, 10)               # near duplicates
    bank[2999] = bank[5]
    index = CodeVectorIndex(bank)
    for thr in (0.95, 0.5, 0.2):
        i, j, s = index.pairs(thr)
        c, sure, maybe = _pairs_ref(bank, thr)
        assert bool((i < j).all())
        got = torch.zeros_like(sure)
        got[i, j] = True
        assert int(got.sum()) == i.numel()                                 # no duplicates
        assert bool((got | ~sure).all()) and bool((~got | sure | maybe).all())
        assert (s.double() - c[i, j]).abs().max().item() <= 3e-6
        di, ds, dj = i[1:] - i[:-1], s[:-1] - s[1:], j[1:] - j[:-1]          # sorted by (i, -sim, j)
        assert bool(((di > 0) | ((di == 0) & ((ds > 0) | ((ds == 0) & (dj > 0))))).all())


def test_pairs_for_given_rows_and_the_raw_capacity_contract():
    bank = _rand(2500, 64, 11)
    bank[2000:2200] = bank[:200] + 0.05 * _rand(200, 64, 12)
    index = CodeVectorIndex(bank)
    rows = torch.tensor([0, 3, 2005, 2499], device=DEV)
    i, j, s = index.pairs(0.3, rows=rows)
    c = _cos64(bank[rows], bank)
    want = {(rows[a].item(), b) for a, b in ((c >= 0.3 + 1e-5).nonzero().tolist()) if b != rows[a].item()}
    got = set(zip(i.tolist(), j.tolist()))
    assert want <= got and len(got) == i.numel()
    assert all(a != b for a, b in got)
    # capacity smaller than the count: the count is exact, the written pairs are a subset of the full run's
    lib = _lib.load()
    N, H = bank.shape
    q = bank[:2048].contiguous()
    prep = torch.empty(lib.c2v_knn_prep_workspace_bytes(N, H), dtype=torch.uint8, device=DEV)
    ws = torch.empty(lib.c2v_knn_pairs_workspace_bytes(N, H, 2048), dtype=torch.uint8, device=DEV)

    def run(cap, flags):
        out = [torch.full((max(cap, 1),), -1, dtype=dt, device=DEV) for dt in (torch.int64, torch.int64, torch.float32)]
        count = torch.zeros(1, dtype=torch.int64, device=DEV)
        rc = lib.c2v_knn_pairs(_ptr(bank), N, H, _ptr(q), 2048, ctypes.c_float(0.3), None, 0, 0, 0, cap, _ptr(out[0]),
                               _ptr(out[1]), _ptr(out[2]), _ptr(count), _ptr(prep), prep.numel(), _ptr(ws), ws.numel(), flags,
                               _stream(DEV))
        _lib.check(rc, "c2v_knn_pairs")
        return int(count.item()), out

    n_big, big = run(1 << 20, 0)
    n_small, small = run(100, 0x100)
    n_zero, _ = run(0, 0x100)
    assert n_big == n_small == n_zero and n_big > 100
    full = set(zip(big[0][:n_big].tolist(), big[1][:n_big].tolist()))
    part = list(zip(small[0].tolist(), small[1].tolist()))
    assert len(set(part)) == 100 and set(part) <= full
    assert all(a < b for a, b in full)                                   # self_offset 0: upper triangle only


def test_pairs_threshold_extremes():
    bank = _rand(50, 36, 13)
    index = CodeVectorIndex(bank)
    i, j, s = index.pairs(-1.0)
    assert i.numel() == 50 * 49 // 2 and bool((i < j).all())
    i, j, s = index.pairs(1.01)
    assert i.numel() == 0
    small = index.pairs(0.0, capacity=3)                                 # overflow: one re-run with the exact size
    full = index.pairs(0.0)
    assert small[0].numel() > 3 and all(torch.equal(a, b) for a, b in zip(small, full))


def test_prep_is_reused_across_chunks_and_rebuilt_after_an_in_place_change():
    bank, q = _rand(4097, 128, 14), _rand(3000, 128, 15)
    index = CodeVectorIndex(bank)
    lib = _lib.load()
    n0 = lib.c2v_launch_count()
    index.search(q[:100], 5)
    n1 = lib.c2v_launch_count()
    index.search(q[:100], 5)
    n2 = lib.c2v_launch_count()
    assert (n1 - n0, n2 - n1) == (4, 3)                                  # bank prep, query prep, GEMM, merge / no bank prep
    a = index.search(q, 10)
    assert index.prep_builds == 1
    bank[100] = bank[7]                                                  # in place: the version counter moves
    b = index.search(q, 10)
    assert index.prep_builds == 2
    fresh = CodeVectorIndex(bank.clone()).search(q, 10)
    assert torch.equal(b[0], fresh[0]) and torch.equal(b[1], fresh[1]) and not torch.equal(a[0], b[0])
    _check(*b, _cos64(q, bank), 10)


def _stable_rows(ref, k):
    """rows whose fp64 ranking has no gap below 1e-5 among its first k + 1 values (no near-tie to resolve differently)"""
    v = torch.sort(ref, dim=1, descending=True).values[:, :k + 1]
    return ((v[:, :-1] - v[:, 1:]) > 1e-5).all(1)


def test_fallbacks_rank_like_the_fused_path():
    bank, q = _rand(4097, 130, 16), _rand(37, 130, 17)
    slow = CodeVectorIndex(bank)
    assert not slow.fused
    fast = CodeVectorIndex(F.pad(bank, (0, 2)))                          # zero padding keeps every cosine
    assert fast.fused
    ref = _cos64(q, bank)
    i40, s40 = slow.search(q, 40)
    _check(i40, s40, ref, 40)
    i16, s16 = fast.search(F.pad(q, (0, 2)), _lib.TOPK_MAX)
    _check(i16, s16, ref, _lib.TOPK_MAX)
    ok = _stable_rows(ref, _lib.TOPK_MAX)
    assert int(ok.sum()) > 20 and torch.equal(i40[ok, :_lib.TOPK_MAX], i16[ok])
    j40, t40 = fast.search(F.pad(q, (0, 2)), 40)                         # k above TOPK_MAX at a fused encode size
    assert torch.equal(j40[ok, :_lib.TOPK_MAX], i16[ok])
    a, b, c = slow.pairs(0.3)
    a2, b2, c2 = fast.pairs(0.3)
    sa, sb = set(zip(a.tolist(), b.tolist())), set(zip(a2.tolist(), b2.tolist()))
    cc = _cos64(bank, bank)
    assert all(abs(cc[x, y].item() - 0.3) <= 1e-5 for x, y in sa ^ sb)


def test_memory_stays_far_below_the_similarity_block():
    N, H, Q = 10 ** 6, 128, 2048
    bank = _rand(N, H, 18)
    q = _rand(Q, H, 19)
    index = CodeVectorIndex(bank)
    lib = _lib.load()
    prep_bytes = lib.c2v_knn_prep_workspace_bytes(N, H)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    idx, sims = index.search(q, 10)
    torch.cuda.synchronize()
    block = Q * N * 4                                                    # the [Q, N] fp32 similarity block: 8.2 GB
    first = torch.cuda.max_memory_allocated() - base
    # bound: the bank image (the size of the bank) + 64 MB for the call workspace and the outputs
    assert first <= prep_bytes + (64 << 20) and first < block // 8, (first, prep_bytes)
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    index.search(q, 10)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base <= 64 << 20          # with the image in place
    _check(idx[:64], sims[:64], _cos64(q[:64], bank), 10)


def test_knn_graph_on_a_small_bank_is_the_fp64_ranking_without_self():
    bank = _rand(300, 64, 20)
    index = CodeVectorIndex(bank)
    idx, sims = index.knn_graph(10)
    ref = _cos64(bank, bank)
    ref.fill_diagonal_(-float("inf"))
    _check(idx, sims, ref, 10)
    ok = _stable_rows(ref, 10)
    want = torch.sort(ref, dim=1, descending=True, stable=True).indices[:, :10]
    assert torch.equal(idx[ok], want[ok]) and int(ok.sum()) > 250


def test_most_similar_and_from_file(tmp_path):
    from code2vec_b200 import corpus
    bank = _rand(2000, 128, 21)
    names = [f"m{i}" for i in range(2000)]
    corpus.write_code_vectors(tmp_path / "v.txt", "w", bank, np.arange(2000), names, header_items=2000)
    index = CodeVectorIndex.from_file(tmp_path / "v.txt", device=DEV)
    assert torch.equal(index.vectors, bank) and index.names == names
    got = index.most_similar([1, 2], [3], topn=5)
    u = F.normalize(bank.double(), dim=1)
    qv = F.normalize((u[1] + u[2] - u[3]) / 3, dim=0)
    ref = u @ qv
    ref[[1, 2, 3]] = -float("inf")
    want = torch.sort(ref, descending=True, stable=True).indices[:5].tolist()
    assert [r for r, _, _ in got] == want and [n for _, n, _ in got] == [names[r] for r in want]
    assert max(abs(s - ref[r].item()) for r, _, s in got) <= 3e-6
    many = index.most_similar([1, 2, 4, 5, 6], [3], topn=5)            # more inputs than the kernel excludes
    assert not {1, 2, 3, 4, 5, 6} & {r for r, _, _ in many}

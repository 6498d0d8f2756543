"""CPU-side checks of the similarity search (c2v_knn_*, code2vec_b200.similarity) and of the vector-file reader: every
argument error returns its code and message before any CUDA call, workspace sizes, the write -> read round trip, and
the host arithmetic of most_similar."""
import ctypes

import numpy as np
import pytest
import torch

from code2vec_b200 import _lib, corpus, similarity

V = ctypes.c_void_p
FAKE = V(0x1000)          # never dereferenced: every call below fails its argument checks first
BIG = 1 << 40


def _topk(bank=FAKE, N=1000, H=128, q=FAKE, Q=8, k=4, ex=None, X=0, idx=FAKE, sims=FAKE, prep=FAKE, prep_bytes=BIG,
          ws=FAKE, ws_bytes=BIG, flags=0):
    return _lib.load().c2v_knn_topk(bank, N, H, q, Q, k, ex, X, idx, sims, prep, prep_bytes, ws, ws_bytes, flags, None)


def _pairs(bank=FAKE, N=1000, H=128, q=FAKE, Q=8, thr=0.9, ex=None, X=0, self_offset=-1, base=0, cap=16, pq=FAKE, pi=FAKE,
           ps=FAKE, count=FAKE, prep=FAKE, prep_bytes=BIG, ws=FAKE, ws_bytes=BIG, flags=0):
    return _lib.load().c2v_knn_pairs(bank, N, H, q, Q, ctypes.c_float(thr), ex, X, self_offset, base, cap, pq, pi, ps, count,
                                     prep, prep_bytes, ws, ws_bytes, flags, None)


def _expect(rc, code, name):
    assert rc == code
    msg = _lib.load().c2v_last_error()
    assert msg and name.encode() in msg, msg


COMMON = {"bank": dict(bank=None), "queries": dict(q=None), "misaligned": dict(q=V(0x1004)), "N<1": dict(N=0),
          "N>=2^32-1": dict(N=(1 << 32) - 1), "H<1": dict(H=0), "Q<1": dict(Q=0), "Q>2048": dict(Q=2049),
          "X<0": dict(X=-1), "X>max": dict(ex=FAKE, X=_lib.KNN_EXCLUDE_MAX + 1), "exclude": dict(X=2), "flags": dict(flags=0x400)}


@pytest.mark.parametrize("case", list(COMMON) + ["idx", "sims", "k<1", "k>TOPK_MAX", "k>N-X"])
def test_knn_topk_rejects_bad_arguments(case):
    kw = dict(COMMON.get(case, {}), **{"idx": dict(idx=None), "sims": dict(sims=None), "k<1": dict(k=0),
                                      "k>TOPK_MAX": dict(k=_lib.TOPK_MAX + 1), "k>N-X": dict(N=5, k=4, ex=FAKE, X=2)}.get(case, {}))
    _expect(_topk(**kw), _lib.C2V_EINVAL, "c2v_knn_topk")


@pytest.mark.parametrize("case", list(COMMON) + ["count", "capacity<0", "outputs", "nan"])
def test_knn_pairs_rejects_bad_arguments(case):
    kw = dict(COMMON.get(case, {}), **{"count": dict(count=None), "capacity<0": dict(cap=-1), "outputs": dict(pq=None),
                                      "nan": dict(thr=float("nan"))}.get(case, {}))
    _expect(_pairs(**kw), _lib.C2V_EINVAL, "c2v_knn_pairs")


@pytest.mark.parametrize("H", [30, 260])
def test_knn_reports_unsupported_encode_sizes(H):
    _expect(_topk(H=H), _lib.C2V_EUNSUPPORTED, "c2v_knn_topk")
    _expect(_pairs(H=H), _lib.C2V_EUNSUPPORTED, "c2v_knn_pairs")
    _expect(_lib.load().c2v_knn_prepare(FAKE, 1000, H, FAKE, BIG, None), _lib.C2V_EUNSUPPORTED, "c2v_knn_prepare")
    assert _lib.load().c2v_knn_prep_workspace_bytes(1000, H) == 0


def test_knn_reports_short_workspaces():
    lib = _lib.load()
    N, H, Q, k = 1000, 128, 8, 4
    prep = lib.c2v_knn_prep_workspace_bytes(N, H)
    wt, wp = lib.c2v_knn_topk_workspace_bytes(N, H, Q, k), lib.c2v_knn_pairs_workspace_bytes(N, H, Q)
    _expect(_topk(prep_bytes=prep - 1), _lib.C2V_EWORKSPACE, "c2v_knn_topk")
    _expect(_topk(prep=None), _lib.C2V_EWORKSPACE, "c2v_knn_topk")
    _expect(_topk(ws_bytes=wt - 1), _lib.C2V_EWORKSPACE, "c2v_knn_topk")
    _expect(_pairs(ws_bytes=wp - 1), _lib.C2V_EWORKSPACE, "c2v_knn_pairs")
    _expect(_pairs(ws=None), _lib.C2V_EWORKSPACE, "c2v_knn_pairs")
    _expect(lib.c2v_knn_prepare(FAKE, N, H, FAKE, prep - 1, None), _lib.C2V_EWORKSPACE, "c2v_knn_prepare")
    _expect(lib.c2v_knn_prepare(None, N, H, FAKE, prep, None), _lib.C2V_EINVAL, "c2v_knn_prepare")


def test_knn_workspace_sizes_are_monotone():
    lib = _lib.load()
    for H in (4, 100, 128, 256):
        preps = [lib.c2v_knn_prep_workspace_bytes(N, H) for N in (1, 127, 128, 129, 4097, 10 ** 6, 10 ** 7)]
        assert all(p > 0 for p in preps) and preps == sorted(preps)
        assert preps[-1] >= 10 ** 7 * H * 4                  # the fp16 hi / lo image is as large as the fp32 bank
        for N in (1, 129, 10 ** 6):
            t = [[lib.c2v_knn_topk_workspace_bytes(N, H, Q, k) for k in (1, 5, 16)] for Q in (1, 37, 2048)]
            assert all(x > 0 for r in t for x in r)
            assert all(r == sorted(r) for r in t) and all(list(c) == sorted(c) for c in zip(*t))
            p = [lib.c2v_knn_pairs_workspace_bytes(N, H, Q) for Q in (1, 37, 2048)]
            assert p == sorted(p) and all(x > 0 for x in p) and p[-1] <= t[-1][0]
        assert [lib.c2v_knn_topk_workspace_bytes(N, H, 2048, 16) for N in (1, 129, 10 ** 6, 10 ** 7)] == \
            sorted(lib.c2v_knn_topk_workspace_bytes(N, H, 2048, 16) for N in (1, 129, 10 ** 6, 10 ** 7))
    assert lib.c2v_knn_topk_workspace_bytes(1000, 128, 2049, 4) == 0
    assert lib.c2v_knn_topk_workspace_bytes(1000, 128, 8, _lib.TOPK_MAX + 1) == 0
    assert lib.c2v_knn_pairs_workspace_bytes(1000, 130, 8) == 0
    assert lib.c2v_knn_prep_workspace_bytes((1 << 32) - 1, 128) == 0
    assert lib.c2v_knn_prep_workspace_bytes((1 << 32) - 2, 128) > 0


# ---- the vector file ---------------------------------------------------------------------------------------------------
SPECIAL = np.array([-0.0, 0.0, 1e-45, 1.4e-45, 1.17549435e-38, 5e-40, -3.4028235e38, np.inf, -np.inf, np.nan, 1.0 / 3, 1e-5,
                    123456789.0, -2.5e-7, 1e16, 1.5e16], np.float32)


def _vectors(n, H, seed):
    rng = np.random.default_rng(seed)
    v = (rng.standard_normal((n, H)) * 10.0 ** rng.integers(-8, 8, (n, H))).astype(np.float32)
    v.reshape(-1)[:SPECIAL.size] = SPECIAL
    return v


def _same_bits(a, b):
    assert a.shape == b.shape and a.dtype == b.dtype == np.float32
    nan = np.isnan(a)
    assert np.array_equal(nan, np.isnan(b))
    assert np.array_equal(a.view(np.uint32)[~nan], b.view(np.uint32)[~nan])


@pytest.mark.parametrize("header", [True, False])
def test_vector_file_round_trip_is_bit_exact(tmp_path, header):
    names = ["get", "set name", "ünïcode", "x"]
    v = _vectors(37, 12, 1)
    lab = np.arange(37) % len(names)
    p = tmp_path / "vectors.txt"
    corpus.write_code_vectors(p, "w", v, lab, names, header_items=37 if header else None)
    got, got_names, items = corpus.read_code_vectors(p)
    _same_bits(got, v)
    assert got_names == [names[i] for i in lab] and items == (37 if header else None)
    got2, _, items2 = corpus.read_code_vectors(p, header=header)
    _same_bits(got2, v)
    assert items2 == items


def test_vector_file_two_writes_in_append_mode(tmp_path):
    a, b = _vectors(5, 8, 2), _vectors(9, 8, 3)
    p = tmp_path / "vectors.txt"
    corpus.write_code_vectors(p, "w", a, np.zeros(5, np.int64), ["a"], header_items=1000)    # the count is not enforced
    corpus.write_code_vectors(p, "a", b, np.ones(9, np.int64), ["a", "b"])
    got, names, items = corpus.read_code_vectors(p)
    _same_bits(got, np.concatenate([a, b]))
    assert names == ["a"] * 5 + ["b"] * 9 and items == 1000


def test_vector_file_without_header_whose_first_name_is_a_number(tmp_path):
    p = tmp_path / "vectors.txt"
    p.write_text("3\t4.0 5.0\n7\t-0.0 1e-45\n")
    got, names, items = corpus.read_code_vectors(p)                 # "4.0 5.0" is not an integer: no header
    assert items is None and names == ["3", "7"] and got.shape == (2, 2)
    with pytest.raises(_lib.C2VError, match="line 1"):
        corpus.read_code_vectors(p, header=True)


@pytest.mark.parametrize("text,line", [("2\t3\na\t1.0 2.0 3.0\nb\t1.0 2.0\n", 3), ("a\t1.0 2.0\nb\t1.0 x\n", 2),
                                       ("a\t1.0 2.0\nno tab here\n", 2), ("2\t2\na\t1.0 2.0\n\nb\t1.0 2.0\n", 3),
                                       ("a\t1.0 2.0\nb\t1.0 2.0 3.0\n", 2), ("a\t\n", 1)])
def test_vector_file_malformed_line_reports_its_number(tmp_path, text, line):
    p = tmp_path / "bad.txt"
    p.write_text(text)
    with pytest.raises(_lib.C2VError, match=f"line {line}:"):
        corpus.read_code_vectors(p)


# ---- most_similar's host arithmetic ------------------------------------------------------------------------------------
@pytest.mark.parametrize("pos,neg", [([3], []), ([1, 4], [2]), ([], [0]), ([5, 5], [6, 7, 8])])
def test_analogy_query_matches_a_numpy_restatement(pos, neg):
    rng = np.random.default_rng(len(pos) * 10 + len(neg))
    v = rng.standard_normal((10, 16)).astype(np.float32)
    v[7] = 0.0                                                       # a zero row contributes a zero unit vector
    q, rows = similarity.analogy_query(torch.from_numpy(v), pos, neg)
    u = v.astype(np.float64) / np.maximum(np.linalg.norm(v.astype(np.float64), axis=1, keepdims=True), 1e-12)
    m = (u[pos].sum(0) - u[neg].sum(0)) / (len(pos) + len(neg))
    ref = m / max(np.linalg.norm(m), 1e-12)
    assert np.abs(q.numpy() - ref).max() <= 1e-6
    assert rows == list(pos) + list(neg)


def test_analogy_query_rejects_bad_rows():
    v = torch.zeros(4, 8)
    with pytest.raises(ValueError):
        similarity.analogy_query(v, [], [])
    with pytest.raises(IndexError):
        similarity.analogy_query(v, [4])
    with pytest.raises(IndexError):
        similarity.analogy_query(v, [0], [-1])

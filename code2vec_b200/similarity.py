"""Similarity search over code vectors (not in the reference): k nearest neighbours, the kNN graph, above-threshold pairs
and word2vec-style analogies, on the tensor cores (c2v_knn_topk / c2v_knn_pairs).  The [Q, N] similarity block is never
written: the label GEMM's epilogue keeps a running top-k per query, or writes only the pairs above the threshold.

    cos(q, b) = (q . b) / (max(|q|, 1e-12) max(|b|, 1e-12))       F.normalize's clamp: a zero vector scores 0

Results rank by similarity descending, then row ascending (torch.sort(descending=True, stable=True)).  Rows are the keys;
names (e.g. the labels of a vector file) are carried along for display only.

Shapes the kernels do not take -- k > _lib.TOPK_MAX, an encode size that is not a multiple of 4 or above 256 -- run
chunked torch (F.normalize, fp32 mm without TF32, stable sort) with the same semantics and a bounded block per chunk."""
import contextlib
import ctypes

import torch
import torch.nn.functional as F

from . import _lib
from .functional import REUSE_PREP, PrepCache, _empty, _ptr, _stream

CHUNK = _lib.KNN_MAX_Q                 # queries per kernel call
FALLBACK_BLOCK_ELEMS = 1 << 26         # torch fallback: at most this many [q, N] similarities per chunk (256 MB fp32)


@contextlib.contextmanager
def _fp32_matmul():
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def analogy_query(vectors, positive, negative=()):
    """-> (query [H], input rows): the unit vector of the mean of +unit(v_r) over the positive rows and -unit(v_r) over the
    negative rows (word2vec's `most_similar` arithmetic), and the rows it was built from (excluded from its results)."""
    pos, neg = [int(r) for r in positive], [int(r) for r in negative]
    rows = pos + neg
    if not rows:
        raise ValueError("most_similar needs at least one positive or negative row")
    n = vectors.shape[0]
    bad = [r for r in rows if not 0 <= r < n]
    if bad:
        raise IndexError(f"rows {bad} outside [0, {n})")
    idx = torch.tensor(rows, dtype=torch.int64, device=vectors.device)
    sign = torch.tensor([1.0] * len(pos) + [-1.0] * len(neg), dtype=torch.float32, device=vectors.device)
    mean = (F.normalize(vectors[idx], dim=1) * sign[:, None]).mean(0)
    return F.normalize(mean, dim=0), rows


class CodeVectorIndex:
    """Cosine similarity search over a bank of code vectors, CUDA fp32 [N, H] (kept by reference: an in-place change of
    the tensor is seen by the next query).  The bank's fp16 hi / lo image and row norms are built once, on the first query,
    and rebuilt only after the vectors change (keyed on data_ptr and the version counter, as the model's weight images)."""

    def __init__(self, vectors, names=None):
        if not isinstance(vectors, torch.Tensor) or not vectors.is_cuda or vectors.dtype != torch.float32 or vectors.dim() != 2:
            raise TypeError("CodeVectorIndex: vectors must be a float32 CUDA tensor [N, H]")
        if not vectors.is_contiguous():
            raise ValueError("CodeVectorIndex: vectors must be contiguous")
        N, H = vectors.shape
        if N < 1 or H < 1:
            raise ValueError(f"CodeVectorIndex: empty bank {tuple(vectors.shape)}")
        if names is not None:
            names = list(names)
            if len(names) != N:
                raise ValueError(f"CodeVectorIndex: {len(names)} names for {N} rows")
        self.vectors, self.names = vectors, names
        self.fused = _lib.load().c2v_knn_prep_workspace_bytes(N, H) > 0      # the kernels take this bank's shape
        self._cache = PrepCache()
        self.prep_builds = 0                   # how often the bank image was (re)built

    @classmethod
    def from_file(cls, path, device="cuda", header="auto"):
        """an index over a vector file (corpus.write_code_vectors' format), names = the file's names"""
        from .corpus import read_code_vectors
        vec, names, _ = read_code_vectors(path, header)
        return cls(torch.from_numpy(vec).to(device), names)

    @property
    def shape(self):
        return tuple(self.vectors.shape)

    def _prep(self):
        lib = _lib.load()
        N, H = self.shape
        buf, reuse = self._cache.get(lib.c2v_knn_prep_workspace_bytes(N, H), self.vectors.device, self.vectors)
        if not reuse:
            self.prep_builds += 1
        return buf, (REUSE_PREP if reuse else 0)

    def _queries(self, queries):
        if not isinstance(queries, torch.Tensor) or queries.dtype != torch.float32 or queries.device != self.vectors.device:
            raise TypeError(f"queries must be a float32 tensor on {self.vectors.device}")
        if queries.dim() != 2 or queries.shape[1] != self.shape[1]:
            raise ValueError(f"queries must be [Q, {self.shape[1]}], got {tuple(queries.shape)}")
        return queries.contiguous()

    def _exclude(self, exclude, Q):
        if exclude is None:
            return None
        ex = torch.as_tensor(exclude, dtype=torch.int64, device=self.vectors.device)
        if ex.dim() == 1:
            ex = ex[:, None]
        if ex.dim() != 2 or ex.shape[0] != Q:
            raise ValueError(f"exclude must be int64 [Q, X] with Q = {Q}, got {tuple(ex.shape)}")
        return ex.contiguous() if ex.shape[1] else None

    # ---- k nearest neighbours -----------------------------------------------------------------------------------------
    def search(self, queries, k=10, exclude=None):
        """-> (indices int64 [Q, k], sims fp32 [Q, k]): the k bank rows most similar to each query.  exclude: int64 [Q, X]
        rows never returned for that query (entries < 0 are ignored)."""
        q = self._queries(queries)
        Q, (N, H), k = q.shape[0], self.shape, int(k)
        ex = self._exclude(exclude, Q)
        X = 0 if ex is None else ex.shape[1]
        if not 1 <= k <= N - X:
            raise ValueError(f"k = {k}: needs 1 <= k <= N - X = {N - X}")
        dev = q.device
        idx = _empty((Q, k), torch.int64, dev)
        sims = _empty((Q, k), torch.float32, dev)
        if Q == 0:
            return idx, sims
        if self.fused and k <= _lib.TOPK_MAX and X <= _lib.KNN_EXCLUDE_MAX:
            lib = _lib.load()
            with torch.cuda.device(dev):
                for lo in range(0, Q, CHUNK):
                    hi = min(Q, lo + CHUNK)
                    prep, flags = self._prep()
                    nbytes = lib.c2v_knn_topk_workspace_bytes(N, H, hi - lo, k)
                    ws = _empty((nbytes,), torch.uint8, dev)
                    qc, ec = q[lo:hi], (ex[lo:hi] if ex is not None else None)
                    rc = lib.c2v_knn_topk(_ptr(self.vectors), N, H, _ptr(qc), hi - lo, k, _ptr(ec), X, _ptr(idx[lo:hi]),
                                          _ptr(sims[lo:hi]), _ptr(prep), prep.numel(), _ptr(ws), nbytes, flags, _stream(dev))
                    _lib.check(rc, "c2v_knn_topk")
            return idx, sims
        bank = F.normalize(self.vectors, dim=1)
        step = max(1, min(CHUNK, FALLBACK_BLOCK_ELEMS // N))
        with _fp32_matmul():
            for lo in range(0, Q, step):
                hi = min(Q, lo + step)
                s = F.normalize(q[lo:hi], dim=1) @ bank.T
                if ex is not None:
                    e = ex[lo:hi]
                    r, c = ((e >= 0) & (e < N)).nonzero(as_tuple=True)
                    s[r, e[r, c]] = -float("inf")
                v, i = torch.sort(s, dim=1, descending=True, stable=True)
                idx[lo:hi], sims[lo:hi] = i[:, :k], v[:, :k]
        return idx, sims

    def neighbours(self, rows, k=10):
        """search() of bank rows, each left out of its own list -> (indices [R, k], sims [R, k])"""
        rows = torch.as_tensor(rows, dtype=torch.int64, device=self.vectors.device).reshape(-1)
        if rows.numel() and (int(rows.min()) < 0 or int(rows.max()) >= self.shape[0]):
            raise IndexError(f"rows outside [0, {self.shape[0]})")
        return self.search(self.vectors[rows], k, exclude=rows[:, None])

    def knn_graph(self, k=10):
        """the k nearest neighbours of every row, itself excluded -> (indices [N, k], sims [N, k])"""
        return self.neighbours(torch.arange(self.shape[0], device=self.vectors.device), k)

    # ---- pairs above a threshold --------------------------------------------------------------------------------------
    def pairs(self, threshold, rows=None, capacity=None):
        """Every pair with cos >= threshold -> (i int64 [P], j int64 [P], sim fp32 [P]) sorted by (i, -sim, j).
        rows=None: the self-join of the bank, each unordered pair once with i < j.  rows given: (i, j) for i in rows and
        every other bank row j.  capacity: the first guess of the pair count (the kernel counts exactly; one re-run with
        the exact size on overflow)."""
        N, H = self.shape
        dev = self.vectors.device
        thr = float(threshold)
        if thr != thr:
            raise ValueError("threshold is NaN")
        if rows is None:
            q_rows, self_join = None, True
            Q = N
        else:
            q_rows = torch.as_tensor(rows, dtype=torch.int64, device=dev).reshape(-1)
            if q_rows.numel() and (int(q_rows.min()) < 0 or int(q_rows.max()) >= N):
                raise IndexError(f"rows outside [0, {N})")
            self_join, Q = False, q_rows.numel()
        if Q == 0:
            e = torch.empty(0, dtype=torch.int64, device=dev)
            return e, e.clone(), torch.empty(0, dtype=torch.float32, device=dev)
        queries = self.vectors if self_join else self.vectors[q_rows]
        if self.fused:
            qi, j, s = self._pairs_fused(queries, thr, q_rows, self_join, capacity)
        else:
            qi, j, s = self._pairs_torch(queries, thr, q_rows, self_join)
        i = qi if self_join else q_rows[qi]
        o = torch.argsort(j, stable=True)
        i, j, s = i[o], j[o], s[o]
        o = torch.argsort(-s, stable=True)
        i, j, s = i[o], j[o], s[o]
        o = torch.argsort(i, stable=True)
        return i[o], j[o], s[o]

    def _pairs_fused(self, queries, thr, q_rows, self_join, capacity):
        lib = _lib.load()
        N, H = self.shape
        Q, dev = queries.shape[0], queries.device
        cap = int(capacity) if capacity is not None else max(1 << 16, 4 * Q)
        with torch.cuda.device(dev):
            for attempt in range(2):
                count = torch.zeros(1, dtype=torch.int64, device=dev)
                pq = _empty((cap,), torch.int64, dev)
                pi = _empty((cap,), torch.int64, dev)
                ps = _empty((cap,), torch.float32, dev)
                for lo in range(0, Q, CHUNK):
                    hi = min(Q, lo + CHUNK)
                    prep, flags = self._prep()
                    nbytes = lib.c2v_knn_pairs_workspace_bytes(N, H, hi - lo)
                    ws = _empty((nbytes,), torch.uint8, dev)
                    ec = None if self_join else q_rows[lo:hi, None].contiguous()
                    rc = lib.c2v_knn_pairs(_ptr(self.vectors), N, H, _ptr(queries[lo:hi]), hi - lo, ctypes.c_float(thr),
                                           _ptr(ec), 0 if ec is None else 1, lo if self_join else -1, lo, cap, _ptr(pq),
                                           _ptr(pi), _ptr(ps), _ptr(count), _ptr(prep), prep.numel(), _ptr(ws), nbytes, flags,
                                           _stream(dev))
                    _lib.check(rc, "c2v_knn_pairs")
                n = int(count.item())
                if n <= cap:
                    return pq[:n], pi[:n], ps[:n]
                cap = n                                    # overflow: the count is exact, so one re-run fits
        raise AssertionError("unreachable")

    def _pairs_torch(self, queries, thr, q_rows, self_join):
        N = self.shape[0]
        bank = F.normalize(self.vectors, dim=1)
        step = max(1, min(CHUNK, FALLBACK_BLOCK_ELEMS // N))
        out = []
        cols = torch.arange(N, device=queries.device)
        with _fp32_matmul():
            for lo in range(0, queries.shape[0], step):
                hi = min(queries.shape[0], lo + step)
                s = F.normalize(queries[lo:hi], dim=1) @ bank.T
                keep = s >= thr
                r = torch.arange(lo, hi, device=queries.device)
                if self_join:
                    keep &= cols[None, :] > r[:, None]
                else:
                    keep[torch.arange(hi - lo, device=queries.device), q_rows[lo:hi]] = False
                a, b = keep.nonzero(as_tuple=True)
                out.append((a + lo, b, s[a, b]))
        return tuple(torch.cat(x) for x in zip(*out))

    # ---- analogies ----------------------------------------------------------------------------------------------------
    def most_similar(self, positive, negative=(), topn=10):
        """word2vec's most_similar over rows -> [(row, name or None, sim)], the input rows excluded"""
        q, rows = analogy_query(self.vectors, positive, negative)
        N = self.shape[0]
        uniq = sorted(set(rows))
        topn = int(topn)
        if not 1 <= topn <= N - len(uniq):
            raise ValueError(f"topn = {topn}: needs 1 <= topn <= {N - len(uniq)}")
        if len(uniq) <= _lib.KNN_EXCLUDE_MAX:
            idx, sims = self.search(q[None], topn, exclude=torch.tensor([uniq], dtype=torch.int64, device=q.device))
            pairs = list(zip(idx[0].tolist(), sims[0].tolist()))
        else:                                              # more inputs than the kernel excludes: drop them afterwards
            idx, sims = self.search(q[None], topn + len(uniq))
            pairs = [(r, s) for r, s in zip(idx[0].tolist(), sims[0].tolist()) if r not in set(uniq)][:topn]
        return [(r, self.names[r] if self.names is not None else None, s) for r, s in pairs]

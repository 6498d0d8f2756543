"""Similarity search over a code-vector bank (code2vec_b200.similarity), fused vs torch, alternating in one process:
  knn    the kNN graph (k = 10) over --chunks query chunks of 2048 bank rows, self excluded:
         fused  CodeVectorIndex.neighbours (c2v_knn_topk: running top-k in the tensor-core GEMM's epilogue)
         torch  F.normalize + fp32 mm (allow_tf32 = False) into a [2048, N] block + torch.topk
  pairs  the self-join at tau = 0.95 over the same query chunks (pairs with i < j):
         fused  c2v_knn_pairs (only the matches are written)
         torch  the same [2048, N] block + (s >= tau) & (j > i) + nonzero
The bank is realistic: predict() code vectors of a bench.synth_params model over bench.synth_pool bags (N = --n per
workload, cfg2 at H = 128 and cfg3 at H = 100).  Before timing, the fused and torch results are checked against each other
(tie-aware: wherever they differ, the fp64 cosines of the differing entries agree within 1e-5).  Every shape is warmed up
first; each JSON line gives the median and the p10 - p90 spread of the per-call times (CUDA events) and the card's name /
power limit / max SM clock from the same run.

    python scripts/time_knn.py [--workloads cfg2,cfg3] [--n 1000000] [--chunks 4] [--steps 10] [--warmup 2]
"""
import argparse
import json
import os
import sys
import types

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench import WORKLOADS, synth_params, synth_pool  # noqa: E402
from code2vec_b200.model import Code2Vec  # noqa: E402
from code2vec_b200.similarity import CHUNK, CodeVectorIndex  # noqa: E402
from scripts.time_angular import card  # noqa: E402

K, TAU = 10, 0.95


def code_vector_bank(w, n, dev):
    o = types.SimpleNamespace(terminal_count=w["T"], path_count=w["P"], label_count=w["C"], terminal_embed_size=w["Et"],
                              path_embed_size=w["Ep"], encode_size=w["H"], dropout_prob=0.0, angular_margin_loss=False,
                              angular_margin=0.5, inverse_temp=30.0, device=dev)
    m = Code2Vec(o)
    m.load_state_dict(synth_params(w, dev))
    m = m.to(dev).eval()
    out, B = [], w["B"]
    with torch.no_grad():
        for i in range((n + B - 1) // B):
            s, p, e, _ = synth_pool(w, 1, dev, 1000 + i)
            out.append(m.predict(s, p, e)[2])
    bank = torch.cat(out)[:n].contiguous()
    del m, out
    torch.cuda.empty_cache()
    return bank


def torch_block(bank_n, lo, hi):
    with torch.no_grad():
        torch.backends.cuda.matmul.allow_tf32 = False
        return bank_n[lo:hi] @ bank_n.T


def torch_knn(bank_n, lo, hi):
    s = torch_block(bank_n, lo, hi)
    s[torch.arange(hi - lo, device=s.device), torch.arange(lo, hi, device=s.device)] = -float("inf")
    v, i = torch.topk(s, K, dim=1)
    return i, v


def torch_pairs(bank_n, lo, hi):
    s = torch_block(bank_n, lo, hi)
    cols = torch.arange(bank_n.shape[0], device=s.device)
    keep = (s >= TAU) & (cols[None, :] > torch.arange(lo, hi, device=s.device)[:, None])
    a, b = keep.nonzero(as_tuple=True)
    return a + lo, b, s[a, b]


def check(index, bank, bank_n, chunks):
    """tie-aware agreement of the two ways on the timed chunks"""
    worst, n_diff, pairs_torch = 0.0, 0, 0
    b64 = F.normalize(bank.double(), dim=1)
    for c in range(chunks):
        lo, hi = c * CHUNK, (c + 1) * CHUNK
        fi, fs = index.neighbours(torch.arange(lo, hi, device=bank.device), K)
        ti, ts = torch_knn(bank_n, lo, hi)
        diff = fi != ti
        n_diff += int(diff.sum())
        q64 = b64[lo:hi]
        c_f = (q64[:, None, :] * b64[fi]).sum(-1)
        c_t = (q64[:, None, :] * b64[ti]).sum(-1)
        worst = max(worst, (c_f - c_t).abs().max().item())
        pairs_torch += torch_pairs(bank_n, lo, hi)[0].numel()
    buf = pair_buffers(index, 1 << 22)
    pairs_fused = sum(int(fused_pairs(index, c * CHUNK, (c + 1) * CHUNK, buf).item()) for c in range(chunks))
    return {"knn_entries_differing": n_diff, "knn_max_fp64_gap_where_differing": worst,
            "pairs_fused": pairs_fused, "pairs_torch": pairs_torch}


def fused_pairs(index, lo, hi, cap_holder):
    import ctypes
    from code2vec_b200 import _lib
    from code2vec_b200.functional import _ptr, _stream
    lib = _lib.load()
    N, H = index.shape
    prep, flags = index._prep()
    ws, count, out = cap_holder
    count.zero_()
    rc = lib.c2v_knn_pairs(_ptr(index.vectors), N, H, _ptr(index.vectors[lo:hi]), hi - lo, ctypes.c_float(TAU), None, 0, lo,
                           lo, out[0].numel(), _ptr(out[0]), _ptr(out[1]), _ptr(out[2]), _ptr(count), _ptr(prep), prep.numel(),
                           _ptr(ws), ws.numel(), flags, _stream(index.vectors.device))
    _lib.check(rc, "c2v_knn_pairs")
    return count


def pair_buffers(index, cap):
    from code2vec_b200 import _lib
    N, H = index.shape
    dev = index.vectors.device
    ws = torch.empty(_lib.load().c2v_knn_pairs_workspace_bytes(N, H, CHUNK), dtype=torch.uint8, device=dev)
    return ws, torch.zeros(1, dtype=torch.int64, device=dev), [torch.empty(cap, dtype=dt, device=dev) for dt in
                                                                (torch.int64, torch.int64, torch.float32)]


def timed(fn, steps, warmup):
    ts = []
    for i in range(warmup + steps):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        if i >= warmup:
            ts.append(e0.elapsed_time(e1))
    return ts


def stats(ts):
    s = sorted(ts)
    q = lambda f: s[min(len(s) - 1, int(f * (len(s) - 1) + 0.5))]
    return {"median_ms": round(q(0.5), 3), "p10_ms": round(q(0.1), 3), "p90_ms": round(q(0.9), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg2,cfg3")
    ap.add_argument("--n", type=int, default=10 ** 6)
    ap.add_argument("--chunks", type=int, default=4, help="query chunks of 2048 rows per timed call")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_knn.py measures on the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    for name in args.workloads.split(","):
        w = dict(WORKLOADS[name])
        bank = code_vector_bank(w, args.n, dev)
        index = CodeVectorIndex(bank)
        bank_n = F.normalize(bank, dim=1)
        chk = check(index, bank, bank_n, args.chunks)
        if chk["knn_max_fp64_gap_where_differing"] > 1e-5 or abs(chk["pairs_fused"] - chk["pairs_torch"]) > max(
                10, chk["pairs_torch"] // 10000):
            raise SystemExit(f"{name}: fused and torch disagree: {chk}")
        buf = pair_buffers(index, 1 << 22)
        rows = [torch.arange(c * CHUNK, (c + 1) * CHUNK, device=dev)[:, None] for c in range(args.chunks)]
        ways = {
            "knn_fused": lambda: [index.search(bank[r[:, 0]], K, exclude=r) for r in rows],
            "knn_torch": lambda: [torch_knn(bank_n, c * CHUNK, (c + 1) * CHUNK) for c in range(args.chunks)],
            "pairs_fused": lambda: [fused_pairs(index, c * CHUNK, (c + 1) * CHUNK, buf) for c in range(args.chunks)],
            "pairs_torch": lambda: [torch_pairs(bank_n, c * CHUNK, (c + 1) * CHUNK) for c in range(args.chunks)],
        }
        for fn in ways.values():                   # warm up every shape before any timed window
            fn()
        times = {k: [] for k in ways}
        for _ in range(args.steps):                # alternate the ways, one timed call each per round
            for k, fn in ways.items():
                times[k] += timed(fn, 1, 0)
        st = {k: stats(v) for k, v in times.items()}
        print(json.dumps({"workload": name, "N": args.n, "H": w["H"], "queries_per_call": args.chunks * CHUNK, "k": K, "tau": TAU,
                          "steps": args.steps, **st,
                          "knn_speedup": round(st["knn_torch"]["median_ms"] / st["knn_fused"]["median_ms"], 2),
                          "pairs_speedup": round(st["pairs_torch"]["median_ms"] / st["pairs_fused"]["median_ms"], 2),
                          "check": chk, "card": info}), flush=True)
        del index, bank, bank_n, buf
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

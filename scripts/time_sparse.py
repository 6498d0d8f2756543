"""Dense vs sparse embedding gradients on the training step, one process, one GPU.

    python scripts/time_sparse.py [--steps 20] [--workloads cfg2,cfg3,big] [--dists uniform,zipf] [--out DIR]

dense   ddp_step(model, ShardedFlatAdam(all parameters), world size 1, fused loss): the default training step
sparse  terminal_embedding.sparse = path_embedding.sparse = True, FusedSparseAdam on the two tables, ShardedFlatAdam
        on the rest: forward_loss, backward, dense.step(), sparse.step(), sparse.zero_grad() -- INTEGRATION.md's recipe
        as written (Code2Vec.fuse_grad_accumulation left off)
Workloads: bench.py's cfg2 and cfg3, and "big" (2 x 10^6 rows per table, E = H = 128, C = 8192, B = 1024, L = 200);
indices uniform over the table or Zipf(1.2)-distributed, full bags.  Before timing, the sparse gradient of each table
is checked against the dense one on the same inputs.  The two steps alternate; each step is timed with CUDA events
around it (the sparse step's one host wait, for U, is inside the window), reported as median and p10-p90.  Also timed:
FusedSparseAdam against torch.optim.SparseAdam on the same gradients, and the host time the backward spends waiting
for U.  Prints one JSON document (also written to DIR/time_sparse.json) with the card's name, power limit and max SM
clock, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time
import zlib
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import WORKLOADS, synth_params                              # noqa: E402
from code2vec_b200.distributed import FusedSparseAdam, ShardedFlatAdam, ddp_step   # noqa: E402
from code2vec_b200.model import Code2Vec                               # noqa: E402

WL = {"cfg2": WORKLOADS["cfg2"], "cfg3": WORKLOADS["cfg3"],
      "big": dict(T=2000000, P=2000000, C=8192, Et=128, Ep=128, H=128, B=1024, L=200)}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def batches(w, dist, n, dev, seed):
    rng = np.random.default_rng(seed)
    B, L = w["B"], w["L"]

    def draw(vocab):
        if dist == "uniform":
            return rng.integers(1, vocab, (n, B, L))
        return np.minimum(rng.zipf(1.2, (n, B, L)), vocab - 1)
    s, p, e = draw(w["T"]), draw(w["P"]), draw(w["T"])
    lab = rng.integers(0, w["C"], (n, B))
    t = lambda a: torch.from_numpy(a.astype(np.int64)).to(dev)
    return [(t(s[i]), t(p[i]), t(e[i]), t(lab[i])) for i in range(n)]


def model(w, params, dev, sparse):
    o = types.SimpleNamespace(terminal_count=w["T"], path_count=w["P"], label_count=w["C"], terminal_embed_size=w["Et"],
                              path_embed_size=w["Ep"], encode_size=w["H"], dropout_prob=0.25, angular_margin_loss=False,
                              angular_margin=0.5, inverse_temp=30.0, device=dev)
    m = Code2Vec(o)
    m.load_state_dict(params)
    m = m.to(dev).train()
    m.terminal_embedding.sparse = m.path_embedding.sparse = sparse
    return m


def stats(ts):
    a = np.array(ts) * 1e3
    return {"median_ms": float(np.median(a)), "p10_ms": float(np.percentile(a, 10)), "p90_ms": float(np.percentile(a, 90))}


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()                          # (not Event.synchronize: WaitClock counts those)
    return a.elapsed_time(b) / 1e3


class WaitClock:
    """host seconds spent in torch.cuda.Event.synchronize (the sparse backward's wait for U is the only caller)"""

    def __init__(self):
        self.t, self.orig = 0.0, torch.cuda.Event.synchronize
        clock = self

        def sync(ev):
            t0 = time.perf_counter()
            clock.orig(ev)
            clock.t += time.perf_counter() - t0
        torch.cuda.Event.synchronize = sync


def run(name, dist, steps, dev, wait):
    w = WL[name]
    params = synth_params(w, dev)
    data = batches(w, dist, 4, dev, seed=zlib.crc32(f"{name}{dist}".encode()))
    res = {"workload": name, "dist": dist, "shape": {k: w[k] for k in ("T", "P", "C", "Et", "Ep", "H", "B", "L")}}

    # ---- the sparse gradient equals the dense one on the same inputs (same seed -> same dropout mask)
    md, ms = model(w, params, dev, False), model(w, params, dev, True)
    for m in (md, ms):
        torch.manual_seed(1)
        m.forward_loss(*data[0])[0].backward()
    worst = 0.0
    for td, ts in ((md.terminal_embedding.weight, ms.terminal_embedding.weight),
                   (md.path_embedding.weight, ms.path_embedding.weight)):
        g = ts.grad
        assert g.is_sparse and g.is_coalesced()
        rows = g.indices()[0]
        ref = td.grad[rows]
        err = float((g.values() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
        outside = td.grad.clone()
        outside[rows] = 0
        assert float(outside.abs().max()) == 0.0, "dense gradient outside the sparse rows"
        worst = max(worst, err)
    assert worst < 1e-4, f"sparse gradient differs from the dense one: {worst}"
    res["max_rel_diff_sparse_vs_dense"] = worst
    res["U"] = {"terminal": int(ms.terminal_embedding.weight.grad._nnz()), "path": int(ms.path_embedding.weight.grad._nnz())}
    res["rows"] = {"terminal": w["T"], "path": w["P"]}

    # ---- FusedSparseAdam against torch.optim.SparseAdam on the same gradients
    tables = [ms.terminal_embedding.weight, ms.path_embedding.weight]
    grads = [t.grad for t in tables]
    for cls in (FusedSparseAdam, torch.optim.SparseAdam):
        copies = [torch.nn.Parameter(t.detach().clone()) for t in tables]
        opt = cls(copies, lr=1e-3)
        ts_ = []
        for i in range(max(steps, 5) + 2):
            for c, g in zip(copies, grads):
                c.grad = g
            ts_.append(timed(opt.step))
        res[f"optimizer_{cls.__name__}"] = stats(ts_[2:])
        del copies, opt
    for t in tables:
        t.grad = None
    md.zero_grad(set_to_none=True)

    # ---- the two training steps, alternating
    dense_opt = ShardedFlatAdam(md.parameters(), lr=0.01)
    rest = [p for p in ms.parameters() if all(p is not t for t in tables)]
    rest_opt, sparse_opt = ShardedFlatAdam(rest, lr=0.01), FusedSparseAdam(tables, lr=0.01)
    # the recipe of INTEGRATION.md as written: fuse_grad_accumulation stays off (only ddp_step switches it on), so autograd
    # adds input_linear's gradient into its bucket view

    def dense_step(b):
        ddp_step(md, dense_opt, None, *b[:3], b[3], None)

    def sparse_step(b):
        loss = ms.forward_loss(*b)[0]
        loss.backward()
        rest_opt.step()
        sparse_opt.step()
        sparse_opt.zero_grad()

    for i in range(3):                                # warm-up of both
        dense_step(data[i % 4]); sparse_step(data[i % 4])
    torch.cuda.synchronize()
    td_, ts_, waits = [], [], []
    peak = {}
    for i in range(steps):
        b = data[i % 4]
        torch.cuda.reset_peak_memory_stats(dev)
        td_.append(timed(lambda: dense_step(b)))
        peak["dense"] = max(peak.get("dense", 0), torch.cuda.max_memory_allocated(dev))
        torch.cuda.reset_peak_memory_stats(dev)
        w0 = wait.t
        ts_.append(timed(lambda: sparse_step(b)))
        waits.append(wait.t - w0)
        peak["sparse"] = max(peak.get("sparse", 0), torch.cuda.max_memory_allocated(dev))
    res["dense_step"], res["sparse_step"] = stats(td_), stats(ts_)
    res["sparse_host_wait_for_U"] = stats(waits)
    res["speedup_median"] = res["dense_step"]["median_ms"] / res["sparse_step"]["median_ms"]
    res["peak_allocated_GB_during_step"] = {k: v / 1e9 for k, v in peak.items()}
    del md, ms, dense_opt, rest_opt, sparse_opt, tables, grads, rest, data, params
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--workloads", default="cfg2,cfg3,big")
    ap.add_argument("--dists", default="uniform,zipf")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_sparse.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    wait = WaitClock()
    out = {"gpu": gpu_info(), "torch": torch.__version__, "steps": a.steps, "results": []}
    for name in a.workloads.split(","):
        for dist in a.dists.split(","):
            r = run(name, dist, a.steps, dev, wait)
            print(json.dumps(r), flush=True)
            out["results"].append(r)
    out["gpu_after"] = gpu_info()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_sparse.json"), "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps({"gpu": out["gpu"], "gpu_after": out["gpu_after"]}))


if __name__ == "__main__":
    main()

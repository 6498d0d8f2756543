"""The device work of FusedSparseAdam's data-parallel step, one process, one GPU, on W emulated ranks' gathered lists.

    python scripts/time_sparse_ddp.py [--iters 30] [--worlds 2,4,8] [--out DIR]

For each case, W row lists per table are drawn with the per-rank row counts U that README.md's sparse table measured
(one rank's batch of 1,024 bags): cfg2 (T = 360,633, P = 342,846) and 2 x 10^6 rows per table, E = 128, indices uniform
or Zipf(1.2) (U distinct rows per rank drawn without replacement, weights 1 / row^1.2).  Then, alternating in one
process on the same gathered lists [W, U_max] / [W, U_max, E]:
  merged  c2v_sparse_union_rows + c2v_sparse_adam_step_merged (what FusedSparseAdam runs after the all-gathers)
  torch   cat of the valid rows + coalesce() + * (1/W) + torch.optim.SparseAdam.step()
timed with CUDA events around both tables, median and p10-p90.  Also reported, computed from the counts: the bytes each
rank exchanges, W * U_max * (E + 2) * 4 per table (rows and values all-gathered), against about 2 * rows * E * 4 for a
dense reduction of the tables.  The two results are checked to agree (allclose: the summation orders differ).  Prints
one JSON line per case and the card's name, power limit and max SM clock, read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from code2vec_b200 import functional as CF     # noqa: E402

E = 128
# (rows per table, U per rank) of README.md's "Sparse embedding gradients" table: terminal, path
CASES = {
    "cfg2 uniform": [(360633, 244586), (342846, 153922)],
    "cfg2 zipf": [(360633, 34810), (342846, 20975)],
    "2e6 uniform": [(2000000, 370154), (2000000, 194753)],
    "2e6 zipf": [(2000000, 43009), (2000000, 25187)],
}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def draw(rng, vocab, U, zipf):
    if not zipf:
        return np.sort(rng.choice(vocab, U, replace=False))
    keys = -1.2 * np.log(np.arange(1, vocab + 1)) + rng.gumbel(size=vocab)     # Gumbel top-U: weighted, no replacement
    return np.sort(np.argpartition(-keys, U)[:U])


def gathered(rng, vocab, U, W, zipf, dev):
    rows = torch.zeros((W, U), dtype=torch.int64, device=dev)
    for r in range(W):
        rows[r] = torch.from_numpy(draw(rng, vocab, U, zipf)).to(dev)
    values = torch.randn((W, U, E), device=dev) * 1e-3
    return rows, values, torch.full((W,), U, dtype=torch.int64, device=dev)


def stats(ts):
    a = np.array(ts)
    return {"median_ms": float(np.median(a)), "p10_ms": float(np.percentile(a, 10)), "p90_ms": float(np.percentile(a, 90))}


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def run(name, W, iters, dev):
    rng = np.random.default_rng(W)
    tables = []
    for vocab, U in CASES[name]:
        rows, values, counts = gathered(rng, vocab, U, W, "zipf" in name, dev)
        w0 = torch.randn((vocab, E), device=dev) * 0.1
        tables.append(dict(vocab=vocab, U=U, rows=rows, values=values, counts=counts,
                           mine=[w0.clone(), torch.zeros_like(w0), torch.zeros_like(w0)],
                           theirs=torch.nn.Parameter(w0.clone())))
    ref = torch.optim.SparseAdam([t["theirs"] for t in tables], lr=1e-3)
    inv = float(torch.tensor(1.0 / W, dtype=torch.float32))
    step = [0]

    def merged():
        step[0] += 1
        for t in tables:
            union, count = CF.sparse_union_rows(t["rows"], t["counts"], t["vocab"])
            CF.sparse_adam_step_merged(*t["mine"], t["values"], t["rows"], t["counts"], union, count, 1e-3, 0.9, 0.999,
                                       1e-8, step[0], inv)

    def torch_step():
        for t in tables:
            valid = torch.arange(t["rows"].shape[1], device=dev)[None, :] < t["counts"][:, None]
            g = torch.sparse_coo_tensor(t["rows"][valid][None], t["values"][valid], (t["vocab"], E))
            t["theirs"].grad = g.coalesce() * inv
        ref.step()

    for _ in range(3):
        merged(); torch_step()
    for t in tables:                                     # same inputs, same number of steps: the results agree
        assert torch.allclose(t["mine"][0], t["theirs"].detach(), rtol=1e-5, atol=1e-6), name
    tm, tt = [], []
    for _ in range(iters):
        tm.append(timed(merged)); tt.append(timed(torch_step))
    exchange = sum(W * t["U"] * (E + 2) * 4 for t in tables)
    dense = sum(2 * t["vocab"] * E * 4 for t in tables)
    return {"case": name, "world": W, "U_per_rank": [t["U"] for t in tables], "rows": [t["vocab"] for t in tables],
            "merged": stats(tm), "torch": stats(tt), "speedup_median": float(np.median(tt) / np.median(tm)),
            "exchange_bytes_per_rank": exchange, "dense_reduction_bytes_per_rank": dense}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--worlds", default="2,4,8")
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_sparse_ddp.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    out = {"gpu": gpu_info(), "torch": torch.__version__, "results": []}
    for name in a.cases.split(","):
        for W in (int(x) for x in a.worlds.split(",")):
            r = run(name, W, a.iters, dev)
            print(json.dumps(r), flush=True)
            out["results"].append(r)
            torch.cuda.empty_cache()
    out["gpu_after"] = gpu_info()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_sparse_ddp.json"), "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps({"gpu": out["gpu"], "gpu_after": out["gpu_after"]}))


if __name__ == "__main__":
    main()

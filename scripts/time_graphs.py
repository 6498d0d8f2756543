"""Eager against CUDA-graph replay of the training step and of predict(), one process, one GPU.

    python scripts/time_graphs.py [--steps 30] [--batches 32,128,1024] [--workloads cfg2,cfg3,small] [--out DIR]

train    Code2Vec with dropout 0.25 and use_device_rng(), FlatAdam(capturable=True), fused loss (forward_loss): ddp_step
         eagerly, against GraphedTrainStep
predict  Code2Vec.predict() eagerly, against GraphedPredict
Workloads: bench.py's cfg2 and cfg3, and "small", the reference's defaults (E = H = 100, T = P = 50,000, C = 1,000), each
at B in --batches and L = 200.  Eager and graphed rounds alternate in one process.  Per case: median and p10-p90 step
time from CUDA events around each step and from a host clock ending in a synchronise, the host time spent enqueueing
(the host clock before the synchronise), c2v_launch_count() per step, and torch.cuda.memory_reserved() after the
warm-up (and, graphed, the capture) of a fresh model minus before, a rough bound on the graph pool: it also counts what
the eager warm-up steps reserved or released.  Prints one JSON document (also written to
DIR/time_graphs.json) with the card's name, power limit and max SM clock, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import WORKLOADS, synth_params                              # noqa: E402
from code2vec_b200 import _lib                                         # noqa: E402
from code2vec_b200.distributed import FlatAdam, FlatGradBucket, ddp_step   # noqa: E402
from code2vec_b200.graphs import GraphedPredict, GraphedTrainStep      # noqa: E402
from code2vec_b200.model import Code2Vec                               # noqa: E402

WL = {"cfg2": WORKLOADS["cfg2"], "cfg3": WORKLOADS["cfg3"],
      "small": dict(T=50000, P=50000, C=1000, Et=100, Ep=100, H=100)}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def make_model(w, dev):
    o = types.SimpleNamespace(terminal_count=w["T"], path_count=w["P"], label_count=w["C"], terminal_embed_size=w["Et"],
                              path_embed_size=w["Ep"], encode_size=w["H"], dropout_prob=0.25, angular_margin_loss=False,
                              angular_margin=0.5, inverse_temp=30.0)
    m = Code2Vec(o)
    params = synth_params(dict(w, B=1, L=1), "cpu")
    m.load_state_dict({k: (v if isinstance(v, torch.Tensor) else torch.from_numpy(v)) for k, v in params.items()})
    return m.to(dev)


def batches(w, B, L, n, dev, seed):
    rng = np.random.default_rng(seed)
    t = lambda a: torch.from_numpy(a.astype(np.int64)).to(dev)
    return [(t(rng.integers(1, w["T"], (B, L))), t(rng.integers(1, w["P"], (B, L))), t(rng.integers(1, w["T"], (B, L))),
             t(rng.integers(0, w["C"], B))) for _ in range(n)]


def stats(v):
    v = np.asarray(v)
    return {"median": float(np.median(v)), "p10": float(np.percentile(v, 10)), "p90": float(np.percentile(v, 90))}


def time_round(fn, data, lib):
    ev, host, enq = [], [], []
    n0 = lib.c2v_launch_count()
    for b in data:
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        fn(*b)
        e1.record()
        t1 = time.perf_counter()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        ev.append(e0.elapsed_time(e1)); enq.append((t1 - t0) * 1e3); host.append((t2 - t0) * 1e3)
    return ev, host, enq, (lib.c2v_launch_count() - n0) / len(data)


def run_case(kind, w, B, L, steps, dev, lib):
    data = batches(w, B, L, steps, dev, seed=B)
    res = {}
    for mode in ("eager", "graph"):
        m = make_model(w, dev)
        if kind == "train":
            m.train().use_device_rng(seed=1)
            opt = FlatAdam(FlatGradBucket(m.parameters()), lr=1e-3, capturable=True)
            if mode == "eager":
                fn = lambda s, p, e, y, m=m, opt=opt: ddp_step(m, opt, opt.bucket, s, p, e, y, None)
            else:
                fn = GraphedTrainStep(m, opt, B, L)
        else:
            m.eval()
            f = m.predict if mode == "eager" else GraphedPredict(m, B, L)
            fn = lambda s, p, e, y, f=f: f(s, p, e)
        torch.cuda.synchronize()
        reserved = torch.cuda.memory_reserved()
        for b in data[:4]:                                   # warm-up (and, graphed, the capture)
            fn(*b)
        torch.cuda.synchronize()
        res[mode] = dict(pool_bytes=torch.cuda.memory_reserved() - reserved)
        res[mode]["fn"], res[mode]["model"] = fn, m
    rounds = {"eager": [[], [], [], []], "graph": [[], [], [], []]}
    for _ in range(3):                                       # alternate eager and graphed rounds
        for mode in ("eager", "graph"):
            ev, host, enq, launches = time_round(res[mode]["fn"], data, lib)
            r = rounds[mode]
            r[0] += ev; r[1] += host; r[2] += enq; r[3].append(launches)
    out = {}
    for mode in ("eager", "graph"):
        r = rounds[mode]
        out[mode] = {"event_ms": stats(r[0]), "host_ms": stats(r[1]), "enqueue_ms": stats(r[2]),
                     "launches_per_step": float(np.mean(r[3])), "extra_reserved_bytes": int(res[mode]["pool_bytes"])}
    out["speedup_host_clock"] = out["eager"]["host_ms"]["median"] / out["graph"]["host_ms"]["median"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--batches", default="32,128,1024")
    ap.add_argument("--workloads", default="cfg2,cfg3,small")
    ap.add_argument("--L", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_graphs.py measures on the GPU and needs one")
    lib = _lib.load()
    dev = torch.device("cuda:0")
    doc = {"gpu": gpu_info(), "L": a.L, "steps": a.steps, "cases": []}
    for wn in a.workloads.split(","):
        w = WL[wn]
        for B in (int(x) for x in a.batches.split(",")):
            for kind in ("train", "predict"):
                r = run_case(kind, w, B, a.L, a.steps, dev, lib)
                r.update(workload=wn, B=B, kind=kind)
                doc["cases"].append(r)
                print(json.dumps({k: r[k] for k in ("workload", "B", "kind", "speedup_host_clock")}), flush=True)
                torch.cuda.empty_cache()
    print(json.dumps(doc))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_graphs.json"), "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()

"""Packed (CSR) against padded [B, L] batches on one GPU: a training step (forward_loss + backward + ShardedFlatAdam step,
bench.py's training leg) and predict(), at the cfg2 and cfg3 shapes of bench.py, for three bag-length distributions:
(a) every bag full (no padding to remove), (b) lengths uniform in [1, L], (c) about 34 % mean fill (geometric lengths),
(d) very short bags, lengths uniform in [1, 4]: one 16-row slice of the tensor-core encode then spans up to 16 bags, the
worst case of its per-bag epilogue loop.

First checks, per shape and distribution, that both layouts give the same loss and gradients (same parameters, same
dropout seed).  Then alternates padded and packed in one process and reports the median of --rounds rounds of each, with
the card name and power limit read in the same run.

    python scripts/time_packed.py [--rounds 20] [--workloads cfg2,cfg3] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import WORKLOADS, synth_params  # noqa: E402
from code2vec_b200 import functional as CF  # noqa: E402
from code2vec_b200.distributed import ShardedFlatAdam, ddp_step  # noqa: E402
from code2vec_b200.model import Code2Vec  # noqa: E402

DROPOUT = 0.25


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name(0)


def lengths(dist, B, L, rng):
    if dist == "full":
        return np.full(B, L, np.int64)
    if dist == "uniform":
        return rng.integers(1, L + 1, B)
    if dist == "short":
        return rng.integers(1, 5, B)
    return np.clip(rng.geometric(1.0 / 72, B), 1, L)        # "fill34": ~34 % of B * L after the clip at L


def batch(w, n, rng, dev):
    B, L = w["B"], w["L"]
    valid = np.arange(L)[None, :] < n[:, None]
    pad = [torch.from_numpy(rng.integers(1, hi, (B, L)) * valid).to(dev) for hi in (w["T"], w["P"], w["T"])]
    off = np.zeros(B + 1, np.int64)
    np.cumsum(n, out=off[1:])
    flat = torch.from_numpy(np.flatnonzero(valid.reshape(-1))).to(dev)
    bags = CF.PackedBags(*(t.reshape(-1)[flat].contiguous() for t in pad), off, L)
    return tuple(pad), bags, torch.from_numpy(rng.integers(0, w["C"], B)).to(dev)


def model(w, dev):
    o = types.SimpleNamespace(terminal_count=w["T"], path_count=w["P"], label_count=w["C"], terminal_embed_size=w["Et"],
                              path_embed_size=w["Ep"], encode_size=w["H"], dropout_prob=DROPOUT, angular_margin_loss=False,
                              angular_margin=0.5, inverse_temp=30.0, device=dev)
    m = Code2Vec(o)
    m.load_state_dict(synth_params(w, dev))
    return m.to(dev)


def check_same(m, pad, bags, label):
    """loss and every gradient of one step in both layouts at one dropout seed -> max relative differences"""
    out = {}
    m.train()
    m._next_seed = lambda: 12345
    for name, inputs in (("padded", pad), ("packed", (bags, None, None))):
        m.zero_grad(set_to_none=True)
        loss = m.forward_loss(*inputs, label)[0]
        loss.backward()
        out[name] = (float(loss.detach()), {k: p.grad.clone() for k, p in m.named_parameters()})
    del m._next_seed
    (l0, g0), (l1, g1) = out["padded"], out["packed"]
    res = {"loss_rel": abs(l1 - l0) / abs(l0)}
    for k in g0:
        res[k] = float((g1[k] - g0[k]).abs().max() / g0[k].abs().max().clamp_min(1e-30))
    m.zero_grad(set_to_none=True)
    return res


def timed(fn, sync_dev):
    torch.cuda.synchronize(sync_dev)
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize(sync_dev)
    return (time.perf_counter() - t) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=20)
    ap.add_argument("--workloads", default="cfg2,cfg3")
    ap.add_argument("--dists", default="full,uniform,fill34,short")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    result = {"card": card(), "rounds": args.rounds, "cases": []}
    print(result["card"], flush=True)
    for wname in args.workloads.split(","):
        w = dict(WORKLOADS[wname])
        m = model(w, dev)
        cases = []
        for dist in args.dists.split(","):
            rng = np.random.default_rng(1)
            pad, bags, label = batch(w, lengths(dist, w["B"], w["L"], rng), rng, dev)
            same = check_same(m, pad, bags, label)
            bad = {k: v for k, v in same.items() if v > (1e-5 if k == "loss_rel" else 1e-3)}
            if bad:
                raise SystemExit(f"{wname} {dist}: packed and padded differ: {bad}")
            cases.append(({"workload": wname, "dist": dist, "fill": bags.N / (w["B"] * w["L"]), "same": same},
                          {"padded": pad, "packed": (bags, None, None)}, label))
        opt = ShardedFlatAdam(m.parameters(), lr=1e-4)      # after the checks: it owns the .grad buffers from here on
        for case, inputs, label in cases:
            def train(layout):
                m.train()
                ddp_step(m, opt, None, *inputs[layout], label, None)

            def predict(layout):
                m.eval()
                m.predict(*inputs[layout])
            for leg, fn in (("train", train), ("predict", predict)):
                for layout in ("padded", "packed"):        # warm-up: workspaces, module loads, allocator
                    for _ in range(3):
                        fn(layout)
                t = {"padded": [], "packed": []}
                for _ in range(args.rounds):
                    for layout in ("padded", "packed"):
                        t[layout].append(timed(lambda: fn(layout), dev))
                med = {k: float(np.median(v)) for k, v in t.items()}
                case[leg] = {"padded_ms": med["padded"], "packed_ms": med["packed"],
                             "speedup": med["padded"] / med["packed"],
                             "padded_spread_ms": float(np.percentile(t["padded"], 90) - np.percentile(t["padded"], 10)),
                             "packed_spread_ms": float(np.percentile(t["packed"], 90) - np.percentile(t["packed"], 10))}
            print(json.dumps(case), flush=True)
            result["cases"].append(case)
        del m, opt, cases
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()

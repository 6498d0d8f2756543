"""Time the training step with the sampled-softmax loss against the full-vocabulary fused loss on the same card.

    python scripts/time_sampled.py [--steps 30] [--warmup 3] [--profile] [--out DIR]

Workloads (B = 1024, L = 200, cfg2's encoder vocabulary):
  * cfg3 (E = H = 100, C = 195,299) at S in {4,096, 8,192, 16,384};
  * the paper's 128 / 128 / 384 at C = 195,299 and S = 8,192;
  * cfg2 (E = H = 128, C = 8,192) at S in {1,024, 2,048}.
Both steps are ddp_step with ShardedFlatAdam and dropout 0.25 on their own copy of the same weights: `full` takes
Code2Vec.forward_loss, `sampled` Code2Vec.forward_sampled_loss with a Zipf proposal (counts 1/rank, power 0.75).  The
two alternate in one process on the same batches; each sample is one step between a device synchronise on either side.
Prints one JSON line per workload: median and p10 / p90 (ms) of both, with the card's name and power limit.
--profile instead runs each step alone under torch.profiler and prints its device time per part of the step.
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)
from bench import WORKLOADS, synth_params, synth_pool  # noqa: E402
from code2vec_b200 import functional as CF  # noqa: E402
from code2vec_b200.distributed import ShardedFlatAdam, ddp_step  # noqa: E402
from code2vec_b200.model import Code2Vec  # noqa: E402

DROPOUT = 0.25
# kernel-name substrings -> part of the step (first match wins)
PARTS = (("sampler", ("sampled_candidates", "sampled_gather")),
         ("sampled loss", ("sampled_row_lse", "sampled_mean", "sampled_dlogits")),
         ("scatter", ("scatter_keys", "scatter_rows", "RadixSort", "Onesweep", "fill", "Fill")),
         ("encode fwd", ("encode_ffma_kernel", "encode_wgmma_kernel", "finalize")),
         ("encode bwd", ("backward_rows", "bag_dot", "transpose_w", "row_bag", "backward_dw", "backward_dc_tc", "split_wt",
                         "wt_absmax")),
         ("Adam", ("adam",)),
         ("label head", ("sgemm", "gemm", "label", "loss", "reduce", "lse", "absmax", "split_rows")))
CASES = [("cfg3", {}, 4096), ("cfg3", {}, 8192), ("cfg3", {}, 16384),
         ("paper", {"Et": 128, "Ep": 128, "H": 384}, 8192),
         ("cfg2", {}, 1024), ("cfg2", {}, 2048)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def workload(name, extra):
    w = dict(WORKLOADS["cfg3" if name == "paper" else name])
    w.update(extra)
    return w


def make_step(w, dev, sampler):
    o = types.SimpleNamespace(terminal_count=w["T"], path_count=w["P"], label_count=w["C"], terminal_embed_size=w["Et"],
                              path_embed_size=w["Ep"], encode_size=w["H"], dropout_prob=DROPOUT,
                              angular_margin_loss=False, angular_margin=0.5, inverse_temp=30.0, device=dev)
    m = Code2Vec(o)
    m.load_state_dict(synth_params(w, dev))
    m = m.to(dev).train()
    opt = ShardedFlatAdam(m.parameters(), lr=0.01)
    return lambda s, p, e, lab: ddp_step(m, opt, None, s, p, e, lab, None, sampler=sampler)


def stats(ms):
    a = np.array(ms)
    return {"median": round(float(np.median(a)), 3), "p10": round(float(np.percentile(a, 10)), 3),
            "p90": round(float(np.percentile(a, 90)), 3)}


def profile_parts(step, batch, warmup, n=5):
    from torch.profiler import ProfilerActivity, profile
    for i in range(warmup):
        step(*batch(i))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(n):
            step(*batch(i))
        torch.cuda.synchronize()
    parts, total = {}, 0.0
    for k in prof.key_averages():
        t = k.device_time_total / n / 1000.0
        if t <= 0:
            continue
        total += t
        part = next((nm for nm, keys in PARTS if any(x in k.key for x in keys)), "other")
        parts[part] = parts.get(part, 0.0) + t
    return prof, total, parts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="directory for the profiler's tables")
    ap.add_argument("--cases", type=int, nargs="*", default=None, help="indices into the workload list")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_sampled.py measures on a GPU; none is available")
    torch.backends.cuda.matmul.fp32_precision = "ieee"
    dev = torch.device("cuda:0")
    name = card()
    for idx in (a.cases if a.cases is not None else range(len(CASES))):
        wname, extra, S = CASES[idx]
        w = workload(wname, extra)
        B, C = w["B"], w["C"]
        s, p, e, lab = synth_pool(w, 4, dev, 1)
        batch = lambda i: tuple(t[(i % 4) * B:(i % 4 + 1) * B] for t in (s, p, e, lab))  # noqa: E731
        sampler = CF.SampledSoftmax(C, S, counts=1.0 / np.arange(1, C + 1), power=0.75)
        steps = {"full": make_step(w, dev, None), "sampled": make_step(w, dev, sampler)}
        head = {"workload": wname, "E": w["Et"], "H": w["H"], "C": C, "S": S, "B": B, "L": w["L"], "card": name}
        if a.profile:
            out = dict(head)
            for nm, fn in steps.items():
                prof, total, parts = profile_parts(fn, batch, a.warmup)
                out[nm] = {"device_ms_per_step": round(total, 3),
                           "parts_ms": {k: round(v, 3) for k, v in sorted(parts.items(), key=lambda x: -x[1])},
                           "shares": {k: round(v / total, 3) for k, v in parts.items()}}
                if a.out:
                    os.makedirs(a.out, exist_ok=True)
                    with open(os.path.join(a.out, f"sampled_profile_{wname}_S{S}_{nm}.txt"), "w") as f:
                        f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=40))
            print(json.dumps(out), flush=True)
        else:
            times = {k: [] for k in steps}
            for i in range(a.warmup + a.steps):
                for nm, fn in steps.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn(*batch(i))
                    torch.cuda.synchronize()
                    if i >= a.warmup:
                        times[nm].append((time.perf_counter() - t0) * 1000.0)
            r = {k: stats(v) for k, v in times.items()}
            print(json.dumps({**head, "ms": r, "speedup_median": round(r["full"]["median"] / r["sampled"]["median"], 3)}),
                  flush=True)
        del steps
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

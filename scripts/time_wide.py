"""Time the training step at the paper's shape (embeddings 128 / 128, encode size 384), against eager torch on the same card.

    python scripts/time_wide.py [--steps 30] [--profile] [--out DIR]

At E = 128, H = 384, B = 1024, L = 200 with cfg2's vocabulary (T = 360,633, P = 342,846) and C in {8,192, 195,299}:
  * ours: Code2Vec.forward_loss through ddp_step with ShardedFlatAdam, dropout 0.25;
  * torch: oracle.torch_forward on the device with autograd (fp32, TF32 off), dropout 0.25, mean NLL, torch.optim.Adam.
The two steps alternate in one process on the same batches; each sample is one step between a device synchronise on
either side.  Prints one JSON line per C: median and p10 / p90 (ms) of both, with the card's name and power limit.
--profile instead runs ours alone under torch.profiler and prints the device time per part of the step.
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
import torch.nn.functional as F

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)
from bench import WORKLOADS, synth_params, synth_pool  # noqa: E402
from code2vec_b200.distributed import ShardedFlatAdam, ddp_step  # noqa: E402
from code2vec_b200.model import Code2Vec  # noqa: E402
from oracle import oracle  # noqa: E402

DROPOUT = 0.25
# kernel-name substrings -> part of the step (first match wins)
PARTS = (("encode fwd", ("encode_ffma_kernel", "encode_wgmma_kernel", "finalize")),
         ("rows", ("backward_rows", "bag_dot", "transpose_w", "row_bag")),
         ("dW", ("backward_dw",)),
         ("dC", ("backward_dc_tc", "split_wt", "wt_absmax")),
         ("Adam", ("adam",)),
         ("label head", ("sgemm", "gemm", "label", "softmax", "loss", "nll", "reduce", "lse")))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def workload(C):
    w = dict(WORKLOADS["cfg2"])
    w.update(H=384, C=C)
    return w


def ours(w, dev):
    o = types.SimpleNamespace(terminal_count=w["T"], path_count=w["P"], label_count=w["C"], terminal_embed_size=w["Et"],
                              path_embed_size=w["Ep"], encode_size=w["H"], dropout_prob=DROPOUT,
                              angular_margin_loss=False, angular_margin=0.5, inverse_temp=30.0, device=dev)
    m = Code2Vec(o)
    m.load_state_dict(synth_params(w, dev))
    m = m.to(dev).train()
    opt = ShardedFlatAdam(m.parameters(), lr=0.01)
    return lambda s, p, e, lab: ddp_step(m, opt, None, s, p, e, lab, None)


def eager(w, dev):
    params = {k: v.clone().requires_grad_() for k, v in synth_params(w, dev).items()}
    opt = torch.optim.Adam(list(params.values()), lr=0.01)

    def step(s, p, e, lab):
        opt.zero_grad(set_to_none=False)
        out, _, _ = oracle.torch_forward(params, s, p, e, lab, drop_p=DROPOUT, training=True)
        loss = F.nll_loss(F.log_softmax(out, dim=1), lab)
        loss.backward()
        opt.step()
        return loss
    return step


def stats(ms):
    a = np.array(ms)
    return {"median": float(np.median(a)), "p10": float(np.percentile(a, 10)), "p90": float(np.percentile(a, 90))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="directory for the profiler's table")
    ap.add_argument("--C", type=int, nargs="*", default=[8192, 195299])
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_wide.py measures on a GPU; none is available")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda:0")
    name = card()
    for C in a.C:
        w = workload(C)
        B = w["B"]
        s, p, e, lab = synth_pool(w, 4, dev, 1)
        batch = lambda i: tuple(t[(i % 4) * B:(i % 4 + 1) * B] for t in (s, p, e, lab))
        step = ours(w, dev)
        if a.profile:
            from torch.profiler import ProfilerActivity, profile
            for i in range(a.warmup):
                step(*batch(i))
            torch.cuda.synchronize()
            n = 5
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
            print(json.dumps({"C": C, "card": name, "device_ms_per_step": round(total, 3),
                              "parts_ms": {k: round(v, 3) for k, v in sorted(parts.items(), key=lambda x: -x[1])},
                              "shares": {k: round(v / total, 3) for k, v in parts.items()}}))
            if a.out:
                os.makedirs(a.out, exist_ok=True)
                with open(os.path.join(a.out, f"wide_profile_C{C}.txt"), "w") as f:
                    f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=40))
            del step
            torch.cuda.empty_cache()
            continue
        ref = eager(w, dev)
        times = {"ours": [], "torch": []}
        for i in range(a.warmup + a.steps):
            for nm, fn in (("ours", step), ("torch", ref)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn(*batch(i))
                torch.cuda.synchronize()
                if i >= a.warmup:
                    times[nm].append((time.perf_counter() - t0) * 1000.0)
        r = {k: stats(v) for k, v in times.items()}
        print(json.dumps({"C": C, "E": w["Et"], "H": w["H"], "B": B, "L": w["L"], "card": name, "ms": r,
                          "speedup_median": r["torch"]["median"] / r["ours"]["median"]}))
        del step, ref
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

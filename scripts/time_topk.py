"""Top-k label prediction (k = 10, with probabilities), timed three ways in the same process, alternating:
  eager  forward() under no_grad ([B, C] logits written) + torch.topk + softmax at the top k -- what a user does today
  fused  predict_topk() (running top-k in the tensor-core label GEMM's epilogue; the logits are never written)
  top1   predict() (fused arg-max): the floor, one label per method
Checks first that eager and fused return the same indices under the stable tie rule (torch.sort(descending=True,
stable=True) of forward()'s logits) and the same values, then prints one JSON line per workload (median call time over
--steps alternating rounds, CUDA events, after --warmup rounds) and the card's name / power limit / max SM clock.

    python scripts/time_topk.py [--workloads cfg2,cfg3] [--steps 20] [--warmup 5] [--k 10]
"""
import argparse
import json
import os
import sys
import types

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)

import torch  # noqa: E402

from bench import WORKLOADS, synth_params, synth_pool  # noqa: E402
from code2vec_b200.model import Code2Vec  # noqa: E402
from scripts.time_angular import card  # noqa: E402


def plain_model(w, dev):
    o = types.SimpleNamespace(terminal_count=w["T"], path_count=w["P"], label_count=w["C"], terminal_embed_size=w["Et"],
                              path_embed_size=w["Ep"], encode_size=w["H"], dropout_prob=0.0, angular_margin_loss=False,
                              angular_margin=0.5, inverse_temp=30.0, device=dev)
    m = Code2Vec(o)
    m.load_state_dict(synth_params(w, dev))
    return m.to(dev).eval()


def run(m, batch, way, k):
    s, p, e, lab = batch
    with torch.no_grad():
        if way == "eager":
            out = m.forward(s, p, e, lab)[0]
            val, idx = torch.topk(out, k, dim=1)
            return idx, val, torch.softmax(out, dim=1).gather(1, idx)
        if way == "fused":
            return m.predict_topk(s, p, e, k=k)[:3]
        return m.predict(s, p, e)[:2]


def compare(m, batch, k):
    s, p, e, lab = batch
    with torch.no_grad():
        out = m.forward(s, p, e, lab)[0]
        ref_val, ref_idx = torch.sort(out, dim=1, descending=True, stable=True)
        ref_idx, ref_val = ref_idx[:, :k], ref_val[:, :k]
        ref_prob = torch.softmax(out.double(), dim=1).gather(1, ref_idx)
        idx, val, prob = m.predict_topk(s, p, e, k=k)[:3]
        tk = torch.topk(out, k, dim=1).indices
    return {"indices_equal": bool(torch.equal(idx, ref_idx)), "values_equal": bool(torch.equal(val, ref_val)),
            "topk_indices_equal": bool(torch.equal(tk, ref_idx)),
            "max_prob_rel_diff": ((prob.double() - ref_prob).abs() / ref_prob).max().item()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg2,cfg3")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--k", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_topk.py measures on the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    ways = ("eager", "fused", "top1")
    for name in args.workloads.split(","):
        w = dict(WORKLOADS[name]); B = w["B"]
        m = plain_model(w, dev)
        n_b = 4
        s, p, e, lab = synth_pool(w, n_b, dev, 1)
        batches = [(s[i * B:(i + 1) * B], p[i * B:(i + 1) * B], e[i * B:(i + 1) * B], lab[i * B:(i + 1) * B]) for i in range(n_b)]
        check = compare(m, batches[0], args.k)
        if not (check["indices_equal"] and check["values_equal"]):
            raise SystemExit(f"{name}: predict_topk disagrees with the stable sort of forward()'s logits: {check}")
        times = {way: [] for way in ways}
        for i in range(args.warmup + args.steps):
            for way in ways:
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run(m, batches[i % n_b], way, args.k)
                e1.record()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[way].append(e0.elapsed_time(e1))
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        print(json.dumps({"workload": name, "B": B, "L": w["L"], "C": w["C"], "H": w["H"], "k": args.k, "steps": args.steps,
                          **{f"{way}_ms": round(med[way], 3) for way in ways},
                          **{f"{way}_ms_min_max": [round(min(times[way]), 3), round(max(times[way]), 3)] for way in ways},
                          "speedup_vs_eager": round(med["eager"] / med["fused"], 2), "check": check, "card": info}),
              flush=True)
        del m, batches, s, p, e, lab
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

"""One training step through the angular-margin head (model.py:71-80), two ways in the same process, alternating:
  eager  forward() (CUDA-core angular head, [B, C] outputs + cosines) + eager log_softmax / nll_loss + backward
  fused  forward_loss() (angular epilogue of the tensor-core label GEMM, logits never written) + backward
Checks first that both give the same loss and parameter gradients on the same batch and dropout seed, then prints one
JSON line per workload (median step time over --steps alternating pairs, CUDA events, after --warmup pairs) and the
card's name / power limit / max SM clock.

    python scripts/time_angular.py [--workloads cfg2,cfg3] [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys
import types

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from bench import WORKLOADS, synth_params, synth_pool  # noqa: E402
from code2vec_b200.model import Code2Vec  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = (x.strip() for x in out.split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as exc:                                    # the timing itself does not depend on it
        return {"error": repr(exc)}


def angular_model(w, dev, dropout):
    o = types.SimpleNamespace(terminal_count=w["T"], path_count=w["P"], label_count=w["C"], terminal_embed_size=w["Et"],
                              path_embed_size=w["Ep"], encode_size=w["H"], dropout_prob=dropout, angular_margin_loss=True,
                              angular_margin=0.5, inverse_temp=30.0, device=dev)
    p = synth_params(w, dev)
    p["output_linear"] = p.pop("output_linear.weight")
    del p["output_linear.bias"]
    m = Code2Vec(o)
    m.load_state_dict(p)
    return m.to(dev).train()


def step(m, batch, fused):
    s, p, e, lab = batch
    if fused:
        loss = m.forward_loss(s, p, e, lab)[0]
    else:
        out = m.forward(s, p, e, lab)[0]
        loss = F.nll_loss(F.log_softmax(out, dim=1), lab)
    loss.backward()
    return loss


def compare(m, batch):
    res = []
    for fused in (False, True):
        m.zero_grad(set_to_none=True)
        torch.manual_seed(123)                                  # same dropout mask both ways
        loss = step(m, batch, fused).item()
        res.append((loss, {k: v.grad.detach().clone() for k, v in m.named_parameters()}))
    (l0, g0), (l1, g1) = res
    grad_rel = {k: (g1[k] - g0[k]).abs().max().item() / max(g0[k].abs().max().item(), 1e-30) for k in g0}
    return {"loss_eager": l0, "loss_fused": l1, "loss_rel_diff": abs(l1 - l0) / max(abs(l0), 1e-30),
            "max_grad_rel_diff": max(grad_rel.values()), "grad_rel_diff": grad_rel}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg2,cfg3")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--dropout", type=float, default=0.25)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_angular.py measures on the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    for name in args.workloads.split(","):
        w = dict(WORKLOADS[name]); B = w["B"]
        m = angular_model(w, dev, args.dropout)
        n_b = 4
        s, p, e, lab = synth_pool(w, n_b, dev, 1)
        batches = [(s[i * B:(i + 1) * B], p[i * B:(i + 1) * B], e[i * B:(i + 1) * B], lab[i * B:(i + 1) * B]) for i in range(n_b)]
        check = compare(m, batches[0])
        times = {"eager": [], "fused": []}
        for i in range(args.warmup + args.steps):
            for way in ("eager", "fused"):
                m.zero_grad(set_to_none=True)
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                step(m, batches[i % n_b], way == "fused")
                e1.record()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[way].append(e0.elapsed_time(e1))
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        print(json.dumps({"workload": name, "B": B, "C": w["C"], "H": w["H"], "dropout": args.dropout, "steps": args.steps,
                          "eager_step_ms": round(med["eager"], 3), "fused_step_ms": round(med["fused"], 3),
                          "eager_ms_min_max": [round(min(times["eager"]), 3), round(max(times["eager"]), 3)],
                          "fused_ms_min_max": [round(min(times["fused"]), 3), round(max(times["fused"]), 3)],
                          "speedup": round(med["eager"] / med["fused"], 2), "check": check, "card": info}), flush=True)
        del m, batches, s, p, e, lab
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

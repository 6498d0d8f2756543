"""A training step (ddp_step with ShardedFlatAdam, dropout 0.25) with and without a criterion, three ways alternating in
one process, and the label-loss call alone:
  none      forward_loss()                                        (fused, all class weights 1, mean)
  fused     forward_loss(criterion=CrossEntropyLoss(weight=w, label_smoothing=0.1))
  eager     forward() + that criterion on the [B, C] logits
  loss_*    the fused forward + backward of the label head alone (code vectors fixed), without / with the criterion
Prints one JSON line per workload: median and p10 / p90 of each (CUDA events, after --warmup rounds), the loss of each
way on the same batch and the card's name / power limit / max SM clock.

    python scripts/time_criterion.py [--workloads cfg2,cfg3] [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import sys
import types

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)
sys.path.insert(0, os.path.join(R, "scripts"))

import torch  # noqa: E402
import torch.nn as nn  # noqa: E402

from bench import WORKLOADS, synth_params, synth_pool  # noqa: E402
from time_angular import card  # noqa: E402
from code2vec_b200 import functional as CF  # noqa: E402
from code2vec_b200.distributed import ShardedFlatAdam, ddp_step  # noqa: E402
from code2vec_b200.model import Code2Vec, _LabelLossFn, _LabelLossOptsFn  # noqa: E402


def model(w, dev, dropout):
    o = types.SimpleNamespace(terminal_count=w["T"], path_count=w["P"], label_count=w["C"], terminal_embed_size=w["Et"],
                              path_embed_size=w["Ep"], encode_size=w["H"], dropout_prob=dropout, angular_margin_loss=False,
                              angular_margin=0.5, inverse_temp=30.0, device=dev)
    m = Code2Vec(o)
    m.load_state_dict(synth_params(w, dev))
    return m.to(dev).train()


def pct(v, q):
    v = sorted(v)
    return v[min(len(v) - 1, int(round(q * (len(v) - 1))))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg2,cfg3")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--dropout", type=float, default=0.25)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_criterion.py measures on the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    for name in args.workloads.split(","):
        w = dict(WORKLOADS[name]); B, C = w["B"], w["C"]
        m = model(w, dev, args.dropout)
        opt = ShardedFlatAdam(m.parameters(), lr=0.01, betas=(0.9, 0.999))
        g = torch.Generator(device="cpu").manual_seed(5)
        crit = nn.CrossEntropyLoss(weight=(0.5 + torch.rand(C, generator=g)).to(dev), label_smoothing=0.1)
        n_b = 4
        s, p, e, lab = synth_pool(w, n_b, dev, 1)
        batches = [(s[i * B:(i + 1) * B], p[i * B:(i + 1) * B], e[i * B:(i + 1) * B], lab[i * B:(i + 1) * B]) for i in range(n_b)]
        # the label head alone: fixed code vectors, the fused loss forward + backward of the label GEMM
        cv = torch.randn(B, w["H"], device=dev).mul_(0.5).requires_grad_()
        W = m.output_linear.weight.detach().clone().requires_grad_()      # (not the parameters: their .grad is the
        b = m.output_linear.bias.detach().clone().requires_grad_()        # optimizer's bucket)
        dims, cache = m._dims(), CF.PrepCache()
        ccrit = CF.LossCriterion(crit, C, dev)

        def head(with_crit):
            if with_crit:
                loss = _LabelLossOptsFn.apply(cv, W, b, batches[0][3], dims, m._label_algo, cache, None, ccrit)[0]
            else:
                loss = _LabelLossFn.apply(cv, W, b, batches[0][3], dims, m._label_algo, cache, None)[0]
            loss.backward()
            return loss

        def run(way, i):
            bs, bp, be, bl = batches[i % n_b]
            if way == "none":
                return ddp_step(m, opt, None, bs, bp, be, bl, None)
            if way == "fused":
                return ddp_step(m, opt, None, bs, bp, be, bl, None, criterion=crit)
            if way == "eager":
                return ddp_step(m, opt, None, bs, bp, be, bl, crit)
            return head(way == "loss_criterion")

        ways = ("none", "fused", "eager", "loss_none", "loss_criterion")
        losses = {k: float(run(k, 0).detach()) for k in ways}
        times = {k: [] for k in ways}
        for i in range(args.warmup + args.steps):
            for way in ways:
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run(way, i)
                e1.record()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[way].append(e0.elapsed_time(e1))
        res = {k: {"median_ms": round(pct(v, 0.5), 3), "p10_ms": round(pct(v, 0.1), 3), "p90_ms": round(pct(v, 0.9), 3)}
               for k, v in times.items()}
        print(json.dumps({"workload": name, "B": B, "C": C, "H": w["H"], "dropout": args.dropout, "steps": args.steps,
                          "step": {k: res[k] for k in ("none", "fused", "eager")},
                          "label_loss_alone": {k: res[k] for k in ("loss_none", "loss_criterion")},
                          "eager_over_fused": round(res["eager"]["median_ms"] / res["fused"]["median_ms"], 2),
                          "first_losses": losses, "card": info}), flush=True)
        del m, opt, batches, s, p, e, lab
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

"""What parameter groups cost in the flat Adam step, one process, one GPU.

    python scripts/time_param_groups.py [--steps 30] [--out DIR]

On the cfg2 and cfg3 models (L = 200), three layouts of the same parameters:
  one    one group: today's kernel (adam_step_kernel<false, false>)
  two    the no-decay recipe: the embedding tables, input_linear and output_linear.weight with weight decay 0.01,
         LayerNorm, attention_parameter and the output bias without, AdamW
  three  three groups interleaved over the parameter order, parameter i in group i % 3, different betas per group
and two cases:
  opt    FlatAdam.step() alone (one launch over the whole flat bucket), CUDA events per step.  FlatAdam keeps the
         model's parameter order, so "two" is 5 runs of the flat buffers and "three" 8
  step   ddp_step with ShardedFlatAdam at B = 1024, dropout 0.25, the fused loss.  ShardedFlatAdam lays the groups out
         one after the other: 2 and 3 runs
The layouts of a case alternate in rounds (3 each) in one process.  Per layout: median and p10-p90 of CUDA-event times
around each step.  Prints one JSON document (also written to DIR/time_param_groups.json) with the card's name, power
limit and max SM clock, read in the same run."""
import argparse
import json
import os

import numpy as np
import torch

from time_graphs import WL, batches, gpu_info, make_model, stats, time_round      # also puts the repository on sys.path
from code2vec_b200 import _lib
from code2vec_b200.distributed import FlatAdam, FlatGradBucket, ShardedFlatAdam, ddp_step

LAYOUTS = ("one", "two", "three")


def groups_of(model, layout):
    named = list(model.named_parameters())
    ps = [p for _, p in named]
    if layout == "one":
        return ps, {}
    if layout == "two":
        decay = [p for n, p in named if n.endswith("embedding.weight") or n in ("input_linear.weight",
                                                                                "output_linear.weight")]
        rest = [p for n, p in named if all(p is not q for q in decay)]
        return [{"params": decay, "weight_decay": 0.01}, {"params": rest, "weight_decay": 0.0}], \
            {"decoupled_weight_decay": True}
    betas = [(0.9, 0.999), (0.8, 0.99), (0.95, 0.9999)]
    return [{"params": ps[k::3], "betas": betas[k], "lr": 1e-3 * (k + 1)} for k in range(3)], {}


def alternate(fns, data, lib, rounds=3):
    acc = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            acc[k].extend(time_round(fn, data, lib)[0])
    return {k: stats(v) for k, v in acc.items()}


def case(wn, kind, steps, dev, lib):
    w = WL[wn]
    data = batches(w, 1024, 200, steps, dev, seed=1024)
    fns, segs = {}, {}
    for layout in LAYOUTS:
        m = make_model(w, dev).train()
        params, kw = groups_of(m, layout)
        if kind == "opt":
            opt = FlatAdam(FlatGradBucket(m.parameters()), lr=1e-3, groups=None if layout == "one" else params, **kw)
            opt.bucket.flat.normal_()
            fn = lambda *b, opt=opt: opt.step(zero_grad=False)
        else:
            opt = ShardedFlatAdam(params, lr=1e-3, **kw)
            fn = lambda s, p, e, y, m=m, opt=opt: ddp_step(m, opt, None, s, p, e, y, None)
        segs[layout] = len(opt._segments)
        for b in data[:4]:
            fn(*b)
        fns[layout] = fn
    torch.cuda.synchronize()
    out = alternate(fns, data, lib)
    return {"workload": wn, "case": kind, "flat_elements": sum(p.numel() for p in make_model(w, "cpu").parameters()),
            "runs_of_the_flat_buffers": segs, "event_ms": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_param_groups.py needs a GPU")
    dev = torch.device("cuda:0")
    lib = _lib.load()
    res = {"gpu": gpu_info(), "cases": [case(wn, kind, a.steps, dev, lib) for wn in ("cfg2", "cfg3")
                                        for kind in ("opt", "step")]}
    for c in res["cases"]:
        print(c["workload"], c["case"], {k: f'{v["median"]:.3f} ({v["p10"]:.3f}-{v["p90"]:.3f})'
                                         for k, v in c["event_ms"].items()})
    doc = json.dumps(res, indent=1)
    print(doc)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_param_groups.json"), "w") as f:
            f.write(doc)


if __name__ == "__main__":
    main()

"""What clipping, learning-rate schedules and checkpoints cost on the flat Adam optimizers, one process, one GPU.

    python scripts/time_optimizer.py [--steps 30] [--out DIR]

clip      cfg2 and cfg3 at B = 1024, L = 200, ddp_step with ShardedFlatAdam (world size 1), dropout 0.25:
          none    no clipping
          fused   ShardedFlatAdam(max_grad_norm=1.0): the norm pass and the clip inside the step
          torch   forward + backward by hand, torch.nn.utils.clip_grad_norm_ on the parameters (views of the flat bucket),
                  then optimizer.step()
norm      c2v_grad_clip_coef alone on cfg2's gradient bucket: time per call over many launches, and the achieved bytes/s
          from the bucket's size (one read of it; not a share of any peak)
schedule  "small" (the reference's defaults) and cfg2 at B = 32 and 128: FlatAdam(lr=tensor, capturable=True) with a
          LambdaLR stepped after every call, ddp_step eagerly against GraphedTrainStep
state     state_dict() and load_state_dict() of ShardedFlatAdam at cfg2, wall time, each ending in a synchronise
The variants of a case alternate in rounds in one process.  Per variant: median and p10-p90 of CUDA-event times around
each step and of a host clock ending in a synchronise.  Prints one JSON document (also written to
DIR/time_optimizer.json) with the card's name, power limit and max SM clock, read in the same run."""
import argparse
import ctypes
import json
import os
import time

import numpy as np
import torch

from time_graphs import WL, batches, gpu_info, make_model, stats, time_round      # also puts the repository on sys.path
from code2vec_b200 import _lib
from code2vec_b200.distributed import FlatAdam, FlatGradBucket, ShardedFlatAdam, ddp_step
from code2vec_b200.graphs import GraphedTrainStep


def alternate(fns, data, lib, rounds=3):
    """{name: step function} -> {name: event / host statistics}, the variants alternating round by round"""
    acc = {k: ([], [], []) for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            ev, host, _, launches = time_round(fn, data, lib)
            acc[k][0].extend(ev); acc[k][1].extend(host); acc[k][2].append(launches)
    return {k: {"event_ms": stats(a[0]), "host_ms": stats(a[1]), "launches_per_step": float(np.mean(a[2]))}
            for k, a in acc.items()}


def clip_case(wn, B, L, steps, dev, lib):
    w = WL[wn]
    data = batches(w, B, L, steps, dev, seed=B)
    fns = {}
    for name in ("none", "fused", "torch"):
        m = make_model(w, dev).train()
        opt = ShardedFlatAdam(m.parameters(), lr=1e-3, max_grad_norm=1.0 if name == "fused" else None)
        if name == "torch":
            def fn(s, p, e, y, m=m, opt=opt, params=list(m.parameters())):
                m.fuse_grad_accumulation = True
                loss = m.forward_loss(s, p, e, y)[0]
                loss.backward()
                torch.nn.utils.clip_grad_norm_(params, 1.0)
                opt.step()
                return loss
        else:
            fn = lambda s, p, e, y, m=m, opt=opt: ddp_step(m, opt, None, s, p, e, y, None)
        for b in data[:4]:
            fn(*b)
        fns[name] = fn
    torch.cuda.synchronize()
    out = alternate(fns, data, lib)
    out.update(workload=wn, B=B)
    return out


def norm_case(wn, dev, lib, launches=200):
    n = sum(p.numel() for p in make_model(WL[wn], "cpu").parameters())
    g = torch.randn(n, device=dev)
    ws = torch.empty(lib.c2v_grad_norm_workspace_bytes(n) // 4, device=dev)
    out = torch.zeros(2, device=dev)
    V = ctypes.c_void_p
    call = lambda: _lib.check(lib.c2v_grad_clip_coef(V(g.data_ptr()), n, 1.0, 1.0, V(out.data_ptr()), V(ws.data_ptr()),
                                                     4 * ws.numel(), V(torch.cuda.current_stream().cuda_stream)),
                              "c2v_grad_clip_coef")
    for _ in range(10):
        call()
    per_call = []
    for _ in range(5):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(launches):
            call()
        e1.record()
        torch.cuda.synchronize()
        per_call.append(e0.elapsed_time(e1) / launches)
    ms = float(np.median(per_call))
    return {"workload": wn, "elements": n, "bucket_bytes": 4 * n, "launches_per_window": launches, "windows_ms_per_call": per_call,
            "ms_per_call_median": ms, "achieved_bytes_per_s": 4 * n / (ms * 1e-3)}


def schedule_case(wn, B, L, steps, dev, lib):
    w = WL[wn]
    data = batches(w, B, L, steps, dev, seed=B)
    fns = {}
    for mode in ("eager", "graph"):
        m = make_model(w, dev).train().use_device_rng(seed=1)
        opt = FlatAdam(FlatGradBucket(m.parameters()), lr=torch.tensor(1e-3, device=dev), capturable=True)
        sch = torch.optim.lr_scheduler.LambdaLR(opt, lambda e: min(1.0, (e + 1) / 100.0))
        step = GraphedTrainStep(m, opt, B, L) if mode == "graph" else \
            (lambda s, p, e, y, m=m, opt=opt: ddp_step(m, opt, opt.bucket, s, p, e, y, None))

        def fn(s, p, e, y, step=step, sch=sch):
            loss = step(s, p, e, y)
            sch.step()
            return loss
        for b in data[:4]:
            fn(*b)
        fns[mode] = fn
    torch.cuda.synchronize()
    out = alternate(fns, data, lib)
    out.update(workload=wn, B=B, speedup_host_clock=out["eager"]["host_ms"]["median"] / out["graph"]["host_ms"]["median"])
    return out


def state_case(wn, dev, repeats=5):
    m = make_model(WL[wn], dev)
    opt = ShardedFlatAdam(m.parameters(), lr=1e-3, early=[m.path_embedding.weight])
    save, load = [], []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sd = opt.state_dict()
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        opt.load_state_dict(sd)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        save.append((t1 - t0) * 1e3); load.append((t2 - t1) * 1e3)
    return {"workload": wn, "state_dict_ms": stats(save), "load_state_dict_ms": stats(load)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--L", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_optimizer.py measures on the GPU and needs one")
    lib = _lib.load()
    dev = torch.device("cuda:0")
    doc = {"gpu": gpu_info(), "L": a.L, "steps": a.steps, "clip": [], "schedule": []}
    for wn in ("cfg2", "cfg3"):
        doc["clip"].append(clip_case(wn, 1024, a.L, a.steps, dev, lib))
        print(json.dumps(doc["clip"][-1]), flush=True)
        torch.cuda.empty_cache()
    doc["norm"] = norm_case("cfg2", dev, lib)
    print(json.dumps(doc["norm"]), flush=True)
    for wn in ("small", "cfg2"):
        for B in (32, 128):
            doc["schedule"].append(schedule_case(wn, B, a.L, a.steps, dev, lib))
            print(json.dumps(doc["schedule"][-1]), flush=True)
            torch.cuda.empty_cache()
    doc["state"] = state_case("cfg2", dev)
    print(json.dumps(doc))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "time_optimizer.json"), "w") as f:
            json.dump(doc, f, indent=1)


if __name__ == "__main__":
    main()

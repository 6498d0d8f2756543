"""What torch's TF32 switch (torch.set_float32_matmul_precision("high")) buys: the library's tensor-core GEMMs in one pass
(C2V_MATMUL_TF32) against the default three passes (C2V_MATMUL_IEEE).

Alternates IEEE and TF32 rounds in one process on one model per case, so that both modes see the same clocks and
neighbours, and reports per workload and mode the median time per call with its p10 - p90 range over the samples (a
sample: CUDA events around --calls back-to-back calls, so that short calls are not timed one launch at a time):
  encode      the encode forward of a batch (eval, no dropout)
  label       the label-loss call: the fused loss forward + backward of the label head on fixed code vectors
  train       the training step: ddp_step with ShardedFlatAdam, the fused loss, dropout 0.25
  predict     Code2Vec.predict()
  topk        Code2Vec.predict_topk(k=10)
The card's name, power limit and max SM clock are read in the same run.

    python scripts/time_precision.py [--steps 30] [--calls 10] [--warmup 5] [--cases cfg2,cfg3,cfg4] [--out f.json]
                                     [--profile cfg2,...]

--profile: afterwards, for each listed case, a separate torch.profiler run (CUDA activities) of --steps rounds per mode:
per kernel and mode the device time per round and the median (p10 - p90) of its single launches.
"""
import argparse
import json
import os
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench import WORKLOADS, synth_params, synth_pool  # noqa: E402
from code2vec_b200.distributed import ShardedFlatAdam, ddp_step  # noqa: E402
from code2vec_b200.model import Code2Vec, _LabelLossFn  # noqa: E402
from time_deterministic import card  # noqa: E402

CASES = ("cfg2", "cfg3", "cfg4")


def set_mode(tf32):
    torch.backends.cuda.matmul.fp32_precision = "tf32" if tf32 else "ieee"


def _build(case, dev):
    w = dict(WORKLOADS[case])
    o = types.SimpleNamespace(terminal_count=w["T"], path_count=w["P"], label_count=w["C"], terminal_embed_size=w["Et"],
                              path_embed_size=w["Ep"], encode_size=w["H"], dropout_prob=0.25, angular_margin_loss=False,
                              angular_margin=0.5, inverse_temp=30.0, device=dev)
    torch.manual_seed(0)
    m = Code2Vec(o)
    m.load_state_dict(synth_params(w, dev))
    m = m.to(dev).train()
    opt = ShardedFlatAdam(m.parameters(), lr=0.01)
    n_b, B = 4, w["B"]
    s, p, e, lab = synth_pool(w, n_b, dev, 1234)
    batches = [(s[i * B:(i + 1) * B], p[i * B:(i + 1) * B], e[i * B:(i + 1) * B], lab[i * B:(i + 1) * B]) for i in range(n_b)]
    g = torch.Generator(device=dev).manual_seed(5)
    cv = (0.3 * torch.randn(B, w["H"], generator=g, device=dev)).requires_grad_()

    def encode(i):
        with torch.no_grad():
            m.eval()
            m._encode_eval(*batches[i % n_b][:3])
            m.train()

    def label(i):
        w_out, b_out = m._head()
        loss, _, _ = _LabelLossFn.apply(cv, w_out, b_out, batches[i % n_b][3], m._dims(), m._label_algo, m._lab_cache, None)
        loss.backward()

    def train(i):
        ddp_step(m, opt, None, *batches[i % n_b], None)

    def predict(i):
        with torch.no_grad():
            m.eval()
            m.predict(*batches[i % n_b][:3])
            m.train()

    def topk(i):
        m.eval()
        m.predict_topk(*batches[i % n_b][:3], k=10)
        m.train()
    return w, {"encode": encode, "label": label, "train": train, "predict": predict, "topk": topk}


def run_case(case, steps, calls, warmup, dev):
    w, fns = _build(case, dev)
    res = {"case": case, "B": w["B"], "L": w["L"], "H": w["H"], "E": w["Et"], "C": w["C"], "samples": steps,
           "calls_per_sample": calls}
    for name, fn in fns.items():
        for i in range(warmup):
            for tf32 in (False, True):
                set_mode(tf32)
                fn(i)
        torch.cuda.synchronize()
        times = {False: [], True: []}
        for i in range(steps):
            for tf32 in ((False, True) if i % 2 == 0 else (True, False)):
                set_mode(tf32)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for j in range(calls):
                    fn(i * calls + j)
                e1.record()
                e1.synchronize()
                times[tf32].append(e0.elapsed_time(e1) / calls)
        r = {}
        for tf32, key in ((False, "ieee"), (True, "tf32")):
            t = np.array(times[tf32])
            r[key] = {"median_ms": float(np.median(t)), "p10_ms": float(np.percentile(t, 10)),
                      "p90_ms": float(np.percentile(t, 90))}
        r["speedup"] = r["ieee"]["median_ms"] / r["tf32"]["median_ms"]
        res[name] = r
    set_mode(False)
    del fns
    torch.cuda.empty_cache()
    return res


def profile_case(case, steps, warmup, dev):
    """device time per round (all five workloads once) of every kernel, per mode, from a torch.profiler run of its own"""
    _, fns = _build(case, dev)
    for i in range(warmup):
        for tf32 in (False, True):
            set_mode(tf32)
            for fn in fns.values():
                fn(i)
    torch.cuda.synchronize()
    out = {"case": case, "steps": steps}
    for tf32, key in ((False, "ieee"), (True, "tf32")):
        set_mode(tf32)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for i in range(steps):
                for fn in fns.values():
                    fn(i)
            torch.cuda.synchronize()
        k = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                k.setdefault(e.name, []).append(e.time_range.elapsed_us() / 1000.0)
        per_round = {n: sum(v) / steps for n, v in k.items()}
        out[key] = {n: {"ms_per_round": round(per_round[n], 4), "launches_per_round": len(k[n]) / steps,
                        "launch_median_ms": round(float(np.median(k[n])), 4),
                        "launch_p10_ms": round(float(np.percentile(k[n], 10)), 4),
                        "launch_p90_ms": round(float(np.percentile(k[n], 90)), 4)}
                    for n in sorted(k, key=lambda n: -per_round[n]) if per_round[n] >= 0.001}
        out[key + "_total_ms"] = round(sum(per_round.values()), 4)
    set_mode(False)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_precision.py measures on the GPU and found none")
    dev = torch.device("cuda:0")
    out = {"card": card(), "results": [], "profiles": []}
    print(json.dumps(out["card"]), flush=True)
    saved = torch.backends.cuda.matmul.fp32_precision
    try:
        for case in a.cases.split(","):
            r = run_case(case, a.steps, a.calls, a.warmup, dev)
            out["results"].append(r)
            print(json.dumps(r), flush=True)
        for case in filter(None, a.profile.split(",")):
            r = profile_case(case, a.steps, a.warmup, dev)
            out["profiles"].append(r)
            print(json.dumps(r), flush=True)
    finally:
        torch.backends.cuda.matmul.fp32_precision = saved
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

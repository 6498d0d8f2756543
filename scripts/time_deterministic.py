"""Cost of torch.use_deterministic_algorithms(True) on the training step.

Alternates the default and the deterministic training step -- bench.py's training leg: ddp_step with ShardedFlatAdam,
dropout 0.25, the fused loss -- in one process on one model, so that both see the same clocks and neighbours, and reports
per mode the median step time with its p10 - p90 range (CUDA events around each step) and the peak device memory of a
step above what was allocated before it.  The card's name and power limit are read in the same run.

    python scripts/time_deterministic.py [--steps 30] [--warmup 5] [--cases cfg2,cfg3,cfg4,cfg2-zipf,cfg2-b32] [--out f.json]
                                         [--profile cfg2,cfg2-zipf]

--profile: afterwards, for each listed case, a separate torch.profiler run (CUDA activities) of --steps steps per mode,
reporting per mode the device time per step of each part of the step (kernel-name groups, see PARTS): where the extra
time of the deterministic step goes.

Note: under the switch torch also fills every torch.empty with NaN (torch.utils.deterministic.fill_uninitialized_memory,
on by default), so the library's per-call workspaces -- the dC rows buffer above all -- pay for a fill; that cost is part of
the deterministic numbers here.
"""
import argparse
import json
import os
import subprocess
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import WORKLOADS, synth_params, synth_pool  # noqa: E402
from code2vec_b200.distributed import ShardedFlatAdam, ddp_step  # noqa: E402
from code2vec_b200.model import Code2Vec  # noqa: E402

# case: (workload, data, batch size override)
CASES = {"cfg2": ("cfg2", "uniform", None), "cfg3": ("cfg3", "uniform", None), "cfg4": ("cfg4", "uniform", None),
         "cfg2-zipf": ("cfg2", "zipf", None), "cfg2-b32": ("cfg2", "uniform", 32)}


def _zipf_batches(w, n, dev, s=1.2):
    """indices with P(i) proportional to (i + 1)^-s (Zipf(1.2)), full bags"""
    g = torch.Generator(device=dev).manual_seed(4321)
    B, L = w["B"], w["L"]

    def draw(m, shape):
        cdf = torch.cumsum(torch.arange(1, m + 1, dtype=torch.float64, device=dev) ** -s, 0)
        cdf /= cdf[-1].clone()
        return torch.searchsorted(cdf, torch.rand(shape, generator=g, device=dev, dtype=torch.float64)).clamp_(max=m - 1)
    out = []
    for _ in range(n):
        out.append((1 + draw(w["T"] - 1, (B, L)), 1 + draw(w["P"] - 1, (B, L)), 1 + draw(w["T"] - 1, (B, L)),
                    draw(w["C"], (B,))))
    return out


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                         # the numbers are still reported, without the card
        return {"name": torch.cuda.get_device_name(0), "error": str(e)}


# parts of a step by kernel name (first match wins); "nan fill" is torch's fill of new memory under the switch
PARTS = (("nan fill", ("fill", "Fill")), ("memset", ("Memset",)),
         ("dC (tensor cores)", ("backward_dc_tc_kernel",)), ("dW (tensor cores)", ("backward_dw_tc_kernel",)),
         ("rows (dx, LN / attention partials)", ("backward_rows",)),
         ("det keys", ("det_keys_kernel",)), ("det sort (CUB radix)", ("cub", "Radix", "Onesweep", "onesweep")),
         ("det chunk sums", ("det_chunk_kernel",)), ("det merge", ("det_merge_kernel",)),
         ("det slab sums", ("det_slab_sum_kernel",)), ("label head", ("label_", "lbt_")),
         ("encode forward", ("encode_",)), ("adam", ("adam",)))


def _part(name):
    for part, keys in PARTS:
        if any(k in name for k in keys):
            return part
    return "other"


def _build(case, dev):
    wname, data, b_override = CASES[case]
    w = dict(WORKLOADS[wname])
    if b_override:
        w["B"] = b_override
    o = types.SimpleNamespace(terminal_count=w["T"], path_count=w["P"], label_count=w["C"], terminal_embed_size=w["Et"],
                              path_embed_size=w["Ep"], encode_size=w["H"], dropout_prob=0.25, angular_margin_loss=False,
                              angular_margin=0.5, inverse_temp=30.0, device=dev)
    torch.manual_seed(0)
    m = Code2Vec(o)
    m.load_state_dict(synth_params(w, dev))
    m = m.to(dev).train()
    opt = ShardedFlatAdam(m.parameters(), lr=0.01)
    n_b = 4
    if data == "zipf":
        batches = _zipf_batches(w, n_b, dev)
    else:
        s, p, e, lab = synth_pool(w, n_b, dev, 1234)
        B = w["B"]
        batches = [(s[i * B:(i + 1) * B], p[i * B:(i + 1) * B], e[i * B:(i + 1) * B], lab[i * B:(i + 1) * B])
                   for i in range(n_b)]

    def step(det, i):
        torch.use_deterministic_algorithms(det)
        try:
            ddp_step(m, opt, None, *batches[i % n_b], None)
        finally:
            torch.use_deterministic_algorithms(False)
    return w, step


def profile_case(case, steps, warmup, dev):
    """device time per step of each part (PARTS), per mode, from a torch.profiler run of its own"""
    _, step = _build(case, dev)
    for i in range(warmup):
        for det in (False, True):
            step(det, i)
    torch.cuda.synchronize()
    out = {"case": case, "steps": steps}
    for det, key in ((False, "default"), (True, "deterministic")):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for i in range(steps):
                step(det, i)
            torch.cuda.synchronize()
        parts = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                k = _part(e.name)
                parts[k] = parts.get(k, 0.0) + e.time_range.elapsed_us() / 1000.0 / steps
        out[key] = {k: round(v, 4) for k, v in sorted(parts.items(), key=lambda kv: -kv[1])}
        out[key + "_total_ms"] = round(sum(parts.values()), 4)
    out["delta_ms"] = {k: round(out["deterministic"].get(k, 0.0) - out["default"].get(k, 0.0), 4)
                       for k in set(out["default"]) | set(out["deterministic"])}
    return out


def run_case(case, steps, warmup, dev):
    w, step = _build(case, dev)
    for i in range(warmup):
        for det in (False, True):
            step(det, i)
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for i in range(steps):
        for det in ((False, True) if i % 2 == 0 else (True, False)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step(det, i)
            e1.record()
            e1.synchronize()
            times[det].append(e0.elapsed_time(e1))
    peak = {}
    for det in (False, True):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        step(det, 0)
        torch.cuda.synchronize()
        peak[det] = torch.cuda.max_memory_allocated() - base
    res = {"case": case, "B": w["B"], "L": w["L"], "H": w["H"], "E": w["Et"], "C": w["C"], "steps": steps}
    for det, key in ((False, "default"), (True, "deterministic")):
        t = np.array(times[det])
        res[key] = {"median_ms": float(np.median(t)), "p10_ms": float(np.percentile(t, 10)),
                    "p90_ms": float(np.percentile(t, 90)), "step_peak_mb": peak[det] / 2 ** 20}
    res["ratio"] = res["deterministic"]["median_ms"] / res["default"]["median_ms"]
    res["peak_delta_mb"] = (peak[True] - peak[False]) / 2 ** 20
    del step
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_deterministic.py measures on the GPU and found none")
    dev = torch.device("cuda:0")
    out = {"card": card(), "results": []}
    print(json.dumps(out["card"]), flush=True)
    for case in a.cases.split(","):
        r = run_case(case, a.steps, a.warmup, dev)
        out["results"].append(r)
        print(json.dumps(r), flush=True)
    out["profiles"] = []
    for case in filter(None, a.profile.split(",")):
        r = profile_case(case, a.steps, a.warmup, dev)
        out["profiles"].append(r)
        print(json.dumps(r), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()

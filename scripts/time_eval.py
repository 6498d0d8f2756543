"""One full eval pass (main.py:267-297) with its metrics, timed two ways in the same process, alternating:
  host    forward_loss per batch; labels, predictions and loss.item() copied to the host every batch; the metrics of all
          three eval methods computed on the host at the end (sklearn for "exact" when importable, else the numpy
          restatement; the subtoken methods row by row in Python) -- what a user does today
  device  the same forward_loss per batch + Evaluator.update, one Evaluator.compute() at the end
The label vocabulary is synthetic: C labels whose subtoken lists hold 1-6 entries drawn from a Zipf(1.2) distribution
over a 50,000-subtoken vocabulary.  Half the labels of the eval set are set to the model's own prediction so that every
metric is away from 0.  Prints one JSON line per workload -- median and p10-p90 of the pass time (host clock, ending in
a device synchronise), whether the two paths' metrics agree, which host implementation ran -- and one line with the time
of Evaluator.update alone (CUDA events over many launches at B = 1024, k = 10, C = 195,299), each with the card's name,
power limit and max SM clock.

    python scripts/time_eval.py [--workloads cfg2,cfg3] [--batches 16] [--steps 10] [--warmup 2]
"""
import argparse
import json
import os
import sys
import time

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench import WORKLOADS, synth_pool  # noqa: E402
from code2vec_b200.metrics import Evaluator  # noqa: E402
from scripts.time_angular import card  # noqa: E402
from scripts.time_topk import plain_model  # noqa: E402

try:
    from sklearn.metrics import precision_recall_fscore_support
    HOST_EXACT = "sklearn"
except ImportError:
    precision_recall_fscore_support = None
    HOST_EXACT = "numpy"


def synthetic_lists(C, seed=0, n_sub=50_000, s=1.2):
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, n_sub + 1) ** s
    lens = rng.integers(1, 7, C)
    toks = rng.choice(n_sub, int(lens.sum()), p=p / p.sum()).tolist()
    out, o = [], 0
    for n in lens.tolist():
        out.append([f"s{t}" for t in toks[o:o + n]]); o += n
    return out


def host_exact(y, p, C):
    """sklearn's weighted precision / recall / F1 (zero_division=0), or the same from per-class counts in numpy"""
    if precision_recall_fscore_support is not None:
        return [float(v) for v in precision_recall_fscore_support(y, p, average="weighted", zero_division=0)[:3]]
    ok = (p >= 0) & (p < C)
    true = np.bincount(y, minlength=C).astype(np.float64)
    pred = np.bincount(p[ok], minlength=C).astype(np.float64)
    hit = np.bincount(y[p == y], minlength=C).astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        prec = np.where(pred > 0, hit / pred, 0.0)
        f1 = np.where(true + pred > 0, 2 * hit / (true + pred), 0.0)
    n = len(y)
    return [float((true * prec).sum() / n), float(hit.sum() / n), float((true * f1).sum() / n)]


def host_metrics(labels, preds, lists):
    """the metrics on the host from the collected labels and predictions (every label of the pass is in [0, C))"""
    y, p = np.concatenate(labels), np.concatenate(preds)
    n = len(y)
    acc = float((y == p).mean())
    tp = fp = fn = 0
    sp = sr = sf = 0.0
    for a, b in zip(y.tolist(), p.tolist()):
        E, P = lists[a], lists[b]
        es, ps = set(E), set(P)
        t = sum(1 for x in P if x in es)
        f, g = len(P) - t, sum(1 for x in E if x not in ps)
        tp += t; fp += f; fn += g
        sp += t / (t + f) if t + f else 0.0
        sr += t / (t + g) if t + g else 0.0
        sf += 2 * t / (2 * t + f + g) if t else 0.0
    ratio = lambda a, b: a / b if b else 0.0
    P, Rc = ratio(tp, tp + fp), ratio(tp, tp + fn)
    ex = host_exact(y, p, len(lists))
    return {"exact": [acc] + ex, "subtoken": [acc, P, Rc, ratio(2 * P * Rc, P + Rc)],
            "ave_subtoken": [acc, sp / n, sr / n, sf / n]}


def pass_host(m, batches, lists):
    labels, preds, test_loss = [], [], 0.0
    with torch.no_grad():
        for s, p, e, lab in batches:
            loss, pred = m.forward_loss(s, p, e, lab)[:2]
            labels.append(lab.cpu().numpy()); preds.append(pred.cpu().numpy())
            test_loss += loss.item()
    return host_metrics(labels, preds, lists), test_loss


def pass_device(m, batches, ev):
    ev.reset()
    with torch.no_grad():
        for s, p, e, lab in batches:
            loss, pred = m.forward_loss(s, p, e, lab)[:2]
            ev.update(pred, lab, loss)
    r = ev.compute()
    return {k: [r[k][x] for x in ("accuracy", "precision", "recall", "f1")] for k in ("exact", "subtoken", "ave_subtoken")}, \
        r["loss_sum"]


def pct(v, q):
    return float(np.percentile(v, q))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="cfg2,cfg3")
    ap.add_argument("--batches", type=int, default=16)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_eval.py measures on the GPU: no CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    for name in args.workloads.split(","):
        w = dict(WORKLOADS[name]); B = w["B"]
        m = plain_model(w, dev)
        lists = synthetic_lists(w["C"])
        s, p, e, lab = synth_pool(w, args.batches, dev, 1)
        batches = []
        for i in range(args.batches):
            sl = slice(i * B, (i + 1) * B)
            own = m.predict(s[sl], p[sl], e[sl])[0]
            keep = torch.rand(B, device=dev, generator=torch.Generator(device=dev).manual_seed(i)) < 0.5
            batches.append((s[sl], p[sl], e[sl], torch.where(keep, own, lab[sl]).contiguous()))
        ev = Evaluator(lists, dev)
        times = {"host": [], "device": []}
        res = {}
        for i in range(args.warmup + args.steps):
            for way in ("host", "device"):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res[way] = pass_host(m, batches, lists) if way == "host" else pass_device(m, batches, ev)
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[way].append((time.perf_counter() - t0) * 1e3)
        (mh, lh), (md, ld) = res["host"], res["device"]
        diff = max(abs(a - b) for k in mh for a, b in zip(mh[k], md[k]))
        agree = diff <= 1e-9 and abs(lh - ld) <= 1e-9 * max(1.0, abs(lh))
        print(json.dumps({"workload": name, "B": B, "L": w["L"], "C": w["C"], "H": w["H"], "batches": args.batches,
                          "rows": args.batches * B, "steps": args.steps, "host_exact": HOST_EXACT,
                          **{f"{way}_ms": round(float(np.median(v)), 3) for way, v in times.items()},
                          **{f"{way}_ms_p10_p90": [round(pct(v, 10), 3), round(pct(v, 90), 3)] for way, v in times.items()},
                          "metrics_agree": bool(agree), "max_metric_diff": diff, "metrics": md, "loss_sum": ld,
                          "card": info}), flush=True)
        del m, batches, s, p, e, lab
        torch.cuda.empty_cache()

    # Evaluator.update alone at the top11 label count
    C, B, k, n = 195_299, 1024, 10, 500
    ev = Evaluator(synthetic_lists(C), dev, topk=k)
    g = torch.Generator(device=dev).manual_seed(0)
    label = torch.randint(0, C, (B,), generator=g, device=dev)
    pred = torch.randint(0, C, (B, k), generator=g, device=dev)
    pred[:B // 2, 0] = label[:B // 2]
    for _ in range(20):
        ev.update(pred, label)
    ms = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            ev.update(pred, label)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / n)
    print(json.dumps({"update_only": True, "B": B, "k": k, "C": C, "launches": n, "repeats": 5,
                      "update_ms_median": round(float(np.median(ms)), 4), "update_ms_min_max": [round(min(ms), 4),
                                                                                               round(max(ms), 4)],
                      "card": info}), flush=True)


if __name__ == "__main__":
    main()

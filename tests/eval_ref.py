"""Python restatement of the evaluation counts and metrics (INTEGRATION.md, "Evaluation"): the reference of
tests/test_eval_abi.py and tests/test_eval_gpu.py for c2v_eval_accumulate and metrics_from_counters."""
import numpy as np


def row_counts(y, p, lists):
    """-> None for a skipped row, else (rank of the first hit or -1, tp, fp, fn) of label y and predictions p (best first)"""
    C = len(lists)
    if not 0 <= y < C:
        return None
    rank = next((j for j, pj in enumerate(p) if pj == y), -1)
    E = lists[y]
    P = lists[p[0]] if 0 <= p[0] < C else []
    es, ps = set(E), set(P)
    tp = sum(1 for t in P if t in es)
    return rank, tp, len(P) - tp, sum(1 for t in E if t not in ps)


def fx(num, den):
    return (num << 32) // den if den else 0


def counts(label, pred, lists, k):
    """-> (counters int64 [8 + k], class_counts int64 [3, C]) as c2v_eval_accumulate adds them from zero"""
    C = len(lists)
    label = np.asarray(label, np.int64).reshape(-1).tolist()
    pred = np.asarray(pred, np.int64).reshape(len(label), -1).tolist()
    cnt = [0] * (8 + k)
    cls = np.zeros((3, C), np.int64)
    s = 2 + k
    for y, p in zip(label, pred):
        r = row_counts(y, p, lists)
        if r is None:
            cnt[1] += 1
            continue
        rank, tp, fp, fn = r
        cnt[0] += 1
        if rank >= 0:
            cnt[2 + rank] += 1
        cnt[s] += tp; cnt[s + 1] += fp; cnt[s + 2] += fn
        cnt[s + 3] += fx(tp, tp + fp); cnt[s + 4] += fx(tp, tp + fn); cnt[s + 5] += fx(2 * tp, 2 * tp + fp + fn)
        cls[0, y] += 1
        if 0 <= p[0] < C:
            cls[1, p[0]] += 1
        if p[0] == y:
            cls[2, y] += 1
    cnt = [v - 2 ** 64 if v >= 2 ** 63 else v for v in cnt]         # unsigned sums, stored as int64 bit patterns
    return np.asarray(cnt, np.int64), cls


def subtoken_metrics(label, pred, lists):
    """-> {"subtoken": (P, R, F1), "ave_subtoken": (P, R, F1)} restated row by row"""
    rows = [row_counts(y, p, lists) for y, p in zip(np.asarray(label).tolist(),
                                                     np.asarray(pred).reshape(len(label), -1).tolist())]
    rows = [r for r in rows if r is not None]
    n = len(rows)
    tp, fp, fn = (sum(r[i] for r in rows) for i in (1, 2, 3))
    ratio = lambda a, b: a / b if b else 0.0
    p, r = ratio(tp, tp + fp), ratio(tp, tp + fn)
    sums = [sum(fx(t, t + f) for _, t, f, _ in rows), sum(fx(t, t + g) for _, t, _, g in rows),
            sum(fx(2 * t, 2 * t + f + g) for _, t, f, g in rows)]
    return {"subtoken": (p, r, ratio(2 * p * r, p + r)),
            "ave_subtoken": tuple(float(v) / 2 ** 32 / n if n else 0.0 for v in sums)}

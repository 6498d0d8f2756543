"""Evaluation metrics on the device: what the reference computes from the labels and predictions of its eval pass
(main.py:267-297) for every `option.eval_method` -- "exact", "subtoken" and "ave_subtoken" -- plus top-k accuracy.

    evaluator = Evaluator(reader.label_vocab, device, topk=1)
    with torch.no_grad():
        for starts, paths, ends, label in corpus.epoch(batch_size, max_path_length, seed=epoch, shuffle=False):
            loss, pred, _, _, _ = model.forward_loss(starts, paths, ends, label)
            evaluator.update(pred, label, loss)          # one metric kernel, no host synchronisation, no allocation
    result = evaluator.compute()                         # one device-to-host copy
    accuracy, precision, recall, f1 = (result[option.eval_method][m] for m in ("accuracy", "precision", "recall", "f1"))

`update` adds integer counts (libc2v_b200.so: `c2v_eval_accumulate`), so the result is bit-identical whatever the batch
split, row order or launch order, and `update` can be captured into a CUDA graph.  The definitions are in INTEGRATION.md,
"Evaluation"; `metrics_from_counters` turns the counts into them with plain torch operations on any device.
"""
import ctypes

import numpy as np
import torch

from . import _lib

METHODS = ("exact", "subtoken", "ave_subtoken")
_FX = 2.0 ** 32                     # the per-row fractions of "ave_subtoken" are summed in units of 2^-32
_MAX_ROWS = 2 ** 31                 # counted rows the int64 fixed-point sums hold


def subtoken_lists(label_vocab):
    """-> [C] lists of subtokens, one per label id.  label_vocab: a corpus.Vocab or the reference's Vocab (the label
    count is its len(); ids without an `itosubtokens` entry have an empty list), or a sequence of subtoken lists."""
    if hasattr(label_vocab, "itosubtokens"):
        sub = label_vocab.itosubtokens
        return [list(sub.get(c) or ()) for c in range(label_vocab.len())]
    lists = []
    for c, s in enumerate(label_vocab):
        if isinstance(s, (str, bytes)):
            raise TypeError(f"label {c}: a subtoken list is a sequence of strings, not a {type(s).__name__}")
        lists.append(list(s) if s is not None else [])
    return lists


def subtoken_table(lists):
    """Interns the subtokens of `lists` in first-occurrence order over the label ids -> (offsets int64 [C + 1],
    ids int32 [S], strings [n]): label c's subtokens are strings[i] for i in ids[offsets[c]:offsets[c + 1]]."""
    index = {}
    ids, offsets = [], [0]
    for s in lists:
        for tok in s:
            ids.append(index.setdefault(tok, len(index)))
        offsets.append(len(ids))
    if len(ids) >= 2 ** 31:
        raise ValueError(f"{len(ids)} subtokens in all: the table holds fewer than 2^31")
    return np.asarray(offsets, np.int64), np.asarray(ids, np.int32), list(index)


def _unsigned(t):
    """an int64 tensor holding unsigned 64-bit sums -> their values as float64"""
    return t.double() + (t < 0).double() * 2.0 ** 64


def metrics_from_counters(counters, class_counts, loss_sum=0.0, batches=0):
    """The metrics of all three eval methods from the counts of c2v_eval_accumulate (counters int64 [8 + k], class_counts
    int64 [3, C], tensors on any device; loss_sum: a float or float64 scalar, batches: an integer or int64 scalar) -> the
    dict Evaluator.compute returns.  Computed in float64 where the counts are, then one copy to the host.  A non-finite
    loss_sum is reported as it is and touches nothing else."""
    counters = torch.as_tensor(counters, dtype=torch.int64)
    dev = counters.device
    class_counts = torch.as_tensor(class_counts, dtype=torch.int64).to(dev)
    k = counters.numel() - _lib.EVAL_SCALARS
    if k < 1 or class_counts.dim() != 2 or class_counts.shape[0] != 3:
        raise ValueError("counters must be int64 [8 + k] (k >= 1) and class_counts int64 [3, C]")
    s = 2 + k                                                  # tp, fp, fn and the fixed-point sums start here
    c = counters.double()
    n = c[_lib.EVAL_N]
    inv_n = torch.where(n > 0, 1.0 / n.clamp(min=1), torch.zeros_like(n))
    top_k = torch.cumsum(c[_lib.EVAL_RANK_HITS:s], 0) * inv_n

    true, pred, hit = class_counts.double()
    exact_p = torch.where(pred > 0, true * hit / pred.clamp(min=1), 0.0).sum() * inv_n
    exact_r = hit.sum() * inv_n
    exact_f = torch.where(true + pred > 0, true * 2.0 * hit / (true + pred).clamp(min=1), 0.0).sum() * inv_n

    tp, fp, fn = c[s + _lib.EVAL_TP], c[s + _lib.EVAL_FP], c[s + _lib.EVAL_FN]
    ratio = lambda a, b: torch.where(b > 0, a / torch.where(b > 0, b, 1.0), 0.0)
    sub_p, sub_r = ratio(tp, tp + fp), ratio(tp, tp + fn)
    sub_f = ratio(2.0 * sub_p * sub_r, sub_p + sub_r)
    fx = _unsigned(counters[s + _lib.EVAL_PREC_FX:s + _lib.EVAL_F1_FX + 1]) / _FX
    ave = torch.where(n > 0, fx / n.clamp(min=1), torch.zeros_like(fx))

    extra = torch.stack([torch.as_tensor(loss_sum, dtype=torch.float64).to(dev).reshape(()),
                         torch.as_tensor(batches, dtype=torch.int64).to(dev).reshape(()).double()])
    flat = torch.cat([c[:2], top_k, torch.stack([exact_p, exact_r, exact_f, sub_p, sub_r, sub_f]), ave, extra]).cpu()
    v = flat.tolist()
    n_rows = int(v[0])
    if n_rows > _MAX_ROWS:
        raise OverflowError(f"{n_rows} counted rows: the fixed-point sums of ave_subtoken hold up to 2^31")
    top = v[2:2 + k]
    m = v[2 + k:2 + k + 9]
    acc = top[0]
    return {"exact": {"accuracy": acc, "precision": m[0], "recall": m[1], "f1": m[2]},
            "subtoken": {"accuracy": acc, "precision": m[3], "recall": m[4], "f1": m[5]},
            "ave_subtoken": {"accuracy": acc, "precision": m[6], "recall": m[7], "f1": m[8]},
            "top_k": top, "n": n_rows, "skipped": int(v[1]), "loss_sum": v[-2], "batches": int(v[-1])}


class Evaluator:
    """Collects every metric of the eval pass on the device.  label_vocab: a corpus.Vocab, the reference's Vocab or a
    sequence of subtoken lists (one per label id; C = their number); topk: the number of ranked predictions per row
    that `update` takes ([B] when topk == 1, [B, topk] from predict_topk).  The subtoken table is built and uploaded
    once.  State: counters int64 [8 + topk], class_counts int64 [3, C], loss_sum float64 [1], batches int64 [1]."""

    def __init__(self, label_vocab, device, topk=1):
        lists = subtoken_lists(label_vocab)
        self.label_count = C = len(lists)
        if C < 1:
            raise ValueError("the label vocabulary is empty")
        self.topk = int(topk)
        if not 1 <= self.topk <= C:
            raise ValueError(f"topk = {topk} is outside [1, label_count = {C}]")
        dev = torch.device(device)
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.device = dev
        off, ids, self.subtokens = subtoken_table(lists)
        self.subtoken_offsets = torch.from_numpy(off).to(dev)
        self.subtoken_ids = torch.from_numpy(ids if ids.size else np.zeros(1, np.int32)).to(dev)
        self.counters = torch.zeros(_lib.EVAL_SCALARS + self.topk, dtype=torch.int64, device=dev)
        self.class_counts = torch.zeros((3, C), dtype=torch.int64, device=dev)
        self.loss_sum = torch.zeros(1, dtype=torch.float64, device=dev)
        self.batches = torch.zeros(1, dtype=torch.int64, device=dev)

    def _check(self, pred, label, loss):
        for name, t in (("pred", pred), ("label", label)):
            if not isinstance(t, torch.Tensor):
                raise TypeError(f"{name} must be a torch.Tensor, not {type(t).__name__}")
            if t.dtype != torch.int64:
                raise TypeError(f"{name} must be int64, not {t.dtype}")
            if t.device != self.device:
                raise ValueError(f"{name} is on {t.device}, the evaluator on {self.device}")
        if label.dim() != 1:
            raise ValueError(f"label must be [B], not {list(label.shape)}")
        B = label.shape[0]
        want = [B] if pred.dim() == 1 and self.topk == 1 else [B, self.topk]
        if list(pred.shape) != want:
            raise ValueError(f"pred must be {want} (topk = {self.topk}), not {list(pred.shape)}")
        if B >= 2 ** 31:
            raise ValueError(f"B = {B}: at most 2^31 - 1 rows per update")
        if loss is not None:
            if not isinstance(loss, torch.Tensor) or not loss.is_floating_point():
                raise TypeError("loss must be a floating-point torch.Tensor")
            if loss.numel() != 1:
                raise ValueError(f"loss must hold one value (what loss.item() reads), not {list(loss.shape)}")
            if loss.device != self.device:
                raise ValueError(f"loss is on {loss.device}, the evaluator on {self.device}")

    def update(self, pred, label, loss=None):
        """Adds one batch on the current stream: pred int64 [B] (forward_loss / predict) or [B, topk] (predict_topk),
        label int64 [B], loss (optional) the batch's scalar loss, added into a float64 sum as the reference's
        `test_loss += loss.item()` adds it, without the read (a NaN or inf loss makes loss_sum NaN or inf, as there, and
        nothing else).  Rows whose label is outside [0, label_count) are skipped."""
        self._check(pred, label, loss)
        if self.device.type != "cuda":
            raise _lib.C2VError("Evaluator.update runs on a CUDA device; there is no CPU path")
        B = label.shape[0]
        if B:
            pred, label = pred.contiguous(), label.contiguous()
            P = lambda t: ctypes.c_void_p(t.data_ptr())
            rc = _lib.load().c2v_eval_accumulate(P(label), P(pred), B, self.topk, self.label_count, P(self.subtoken_offsets),
                                                 P(self.subtoken_ids), P(self.counters), P(self.class_counts),
                                                 ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
            _lib.check(rc, "c2v_eval_accumulate")
        if loss is not None:
            self.loss_sum.add_(loss.detach().reshape(1))
        self.batches.add_(1)

    def compute(self, group=None):
        """-> {"exact" | "subtoken" | "ave_subtoken": {"accuracy", "precision", "recall", "f1"}, "top_k": [topk],
        "n", "skipped", "loss_sum", "batches"}.  With torch.distributed initialised and more than one rank in `group`,
        the counts and the loss sum of all ranks are summed first (every rank gets the same result).  Synchronises the
        device, so it cannot run under CUDA-graph capture."""
        if self.device.type == "cuda" and torch.cuda.is_current_stream_capturing():
            raise RuntimeError("Evaluator.compute() synchronises the device and cannot run under CUDA-graph capture")
        state = (self.counters, self.class_counts, self.loss_sum, self.batches)
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            state = tuple(t.clone() for t in state)
            for t in state:
                dist.all_reduce(t, group=group)
        return metrics_from_counters(*state)

    def reset(self):
        """Zeroes the counts, the loss sum and the batch count (on the current stream)."""
        self.counters.zero_()
        self.class_counts.zero_()
        self.loss_sum.zero_()
        self.batches.zero_()

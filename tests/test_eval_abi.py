"""CPU tests of the evaluation metrics (code2vec_b200/metrics.py, c2v_eval_accumulate): argument checks of the C entry
point, the subtoken table, the finalisation from counts against sklearn and the Python restatement (tests/eval_ref.py),
and the all-reduce of the counts at world size 2 (gloo)."""
import ctypes
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import eval_ref
from code2vec_b200 import _lib
from code2vec_b200 import corpus as cc
from code2vec_b200.metrics import Evaluator, metrics_from_counters, subtoken_lists, subtoken_table
from oracle import corpus_oracle as co

FAKE = ctypes.c_void_p(0x1000)        # never dereferenced: every check runs before any CUDA call


def _call(**kw):
    a = dict(label=FAKE, pred=FAKE, B=4, k=2, C=10, subtoken_offsets=FAKE, subtoken_ids=FAKE, counters=FAKE,
             class_counts=FAKE)
    a.update(kw)
    lib = _lib.load()
    rc = lib.c2v_eval_accumulate(a["label"], a["pred"], a["B"], a["k"], a["C"], a["subtoken_offsets"], a["subtoken_ids"],
                                 a["counters"], a["class_counts"], None)
    return rc, lib.c2v_last_error().decode()


@pytest.mark.parametrize("arg", ["label", "pred", "subtoken_offsets", "subtoken_ids", "counters", "class_counts"])
def test_null_pointers_are_rejected_by_name(arg):
    rc, msg = _call(**{arg: None})
    assert rc == _lib.C2V_EINVAL and f"{arg} is NULL" in msg


@pytest.mark.parametrize("kw, name", [({"B": 0}, "B ="), ({"B": -3}, "B ="), ({"k": 0}, "k ="), ({"k": 11}, "k ="),
                                      ({"C": 0, "k": 1}, "C ="), ({"C": -1, "k": 1}, "C =")])
def test_sizes_are_rejected_by_name(kw, name):
    rc, msg = _call(**kw)
    assert rc == _lib.C2V_EINVAL and name in msg, msg


def test_counter_layout_matches_the_header():
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "c2v_b200.h")).read()
    assert "#define C2V_EVAL_COUNTERS(k) (8 + (k))" in src and _lib.EVAL_SCALARS == 8
    for name, off in (("TP", _lib.EVAL_TP), ("FP", _lib.EVAL_FP), ("FN", _lib.EVAL_FN), ("PREC_FX", _lib.EVAL_PREC_FX),
                      ("REC_FX", _lib.EVAL_REC_FX), ("F1_FX", _lib.EVAL_F1_FX)):
        assert f"#define C2V_EVAL_{name}(k) ({2 + off} + (k))" in src


# ---- subtoken table ------------------------------------------------------------------------------------------------
def _decode(lists):
    off, ids, strings = subtoken_table(lists)
    assert off[0] == 0 and off[-1] == ids.size and off.size == len(lists) + 1 and ids.dtype == np.int32
    return [[strings[i] for i in ids[off[c]:off[c + 1]]] for c in range(len(lists))], ids, strings


def _reader(tmp_path, seed, infer_method, infer_variable):
    text, term, path = co.synthetic_corpus(seed)
    files = []
    for name, t in (("corpus.txt", text), ("path_idxs.txt", path), ("terminal_idxs.txt", term)):
        p = tmp_path / name
        with open(p, "w", encoding="utf-8", newline="") as f:
            f.write(t)
        files.append(str(p))
    return cc.CorpusReader(*files, infer_method=infer_method, infer_variable=infer_variable)


@pytest.mark.parametrize("task", [(True, False), (False, True)], ids=["method", "variable"])
@pytest.mark.parametrize("seed", [1, 2])
def test_subtoken_table_of_a_corpus_reader_matches_its_itosubtokens(tmp_path, seed, task):
    vocab = _reader(tmp_path, seed, *task).label_vocab
    lists = subtoken_lists(vocab)
    assert len(lists) == vocab.len() > 1
    assert lists == [list(vocab.itosubtokens.get(c, [])) for c in range(vocab.len())]
    decoded, ids, strings = _decode(lists)
    assert decoded == lists
    seen = []                                              # interned in first-occurrence order over label ids
    for s in lists:
        seen += [t for t in s if t not in seen]
    assert strings == seen and len(set(strings)) == len(strings)


def test_subtoken_table_keeps_duplicates_and_empty_lists():
    v = cc.Vocab()
    v.append("getgetvalue", subtokens=["get", "get", "value"])
    v.append("nothing")                                    # no itosubtokens entry: empty list
    v.append("empty", subtokens=[])
    v.append("value", subtokens=["value"])
    lists = subtoken_lists(v)
    assert lists == [["get", "get", "value"], [], [], ["value"]]
    decoded, ids, strings = _decode(lists)
    assert decoded == lists and ids.tolist() == [0, 0, 1, 1] and strings == ["get", "value"]
    assert subtoken_lists([["a"], None, ()]) == [["a"], [], []]
    with pytest.raises(TypeError):
        subtoken_lists(["getValue"])


# ---- finalisation --------------------------------------------------------------------------------------------------
def _random_case(seed, C=40, n=600, k=5, n_sub=30):
    rng = np.random.default_rng(seed)
    lists = [[f"s{int(t)}" for t in rng.integers(0, n_sub, int(rng.integers(0, 5)))] for _ in range(C)]
    label = rng.integers(0, C // 2, n)                     # half of the classes never occur as a label
    label[rng.random(n) < 0.05] = -1
    label[rng.random(n) < 0.03] = -100
    label[rng.random(n) < 0.02] = C
    pred = rng.integers(0, C, (n, k))
    close = rng.random(n) < 0.4
    pred[close, 0] = np.clip(label[close], 0, C - 1)       # plenty of hits at rank 0 ...
    deep = rng.random(n) < 0.2
    pred[deep, k - 1] = np.clip(label[deep], 0, C - 1)     # ... and at deeper ranks
    pred[rng.random(n) < 0.03, 0] = -7                     # predictions outside [0, C)
    pred[rng.random(n) < 0.03, 0] = C + 3
    return lists, label.astype(np.int64), pred.astype(np.int64), k


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_metrics_from_counters_equals_sklearn_for_exact(seed):
    sk = pytest.importorskip("sklearn.metrics")
    lists, label, pred, k = _random_case(seed)
    cnt, cls = eval_ref.counts(label, pred, lists, k)
    m = metrics_from_counters(torch.from_numpy(cnt), torch.from_numpy(cls))
    keep = (label >= 0) & (label < len(lists))
    y, p = label[keep], pred[keep]
    assert m["n"] == keep.sum() and m["skipped"] == (~keep).sum()
    assert m["exact"]["accuracy"] == pytest.approx(sk.accuracy_score(y, p[:, 0]), abs=1e-15)
    prf = sk.precision_recall_fscore_support(y, p[:, 0], average="weighted", zero_division=0)
    for name, ref in zip(("precision", "recall", "f1"), prf[:3]):
        assert m["exact"][name] == pytest.approx(ref, rel=1e-12, abs=1e-15), name
    for j in range(k):
        assert m["top_k"][j] == pytest.approx(np.mean([y[i] in p[i, :j + 1] for i in range(len(y))]), abs=1e-15)
    assert m["subtoken"]["accuracy"] == m["ave_subtoken"]["accuracy"] == m["exact"]["accuracy"]


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_metrics_from_counters_equals_the_restatement_for_subtokens(seed):
    lists, label, pred, k = _random_case(seed)
    cnt, cls = eval_ref.counts(label, pred, lists, k)
    m = metrics_from_counters(torch.from_numpy(cnt), torch.from_numpy(cls), loss_sum=torch.tensor(2.5, dtype=torch.float64),
                              batches=3)
    ref = eval_ref.subtoken_metrics(label, pred, lists)
    for mode in ("subtoken", "ave_subtoken"):
        assert (m[mode]["precision"], m[mode]["recall"], m[mode]["f1"]) == ref[mode], mode
    assert m["loss_sum"] == 2.5 and m["batches"] == 3
    # the fixed-point mean is within 2^-32 of the real mean of the per-row fractions
    rows = [r for r in (eval_ref.row_counts(y, p, lists) for y, p in zip(label.tolist(), pred.tolist())) if r]
    real = np.mean([tp / (tp + fp) if tp + fp else 0.0 for _, tp, fp, _ in rows])
    assert abs(m["ave_subtoken"]["precision"] - real) <= 2.0 ** -32


@pytest.mark.parametrize("loss", [float("nan"), float("inf")])
def test_a_non_finite_loss_sum_leaves_the_metrics_and_the_batch_count(loss):
    lists, label, pred, k = _random_case(4)
    cnt, cls = eval_ref.counts(label, pred, lists, k)
    ref = metrics_from_counters(torch.from_numpy(cnt), torch.from_numpy(cls), 1.0, 3)
    m = metrics_from_counters(torch.from_numpy(cnt), torch.from_numpy(cls), torch.tensor([loss], dtype=torch.float64),
                              torch.tensor([3]))
    assert m["batches"] == 3 and (m["loss_sum"] == loss or (np.isnan(loss) and np.isnan(m["loss_sum"])))
    assert {key: v for key, v in m.items() if key != "loss_sum"} == {key: v for key, v in ref.items() if key != "loss_sum"}


def test_metrics_of_nothing_are_zero_and_too_many_rows_raise():
    cnt, cls = np.zeros(9, np.int64), np.zeros((3, 4), np.int64)
    m = metrics_from_counters(cnt, cls)
    assert m["n"] == 0 and m["top_k"] == [0.0] and all(v == 0.0 for mode in ("exact", "subtoken", "ave_subtoken")
                                                        for v in m[mode].values())
    cnt[0] = 2 ** 31 + 1
    with pytest.raises(OverflowError):
        metrics_from_counters(cnt, cls)
    cnt[0] = cnt[2] = 2 ** 31                              # every row perfect: the unsigned sums 2^63 read back exactly
    cnt[6:9] = -(2 ** 63)                                  # k = 1: the fixed-point sums are counters 6, 7, 8
    m = metrics_from_counters(cnt, cls)
    assert m["ave_subtoken"] == {"accuracy": 1.0, "precision": 1.0, "recall": 1.0, "f1": 1.0}


def test_update_checks_on_the_host():
    ev = Evaluator([["a"], ["b"], ["a", "c"]], "cpu", topk=2)
    good_p, good_l = torch.zeros(4, 2, dtype=torch.int64), torch.zeros(4, dtype=torch.int64)
    with pytest.raises(TypeError):
        ev.update(good_p.int(), good_l)
    with pytest.raises(TypeError):
        ev.update(good_p, good_l.float())
    with pytest.raises(ValueError):
        ev.update(good_p[:, :1], good_l)                   # [B, 1] for topk = 2
    with pytest.raises(ValueError):
        ev.update(good_p[:, 0], good_l)                    # [B] needs topk = 1
    with pytest.raises(ValueError):
        ev.update(good_p, good_l[:3])
    with pytest.raises(ValueError):
        ev.update(good_p, good_l, loss=torch.zeros(4))
    with pytest.raises(_lib.C2VError, match="no CPU path"):
        ev.update(good_p, good_l)
    with pytest.raises(ValueError):
        Evaluator([["a"]], "cpu", topk=2)


# ---- world size 2 ------------------------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        lists, label, pred, k = _random_case(5)
        ev = Evaluator(lists, "cpu", topk=k)
        cnt, cls = eval_ref.counts(label[rank::world], pred[rank::world], lists, k)
        ev.counters.copy_(torch.from_numpy(cnt)); ev.class_counts.copy_(torch.from_numpy(cls))
        ev.loss_sum.fill_(0.25 + rank); ev.batches.fill_(2)
        ret[rank] = ev.compute()
        ret[f"state{rank}"] = ev.counters.clone()          # compute() reduces copies, not the rank's own counts
    finally:
        dist.destroy_process_group()


def test_two_ranks_compute_the_single_process_result():
    world, port = 2, _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)
    lists, label, pred, k = _random_case(5)
    cnt, cls = eval_ref.counts(label, pred, lists, k)
    ref = metrics_from_counters(torch.from_numpy(cnt), torch.from_numpy(cls), 1.5, 4)
    assert ret[0] == ref and ret[1] == ref
    assert torch.equal(ret["state0"], torch.from_numpy(eval_ref.counts(label[0::2], pred[0::2], lists, k)[0]))

"""-m gpu: the evaluation metrics on the device (code2vec_b200/metrics.py, c2v_eval_accumulate).  The counts are integers,
so they must equal the Python restatement (tests/eval_ref.py) bit for bit at the top11 label count, for any batch split
and under CUDA-graph replay; end to end, forward_loss + Evaluator.update over a DeviceCorpus epoch must give what the
reference-style host loop (labels, predictions and loss.item() copied to the host every batch) gives."""
import numpy as np
import pytest
import torch

import eval_ref
from gpu_util import option_from, random_params
from code2vec_b200 import corpus as cc
from code2vec_b200.batch_builder import DeviceCorpus
from code2vec_b200.metrics import Evaluator, metrics_from_counters
from code2vec_b200.model import Code2Vec
from oracle import corpus_oracle as co

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
C_TOP11 = 195_299


def _lists(C, seed=0, n_sub=30_000):
    """Zipf subtoken lists of 1-6 entries, plus the edge cases at labels 0-4: empty, duplicates, 70 entries (longer than
    a warp), and a second long list that shares part of it"""
    rng = np.random.default_rng(seed)
    lens = rng.integers(1, 7, C)
    toks = (rng.zipf(1.3, int(lens.sum())) % n_sub).tolist()
    lists, o = [], 0
    for n in lens.tolist():
        lists.append([f"t{t}" for t in toks[o:o + n]]); o += n
    long = [f"t{t}" for t in rng.integers(0, 50, 70).tolist()]
    lists[0], lists[1], lists[2], lists[3], lists[4] = [], ["t5", "t5", "t7"], long, [], long[35:] + ["t5", "x"]
    return lists


@pytest.fixture(scope="module")
def top11_lists():
    return _lists(C_TOP11)


def _batch(rng, C, B, k):
    label = rng.integers(0, C, B)
    special = rng.random(B) < 0.15
    label[special] = rng.integers(0, 5, int(special.sum()))
    for v in (-1, -100, C):                                # skipped rows
        label[rng.random(B) < 0.02] = v
    pred = rng.integers(0, C, (B, k))
    top = rng.random(B) < 0.3
    pred[top, 0] = np.clip(label[top], 0, C - 1)
    if k > 1:
        deep = rng.random(B) < 0.3
        pred[deep, rng.integers(1, k, int(deep.sum()))] = np.clip(label[deep], 0, C - 1)
    near = rng.random(B) < 0.15
    pred[near, 0] = rng.integers(0, 5, int(near.sum()))    # the edge-case lists on the prediction side
    pred[rng.random(B) < 0.03, 0] = -3                     # predictions outside [0, C)
    pred[rng.random(B) < 0.03, 0] = C + 5
    return label.astype(np.int64), pred.astype(np.int64)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.parametrize("k", [1, 10, 16, 50, 1100])
def test_counts_equal_the_restatement_bit_for_bit_at_top11(top11_lists, k):
    rng = np.random.default_rng(k)
    B = 1024
    label, pred = _batch(rng, C_TOP11, B, k)
    ev = Evaluator(top11_lists, DEV, topk=k)
    ev.update(_dev(pred[:, 0] if k == 1 else pred), _dev(label))
    ev.update(_dev(pred[:, 0] if k == 1 else pred), _dev(label))       # adds, does not overwrite
    torch.cuda.synchronize()
    cnt, cls = eval_ref.counts(np.concatenate([label, label]), np.concatenate([pred, pred]), top11_lists, k)
    assert np.array_equal(ev.counters.cpu().numpy(), cnt)
    assert np.array_equal(ev.class_counts.cpu().numpy(), cls)
    assert cnt[1] > 0 and cnt[2] > 0 and (k == 1 or cnt[3:2 + k].sum() > 0)
    m = ev.compute()
    ref = metrics_from_counters(torch.from_numpy(cnt), torch.from_numpy(cls), 0.0, 2)
    _close(m, ref)


def _close(a, b):
    """metrics of the same counts, finalised on the device and on the host (float64 sums in a different order)"""
    for key in ("n", "skipped", "batches"):
        assert a[key] == b[key], key
    assert a["top_k"] == pytest.approx(b["top_k"], rel=1e-13, abs=0)
    assert a["loss_sum"] == pytest.approx(b["loss_sum"], rel=1e-13, abs=1e-12)
    for mode in ("exact", "subtoken", "ave_subtoken"):
        for name in ("accuracy", "precision", "recall", "f1"):
            assert a[mode][name] == pytest.approx(b[mode][name], rel=1e-12, abs=1e-15), (mode, name)


def test_any_batch_split_gives_the_same_counts(top11_lists):
    rng = np.random.default_rng(7)
    k, B = 10, 1024
    label, pred = _batch(rng, C_TOP11, B, k)
    perm = rng.permutation(B)
    cuts = np.sort(rng.choice(np.arange(1, B), 6, replace=False))
    splits = {"one": [np.arange(B)], "eight": np.array_split(np.arange(B), 8),
              "uneven, shuffled": np.split(perm, cuts)}
    got = []
    for name, parts in splits.items():
        ev = Evaluator(top11_lists, DEV, topk=k)
        for idx in parts:
            ev.update(_dev(pred[idx]), _dev(label[idx]))
        torch.cuda.synchronize()
        got.append((ev.counters.cpu(), ev.class_counts.cpu()))
    for c, cl in got[1:]:
        assert torch.equal(c, got[0][0]) and torch.equal(cl, got[0][1])


def test_update_replays_in_a_cuda_graph_and_compute_refuses_capture(top11_lists):
    rng = np.random.default_rng(3)
    k, B = 16, 512
    label, pred = _batch(rng, C_TOP11, B, k)
    p, lab, loss = _dev(pred), _dev(label), torch.tensor(0.7312, device=DEV)
    once = Evaluator(top11_lists, DEV, topk=k)
    once.update(p, lab, loss)
    ev = Evaluator(top11_lists, DEV, topk=k)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                          # warm-up outside the capture, as torch.cuda.graph asks
        ev.update(p, lab, loss)
    torch.cuda.current_stream().wait_stream(side)
    ev.reset()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        with pytest.raises(RuntimeError, match="capture"):
            ev.compute()
        ev.update(p, lab, loss)
    torch.cuda.synchronize()
    assert int(ev.counters.abs().sum()) == 0               # capturing ran nothing
    for _ in range(3):
        g.replay()
    torch.cuda.synchronize()
    assert torch.equal(ev.counters, 3 * once.counters) and torch.equal(ev.class_counts, 3 * once.class_counts)
    assert ev.loss_sum.tolist() == [3 * float(loss)] and ev.batches.tolist() == [3]
    assert ev.compute()["batches"] == 3


@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
def test_a_non_finite_batch_loss_changes_only_the_loss_sum(top11_lists, bad):
    """a diverged checkpoint, or a batch whose rows are all ignored under a mean-reduced criterion, gives a NaN loss: the
    loss sum becomes NaN (inf), as the reference's `test_loss += loss.item()` does, and every metric and count stays"""
    rng = np.random.default_rng(11)
    k, B = 10, 256
    batches = [_batch(rng, C_TOP11, B, k) for _ in range(3)]
    losses = [0.5, bad, 0.25]
    ev, ref = Evaluator(top11_lists, DEV, topk=k), Evaluator(top11_lists, DEV, topk=k)
    for (label, pred), loss in zip(batches, losses):
        ev.update(_dev(pred), _dev(label), torch.tensor(loss, device=DEV))
        ref.update(_dev(pred), _dev(label), torch.tensor(1.0, device=DEV))
    got, want = ev.compute(), ref.compute()
    assert got["batches"] == 3 and got["n"] > 0
    assert got["loss_sum"] == bad or (np.isnan(bad) and np.isnan(got["loss_sum"]))
    assert {key: v for key, v in got.items() if key != "loss_sum"} == {key: v for key, v in want.items() if key != "loss_sum"}
    assert all(np.isfinite(v) for mode in ("exact", "subtoken", "ave_subtoken") for v in got[mode].values())


def _reader(tmp_path, infer_method, infer_variable):
    text, term, path = co.synthetic_corpus(3, n_items=120)
    files = []
    for name, t in (("corpus.txt", text), ("path_idxs.txt", path), ("terminal_idxs.txt", term)):
        f = tmp_path / name
        f.write_text(t, encoding="utf-8")
        files.append(str(f))
    return cc.CorpusReader(*files, infer_method=infer_method, infer_variable=infer_variable)


@pytest.mark.parametrize("task", ["method", "variable"])
def test_forward_loss_and_update_over_an_epoch_equal_the_host_loop(tmp_path, task):
    reader = _reader(tmp_path, task == "method", task == "variable")
    corpus = DeviceCorpus.from_corpus(reader, DEV)
    T, P = max(reader.terminal_vocab.itos) + 1, max(reader.path_vocab.itos) + 1
    C, E = reader.label_vocab.len(), 128
    model = Code2Vec(option_from({"T": T, "P": P, "C": C, "Et": E, "Ep": E, "H": E}))
    model.load_state_dict({k: torch.from_numpy(v) for k, v in random_params(np.random.default_rng(0), T, P, C, E, E, E).items()})
    model = model.to(DEV).eval()
    epoch = corpus.epoch if task == "method" else corpus.epoch_vars
    lists = [list(reader.label_vocab.itosubtokens.get(c, [])) for c in range(C)]

    ev = Evaluator(reader.label_vocab, DEV)
    labels, preds, test_loss, batches = [], [], 0.0, 0
    with torch.no_grad():
        for starts, paths, ends, label in epoch(16, 30, seed=5, shuffle=False):
            loss, pred, _, _, _ = model.forward_loss(starts, paths, ends, label)
            ev.update(pred, label, loss)
            labels.append(label.cpu().numpy()); preds.append(pred.cpu().numpy())      # the host loop
            test_loss += loss.item(); batches += 1
    got = ev.compute()
    label, pred = np.concatenate(labels), np.concatenate(preds)
    cnt, cls = eval_ref.counts(label, pred, lists, 1)
    ref = metrics_from_counters(torch.from_numpy(cnt), torch.from_numpy(cls), test_loss, batches)
    assert batches > 2 and got["n"] == len(label) and got["batches"] == batches
    _close(got, ref)
    assert got["exact"]["accuracy"] == pytest.approx(float(np.mean(pred == label)), abs=1e-15)
    sub = eval_ref.subtoken_metrics(label, pred, lists)
    for mode in ("subtoken", "ave_subtoken"):
        assert (got[mode]["precision"], got[mode]["recall"], got[mode]["f1"]) == sub[mode]

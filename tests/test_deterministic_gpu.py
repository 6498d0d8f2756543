"""-m gpu: torch.use_deterministic_algorithms(True) makes the training step bit-reproducible.

The switch is on only around the model and optimizer calls (the `deterministic` context manager): the fp64 judge and the
torch references run outside it, because PyTorch raises under it for cuBLAS without CUBLAS_WORKSPACE_CONFIG and for
NLLLoss on CUDA.

  repeated runs     one training step three times from the same state, with an allocation between the runs so that every
                    buffer moves: torch.equal on the loss, code_vector, attention and every gradient
  cross-process     two child processes train 5 steps each and print the same SHA-256 of parameters and Adam state; eager
                    steps and GraphedTrainStep replays end on bit-identical parameters
  accuracy          the deterministic training step passes test_train_step_gpu's fp64 criterion (its LOOSER table)
  switch off        the library launches as many kernels per training step as without this mode
"""
import contextlib
import hashlib
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import test_train_step_gpu as tts
from bench import WORKLOADS, synth_params, synth_pool
from code2vec_b200 import _lib
from code2vec_b200 import functional as CF
from code2vec_b200.distributed import ShardedFlatAdam, ddp_step
from code2vec_b200.graphs import GraphedTrainStep
from code2vec_b200.model import Code2Vec

pytestmark = pytest.mark.gpu

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda:0")


@contextlib.contextmanager
def deterministic(on=True):
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


def _option(T, P, C, Et, Ep, H, dropout=0.25, angular=False):
    return types.SimpleNamespace(terminal_count=T, path_count=P, label_count=C, terminal_embed_size=Et, path_embed_size=Ep,
                                 encode_size=H, dropout_prob=dropout, angular_margin_loss=angular, angular_margin=0.5,
                                 inverse_temp=30.0, device=DEV)


def _model(opt, algo="auto", sparse=False, seed=0):
    torch.manual_seed(seed)
    m = Code2Vec(opt, algo=algo)
    with torch.no_grad():                        # trained-like scales: the gradients are not all tiny
        for p in m.parameters():
            p.add_(0.05 * torch.randn_like(p))
    m.terminal_embedding.sparse = m.path_embedding.sparse = sparse
    return m.to(DEV).train()


def _batch(opt, B, L, seed, hot_row=None):
    g = torch.Generator(device=DEV).manual_seed(seed)
    s = torch.randint(1, opt.terminal_count, (B, L), generator=g, device=DEV)
    p = torch.randint(1, opt.path_count, (B, L), generator=g, device=DEV)
    e = torch.randint(1, opt.terminal_count, (B, L), generator=g, device=DEV)
    if hot_row is not None:                      # one terminal in most contexts of every bag: one key segment, many chunks
        s[:, : (3 * L) // 4] = hot_row
    n = torch.randint(1, L + 1, (B,), generator=g, device=DEV)
    n[0] = 0                                     # an all-pad bag
    valid = (torch.arange(L, device=DEV)[None, :] < n[:, None]).long()
    lab = torch.randint(0, opt.label_count, (B,), generator=g, device=DEV)
    return s * valid, p * valid, e * valid, lab


def _packed(s, p, e):
    n = (s > 0).sum(1).clamp(min=1).cpu()
    keep = torch.arange(s.shape[1])[None, :] < n[:, None]
    k = keep.to(DEV)
    off = np.concatenate([[0], np.cumsum(n.numpy())])
    return CF.PackedBags(s[k], p[k], e[k], off, s.shape[1])


def _grads(m):
    out = {}
    for n, p in m.named_parameters():
        g = p.grad
        if g is not None and g.is_sparse:
            g = g.coalesce()
            out[n + ".indices"], out[n + ".values"] = g.indices(), g.values()
        elif g is not None:
            out[n] = g
    return {k: v.detach().clone() for k, v in out.items()}


def _step_plain(m, batch, packed):
    s, p, e, lab = batch
    m.zero_grad(set_to_none=True)
    if packed:
        res = m.forward_loss(_packed(s, p, e), None, None, lab)
    else:
        res = m.forward_loss(s, p, e, lab)
    loss, am, mx, cv, att = res
    loss.backward()
    out = {"loss": loss.detach().clone(), "am": am.clone(), "mx": mx.clone(), "cv": cv.detach().clone(),
           "att": att.detach().clone()}
    out.update(_grads(m))
    return out


# case: option, B, L, model kwargs, step kind
CASES = {
    "tc-100": (_option(5000, 7000, 300, 100, 100, 100), 64, 50, {}, "plain"),
    "tc-128": (_option(5000, 7000, 300, 128, 128, 128), 64, 50, {}, "plain"),
    "tc-256": (_option(5000, 7000, 300, 256, 256, 256), 32, 50, {}, "plain"),
    "cuda-core-odd": (_option(3000, 4000, 257, 37, 29, 45), 48, 33, {}, "plain"),
    "ffma": (_option(5000, 7000, 300, 128, 128, 128), 64, 50, {"algo": "ffma"}, "plain"),
    "packed": (_option(5000, 7000, 300, 128, 128, 128), 64, 50, {}, "packed"),
    "sparse": (_option(5000, 7000, 300, 128, 128, 128), 64, 50, {"sparse": True}, "plain"),
    "sparse-packed-odd": (_option(3000, 4000, 257, 37, 29, 45), 48, 33, {"sparse": True}, "packed"),
    "angular": (_option(5000, 7000, 300, 128, 128, 128, angular=True), 64, 50, {}, "plain"),
    "angular-ffma": (_option(5000, 7000, 300, 128, 128, 128, angular=True), 64, 50, {"algo": "ffma"}, "plain"),
    "hot-row": (_option(5000, 7000, 300, 128, 128, 128), 256, 200, {}, "hot"),
    "ddp-fused": (_option(5000, 7000, 300, 128, 128, 128), 64, 50, {}, "ddp"),
}


def _one_run(case, junk):
    opt, B, L, kw, kind = CASES[case]
    m = _model(opt, **kw)
    batch = _batch(opt, B, L, seed=11, hot_row=7 if kind == "hot" else None)
    torch.manual_seed(5)                                        # the dropout key
    junk.append(torch.empty(int(1 + 4096 * np.random.randint(1, 64)), device=DEV))   # move the next allocations
    with deterministic():
        if kind == "ddp":
            o = ShardedFlatAdam(m.parameters(), lr=0.01)
            loss = ddp_step(m, o, None, *batch, None)
            out = {"loss": loss.detach().clone(), "params": o.flat_param.clone(), "m": o.exp_avg.clone(),
                   "v": o.exp_avg_sq.clone()}
        else:
            out = _step_plain(m, batch, kind == "packed")
        # the forward's label call set the library's mode on this thread from the switch
        assert _lib.load().c2v_get_deterministic() == 1
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("case", list(CASES))
def test_repeated_runs_are_bit_identical(case):
    junk = []
    runs = [_one_run(case, junk) for _ in range(3)]
    for r in runs[1:]:
        assert r.keys() == runs[0].keys()
        for k in r:
            assert torch.equal(r[k], runs[0][k]), f"{case}: {k} differs between runs"


def test_repeated_cfg2_batch_is_bit_identical():
    """one full benchmark-size batch (cfg2: 1,024 bags of 200 contexts, dropout 0.25, fused loss)"""
    w = dict(WORKLOADS["cfg2"])
    o = types.SimpleNamespace(terminal_count=w["T"], path_count=w["P"], label_count=w["C"], terminal_embed_size=w["Et"],
                              path_embed_size=w["Ep"], encode_size=w["H"], dropout_prob=0.25, angular_margin_loss=False,
                              angular_margin=0.5, inverse_temp=30.0, device=DEV)
    m = Code2Vec(o)
    m.load_state_dict(synth_params(w, DEV))
    m = m.to(DEV).train()
    s, p, e, lab = synth_pool(w, 1, DEV, 99)
    runs, junk = [], []
    for _ in range(2):
        torch.manual_seed(3)
        junk.append(torch.empty(int(1 + 65536 * np.random.randint(1, 64)), device=DEV))
        with deterministic():
            runs.append(_step_plain(m, (s, p, e, lab), False))
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), f"cfg2: {k} differs between runs"


@pytest.mark.parametrize("kind", ["hot", "plain"])
def test_gradients_match_the_atomic_path(kind):
    """the same backward with the switch off (atomics) and on (sorted keys, chunk sums, merge) differs only in the order of
    its sums.  "hot": one terminal row in 3/4 of the contexts of every bag -- its sorted keys span about 900 chunks, so
    the merge's cooperative path sums them"""
    opt_ = _option(5000, 7000, 300, 128, 128, 128)
    batch = _batch(opt_, 256, 200, seed=11, hot_row=7 if kind == "hot" else None)
    res = []
    for on in (False, True):
        m = _model(opt_)
        torch.manual_seed(5)
        with deterministic(on):
            res.append(_step_plain(m, batch, False))
    for k, ref in res[0].items():
        if k in ("am",):
            continue
        d = (res[1][k] - ref).abs().max().item()
        scale = ref.abs().max().item()
        assert d <= 1e-5 * scale + 1e-30, f"{kind}: {k}: max |det - atomic| = {d:.3g} of max |g| = {scale:.3g}"


CHILD = r"""
import hashlib, sys, types
import torch
sys.path.insert(0, {repo!r})
from code2vec_b200.model import Code2Vec
from code2vec_b200.distributed import ShardedFlatAdam, ddp_step
torch.use_deterministic_algorithms(True)
dev = torch.device("cuda:0")
o = types.SimpleNamespace(terminal_count=5000, path_count=7000, label_count=300, terminal_embed_size=128,
                          path_embed_size=128, encode_size=128, dropout_prob=0.25, angular_margin_loss=False,
                          angular_margin=0.5, inverse_temp=30.0, device=dev)
torch.manual_seed(0)
m = Code2Vec(o).to(dev).train()
opt = ShardedFlatAdam(m.parameters(), lr=0.01)
g = torch.Generator(device=dev).manual_seed(1)
for step in range(5):
    s = torch.randint(0, 5000, (64, 50), generator=g, device=dev)
    p = torch.randint(0, 7000, (64, 50), generator=g, device=dev)
    e = torch.randint(0, 5000, (64, 50), generator=g, device=dev)
    lab = torch.randint(0, 300, (64,), generator=g, device=dev)
    ddp_step(m, opt, None, s, p, e, lab, None)
torch.cuda.synchronize()
h = hashlib.sha256()
for k, v in sorted(m.state_dict().items()):
    h.update(k.encode()); h.update(v.detach().cpu().numpy().tobytes())
h.update(opt.exp_avg.cpu().numpy().tobytes()); h.update(opt.exp_avg_sq.cpu().numpy().tobytes())
print("DIGEST", h.hexdigest())
"""


def test_two_processes_train_to_the_same_digest():
    digests = []
    for _ in range(2):
        r = subprocess.run([sys.executable, "-c", CHILD.format(repo=REPO)], cwd=REPO, capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0, r.stderr[-4000:]
        line = [x for x in r.stdout.splitlines() if x.startswith("DIGEST")]
        assert line, r.stdout[-2000:]
        digests.append(line[-1])
    assert digests[0] == digests[1], digests


def test_eager_steps_and_graph_replays_agree():
    opt_ = _option(5000, 7000, 300, 128, 128, 128)
    B, L = 64, 50
    batches = [_batch(opt_, B, L, seed=20 + i) for i in range(5)]
    params = []
    for graphed in (False, True):
        m = _model(opt_)
        m.use_device_rng(seed=77)
        o = ShardedFlatAdam(m.parameters(), lr=0.01, capturable=True)
        with deterministic():
            step = GraphedTrainStep(m, o, B, L) if graphed else None
            for b in batches:
                if graphed:
                    step(*b)
                else:
                    ddp_step(m, o, None, *b, None)
        torch.cuda.synchronize()
        params.append(o.flat_param.clone())
    assert torch.equal(params[0], params[1])


def test_graphed_step_refuses_a_mode_change():
    opt_ = _option(5000, 7000, 300, 128, 128, 128)
    B, L = 32, 20
    m = _model(opt_)
    m.use_device_rng(seed=5)
    o = ShardedFlatAdam(m.parameters(), lr=0.01, capturable=True)
    step = GraphedTrainStep(m, o, B, L)
    b = _batch(opt_, B, L, seed=1)
    for _ in range(3):                           # warm-up, warm-up, capture
        step(*b)
    with deterministic():
        with pytest.raises(RuntimeError, match="deterministic"):
            step(*b)


@pytest.mark.parametrize("case", ["cfg2", "cfg3", "cfg4"])
def test_deterministic_step_matches_fp64_reference(case, monkeypatch):
    """test_train_step_gpu's case with the switch on around the training step only"""
    plain = tts.ddp_step

    def det_step(*a, **k):
        with deterministic():
            return plain(*a, **k)
    monkeypatch.setattr(tts, "ddp_step", det_step)
    report, failures = tts._run_case(case)
    print(f"\n[deterministic train-step {case}] {report}")
    assert not failures, "\n".join(failures)


# c2v_launch_count() of one training step with the switch off, at _option(5000, 7000, 300, 128, 128, 128), B = 64,
# L = 50 (fused loss + backward, then a ShardedFlatAdam ddp_step), as the library launched before this mode existed;
# recorded with the library of the parent commit on an H100 80GB HBM3.
LAUNCHES_OFF = {"forward_loss+backward": 17, "ddp_step": 21}


def _count_launches():
    lib = _lib.load()
    opt_ = _option(5000, 7000, 300, 128, 128, 128)
    b = _batch(opt_, 64, 50, seed=3)
    m = _model(opt_)
    _step_plain(m, b, False)                     # warm-up: persistent workspaces
    n0 = lib.c2v_launch_count()
    _step_plain(m, b, False)
    n1 = lib.c2v_launch_count()
    o = ShardedFlatAdam(m.parameters(), lr=0.01)
    ddp_step(m, o, None, *b, None)
    n2 = lib.c2v_launch_count()
    ddp_step(m, o, None, *b, None)
    n3 = lib.c2v_launch_count()
    return {"forward_loss+backward": n1 - n0, "ddp_step": n3 - n2}


def test_switch_off_launches_as_before():
    with deterministic(False):
        got = _count_launches()
    with deterministic(True):
        on = _count_launches()
    print(f"\nlaunches per step with the switch off: {got}, on: {on}")
    assert got == LAUNCHES_OFF
    # with it on the fixed-order kernels run (key build, sort, chunk sums, merge, slab sums): more launches
    assert on["forward_loss+backward"] > got["forward_loss+backward"] and on["ddp_step"] > got["ddp_step"]

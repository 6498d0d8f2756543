"""-m gpu: the data-parallel SparseAdam step.  c2v_sparse_union_rows + c2v_sparse_adam_step_merged against torch bit for
bit (the gradient summed in fp32 in rank order, times 1/W, then torch.optim.SparseAdam on CUDA), and FusedSparseAdam's
data-parallel step on one GPU with emulated ranks (threads meeting in a substituted all-gather) on a real Code2Vec
against a single-process step, judged against fp64 (scripts/check_sparse_ddp.py's reference)."""
import os
import sys
import threading

import numpy as np
import pytest
import torch
import torch.nn as nn

from conftest import ROOT
from code2vec_b200 import functional as CF
from code2vec_b200.distributed import FusedSparseAdam

sys.path.insert(0, os.path.join(ROOT, "scripts"))
import check_sparse_ddp as ref    # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
VOCAB = 300
KINDS = ("random", "disjoint", "identical", "nested", "one_empty", "all_empty", "edges", "full")


def _lists(rng, W, kind):
    """W ascending row lists of a table of VOCAB rows"""
    pick = lambda n: np.sort(rng.choice(VOCAB, n, replace=False))
    if kind == "random":
        return [pick(int(rng.integers(0, 60))) for _ in range(W)]
    if kind == "disjoint":
        perm = rng.permutation(VOCAB)
        return [np.sort(perm[r::W][:40]) for r in range(W)]
    if kind == "identical":
        a = pick(50)
        return [a.copy() for _ in range(W)]
    if kind == "nested":                              # each list a subset of the one before
        a, out = pick(120), []
        for _ in range(W):
            out.append(a)
            a = np.sort(rng.choice(a, max(len(a) * 2 // 3, 1), replace=False))
        return out
    if kind == "one_empty":
        return [pick(30) if r != W // 2 else np.zeros(0, np.int64) for r in range(W)]
    if kind == "all_empty":
        return [np.zeros(0, np.int64) for _ in range(W)]
    if kind == "edges":                               # row 0 and row VOCAB - 1 on some ranks only
        return [np.unique(np.concatenate([pick(10), [0] if r % 2 == 0 else [], [VOCAB - 1] if r == W - 1 else []]))
                .astype(np.int64) for r in range(W)]
    assert kind == "full"                             # the union covers the whole table
    return [np.arange(VOCAB)[r::W] if W > 1 else np.arange(VOCAB) for r in range(W)]


def _gathered(rng, lists, E):
    """what the all-gathers leave: rows [W, u_max], values [W, u_max, E], counts [W] (padding: garbage, never read)"""
    W = len(lists)
    u_max = max(len(a) for a in lists)
    rows = torch.from_numpy(rng.integers(-5, 2 * VOCAB, (W, u_max))).to(DEV)
    values = torch.full((W, u_max, E), float("nan"), device=DEV)
    vals = []
    for r, a in enumerate(lists):
        v = torch.from_numpy(rng.standard_normal((len(a), E)).astype(np.float32)).to(DEV)
        rows[r, :len(a)] = torch.from_numpy(a.astype(np.int64)).to(DEV)
        values[r, :len(a)] = v
        vals.append(v)
    counts = torch.tensor([len(a) for a in lists], dtype=torch.int64, device=DEV)
    return rows, values, counts, vals


def _reference_grad(lists, vals, E, W):
    """the union's gradient in torch: fp32 sum in rank order, times the fp32 1/W"""
    total = torch.zeros(VOCAB, E, device=DEV)
    for a, v in zip(lists, vals):
        total[torch.from_numpy(a.astype(np.int64)).to(DEV)] += v
    union = torch.unique(torch.from_numpy(np.concatenate(lists + [np.zeros(0)]).astype(np.int64))).to(DEV)
    inv = torch.tensor(1.0 / W, dtype=torch.float32).item()
    return union, total[union] * inv


@pytest.mark.parametrize("E", [4, 37, 100, 128, 256])
@pytest.mark.parametrize("W", [1, 2, 3, 8, 16])
def test_union_and_merged_step_match_torch_bitwise(W, E):
    rng = np.random.default_rng(100 * W + E)
    kw = dict(lr=0.0123, betas=(0.85, 0.995), eps=1e-6)
    for kind in KINDS:
        w0 = torch.from_numpy(rng.standard_normal((VOCAB, E)).astype(np.float32)).to(DEV)
        p_ref, p = nn.Parameter(w0.clone()), w0.clone()
        opt = torch.optim.SparseAdam([p_ref], **kw)
        m, v = torch.zeros_like(p), torch.zeros_like(p)
        for step in (1, 2):
            lists = _lists(rng, W, kind)
            rows, values, counts, vals = _gathered(rng, lists, E)
            union, count = CF.sparse_union_rows(rows, counts, VOCAB)
            exp_union, g = _reference_grad(lists, vals, E, W)
            U = int(count.item())
            assert U == exp_union.numel() and torch.equal(union[:U], exp_union), kind
            assert union.numel() == min(VOCAB, W * rows.shape[1])
            p_ref.grad = torch.sparse_coo_tensor(exp_union[None], g, p_ref.shape, is_coalesced=True)
            opt.step()
            again = [t.clone() for t in (p, m, v)]
            CF.sparse_adam_step_merged(p, m, v, values, rows, counts, union, count, kw["lr"], *kw["betas"], kw["eps"], step,
                                       torch.tensor(1.0 / W, dtype=torch.float32).item())
            CF.sparse_adam_step_merged(*again, values, rows, counts, union, count, kw["lr"], *kw["betas"], kw["eps"], step,
                                       torch.tensor(1.0 / W, dtype=torch.float32).item())
            st = opt.state[p_ref]
            assert torch.equal(p, p_ref.detach()), (kind, step)
            assert torch.equal(m, st["exp_avg"]) and torch.equal(v, st["exp_avg_sq"]), (kind, step)
            assert all(torch.equal(a, b) for a, b in zip(again, (p, m, v))), (kind, step)   # two runs, the same bits


@pytest.mark.parametrize("maximize,tensor_lr", [(True, False), (False, True), (True, True)])
@pytest.mark.parametrize("W", [2, 3])
def test_data_parallel_step_options_match_torch_bitwise(W, maximize, tensor_lr):
    """FusedSparseAdam at world size W (emulated ranks) with maximize and a tensor lr, against torch.optim.SparseAdam on
    the reduced gradient"""
    rng = np.random.default_rng(W)
    E = 64
    w0 = torch.from_numpy(rng.standard_normal((VOCAB, E)).astype(np.float32)).to(DEV)
    lr = torch.tensor(0.02, dtype=torch.float64) if tensor_lr else 0.02
    p_ref = nn.Parameter(w0.clone())
    opt_ref = torch.optim.SparseAdam([p_ref], lr=0.02, maximize=maximize)
    reps = [nn.Parameter(w0.clone()) for _ in range(W)]
    opts = [FusedSparseAdam([q], lr=lr, maximize=maximize) for q in reps]
    for _ in range(3):
        lists = _lists(rng, W, "random")
        _, _, _, vals = _gathered(rng, lists, E)
        for q, a, v in zip(reps, lists, vals):
            q.grad = torch.sparse_coo_tensor(torch.from_numpy(a.astype(np.int64))[None].to(DEV), v, q.shape)
        _emulated_step(opts)
        union, g = _reference_grad(lists, vals, E, W)
        p_ref.grad = torch.sparse_coo_tensor(union[None], g, p_ref.shape, is_coalesced=True)
        opt_ref.step()
        for q, o in zip(reps, opts):
            assert torch.equal(q.detach(), p_ref.detach())
            assert torch.equal(o.state[q]["exp_avg"], opt_ref.state[p_ref]["exp_avg"])
            assert o.state[q]["step"] == opt_ref.state[p_ref]["step"]


class _Ranks:
    """W emulated ranks in threads of one process: all_gather stacks every rank's tensor once all have arrived"""

    def __init__(self, world):
        self.world, self.slots, self.barrier = world, [None] * world, threading.Barrier(world)

    def gather(self, rank, t):
        self.slots[rank] = t.clone()
        self.barrier.wait()
        out = torch.stack(self.slots)
        self.barrier.wait()                           # every rank has read the slots before they are refilled
        return out


def _emulated_step(opts):
    """one data-parallel step of the W optimizers (rank = position), each in a thread, through _Ranks"""
    ranks = _Ranks(len(opts))
    errors = []
    for r, o in enumerate(opts):
        o._world_size = lambda: ranks.world
        o._all_gather = (lambda r_: lambda t: ranks.gather(r_, t))(r)

    def run(o):
        try:
            o.step()
        except BaseException as e:                    # noqa: BLE001 -- re-raised below
            errors.append(e)
            ranks.barrier.abort()
    threads = [threading.Thread(target=run, args=(o,)) for o in opts]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    torch.cuda.synchronize()
    if errors:
        raise errors[0]


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("W", [2, 4])
@pytest.mark.parametrize("dims", [(128, 128, 128), (100, 100, 100)])
def test_emulated_data_parallel_step_on_code2vec(dims, W, packed):
    params, batch = ref.make_case(31 + W, dims, 8 * W)
    model = ref.make_model(params, dims, DEV)
    tables = [model.terminal_embedding.weight, model.path_embedding.weight]
    shards = [ref.shard_grads(model, batch, W, r, packed, DEV) for r in range(W)]
    reps = [[nn.Parameter(t.detach().clone()) for t in tables] for _ in range(W)]
    opts = [FusedSparseAdam(ps, lr=ref.LR, betas=ref.BETAS, eps=ref.EPS) for ps in reps]
    for ps, gs in zip(reps, shards):
        for p, g in zip(ps, gs):
            p.grad = g
    _emulated_step(opts)
    for ps, o in zip(reps[1:], opts[1:]):                 # bit-identical replicas
        for i, p in enumerate(ps):
            assert torch.equal(p.detach(), reps[0][i].detach())
            for k in ("exp_avg", "exp_avg_sq"):
                assert torch.equal(o.state[p][k], opts[0].state[reps[0][i]][k])
    single, _ = ref.step_copy(tables, ref.table_grads(model, ref.inputs(batch, 0, 8 * W, packed, DEV)))
    for i in range(2):
        p64, rows = ref.fp64_sparse_adam(tables[i], [s[i] for s in shards])
        assert torch.equal(rows, single[i].grad.coalesce().indices()[0])     # the union is the whole batch's rows
        ref.judge(reps[0][i].detach(), single[i].detach(), p64, rows)

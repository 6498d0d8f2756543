"""world_size-2 gloo tests (CPU) of FusedSparseAdam's data-parallel step: the count / rows / values all-gathers and the
step rules (union of the ranks' rows, mean of their gradients, None and empty gradients) with the device work replaced
by a torch restatement of c2v_sparse_union_rows + c2v_sparse_adam_step_merged."""
import os

import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn
import torch.nn.functional as F

from code2vec_b200.distributed import FusedSparseAdam, ShardedFlatAdam, broadcast_parameters, shard_items
from test_distributed_gloo import _free_port, _torch_adam_slice

LR, STEPS, N = 0.01, 3, 16


def _torch_merged_step(self, p, state, rows, values, counts, lr, beta1, beta2, eps, scale):
    """the union of the lists and torch's sparse_adam on their rank-ordered fp32 sum times `scale`"""
    W = rows.shape[0]
    E = p[0].numel()
    total = torch.zeros(p.shape[0], E, dtype=torch.float32)
    seen = torch.zeros(p.shape[0], dtype=torch.bool)
    for r in range(W):                                     # rank order; each list holds a row at most once
        n = max(int(counts[r]), 0)
        total[rows[r, :n]] += values[r, :n].reshape(n, E)
        seen[rows[r, :n]] = True
    union = seen.nonzero()[:, 0]
    if union.numel() == 0:
        return
    grad = torch.sparse_coo_tensor(union[None], (total[union] * scale).reshape((-1,) + tuple(p.shape[1:])), p.shape)
    torch.optim._functional.sparse_adam([p], [grad.coalesce()], [state["exp_avg"]], [state["exp_avg_sq"]],
                                        [state["step"]], eps=eps, beta1=beta1, beta2=beta2, lr=lr, maximize=False)


class SparseBag(nn.Module):
    """TinyBag with sparse tables: terminal and path embeddings with nn.Embedding(sparse=True) + a dense head"""

    def __init__(self):
        super().__init__()
        self.term = nn.Embedding(50, 8, sparse=True)
        self.path = nn.Embedding(40, 8, sparse=True)
        self.lin = nn.Linear(8, 5)

    def forward(self, starts, paths, ends):
        return self.lin(torch.tanh(self.term(starts) + self.path(paths) + self.term(ends)).mean(1))


def _batch(g):
    # rank 1's shard never indexes rows 40..49 of the terminal table: those rows come from rank 0 alone
    starts = torch.randint(0, 50, (N, 6), generator=g); ends = torch.randint(0, 50, (N, 6), generator=g)
    starts[N // 2:] %= 40; ends[N // 2:] %= 40
    return starts, torch.randint(0, 40, (N, 6), generator=g), ends, torch.randint(0, 5, (N,), generator=g)


def _loss(model, starts, paths, ends, label):
    return F.nll_loss(F.log_softmax(model(starts, paths, ends), dim=1), label)


def _extra():
    torch.manual_seed(11)
    return [nn.Parameter(torch.randn(20, 3)) for _ in range(4)]


def _sp(rows, vals, shape):
    return torch.sparse_coo_tensor(torch.tensor(rows, dtype=torch.int64)[None], vals, shape)


def _extra_grads(rank, extra):
    """a: rank 0 only (None on rank 1); b: empty on rank 0; c: None on both; d: empty on both"""
    a, b, c, d = extra
    g = torch.Generator().manual_seed(5 + rank)
    a.grad = _sp([1, 5, 19], torch.randn(3, 3, generator=g), a.shape) if rank == 0 else None
    b.grad = _sp([], torch.zeros(0, 3), b.shape) if rank == 0 else _sp([0, 5], torch.randn(2, 3, generator=g), b.shape)
    c.grad = None
    d.grad = _sp([], torch.zeros(0, 3), d.shape)


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ShardedFlatAdam._adam_slice = _torch_adam_slice
        FusedSparseAdam._merged_step = _torch_merged_step
        torch.manual_seed(100 + rank)                       # different init per rank: the broadcast makes them equal
        model = SparseBag()
        broadcast_parameters(model, src=0)
        tables = [model.term.weight, model.path.weight]
        dense = ShardedFlatAdam([model.lin.weight, model.lin.bias], lr=LR)
        sparse = FusedSparseAdam(tables, lr=LR, group=dist.group.WORLD)
        g = torch.Generator().manual_seed(7)
        idx = shard_items(list(range(N)))
        for _ in range(STEPS):
            starts, paths, ends, label = _batch(g)
            _loss(model, starts[idx], paths[idx], ends[idx], label[idx]).backward()
            assert model.term.weight.grad.is_sparse
            dense.step(); sparse.step(); sparse.zero_grad()
        ret[f"model{rank}"] = {k: v.clone() for k, v in model.state_dict().items()}
        ret[f"sd{rank}"] = sparse.state_dict()
        extra = _extra()
        opt = FusedSparseAdam(extra, lr=LR, betas=(0.8, 0.99))
        _extra_grads(rank, extra)
        opt.step()
        ret[f"extra{rank}"] = [p.detach().clone() for p in extra]
        ret[f"extra_sd{rank}"] = opt.state_dict()
    finally:
        dist.destroy_process_group()


def test_two_rank_sparse_step_equals_single_process_sparse_adam_on_the_global_batch():
    world, port = 2, _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)
    # the replicas are identical, parameters and optimizer state
    for k, v in ret["model0"].items():
        assert torch.equal(ret["model1"][k], v), k
    sd0, sd1 = ret["sd0"], ret["sd1"]
    assert sd0["param_groups"] == sd1["param_groups"]
    for i in sd0["state"]:
        assert sd0["state"][i]["step"] == sd1["state"][i]["step"] == STEPS
        for name in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(sd0["state"][i][name], sd1["state"][i][name]), (i, name)
    # ... and match one process with torch.optim.SparseAdam + Adam on the whole batch, rank 0's init
    torch.manual_seed(100)
    model = SparseBag()
    sparse = torch.optim.SparseAdam([model.term.weight, model.path.weight], lr=LR)
    dense = torch.optim.Adam([model.lin.weight, model.lin.bias], lr=LR)
    g = torch.Generator().manual_seed(7)
    for _ in range(STEPS):
        _loss(model, *_batch(g)).backward()
        dense.step(); sparse.step(); dense.zero_grad(); sparse.zero_grad()
    for k, v in model.state_dict().items():
        assert torch.allclose(ret["model0"][k], v, atol=2e-6), k
    ref_sd = sparse.state_dict()
    for i in ref_sd["state"]:
        for name in ("exp_avg", "exp_avg_sq"):
            assert torch.allclose(sd0["state"][i][name], ref_sd["state"][i][name], atol=1e-6), (i, name)


def test_none_and_empty_gradients_follow_torchs_rules_on_every_rank():
    world, port = 2, _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)
    for a, b in zip(ret["extra0"], ret["extra1"]):
        assert torch.equal(a, b)
    sd0, sd1 = ret["extra_sd0"], ret["extra_sd1"]
    # a (None on rank 1), b (empty on rank 0) and d (empty on both) are stepped; c (None on both) is not
    assert sorted(sd0["state"]) == sorted(sd1["state"]) == [0, 1, 3]
    assert all(sd0["state"][i]["step"] == 1 for i in (0, 1, 3))
    # the reference: torch.optim.SparseAdam on the mean of the two ranks' gradients (a missing one counts as empty)
    extra = _extra()
    grads = []
    for rank in (0, 1):
        _extra_grads(rank, extra)
        grads.append([p.grad for p in extra])
    ref = torch.optim.SparseAdam(extra, lr=LR, betas=(0.8, 0.99))
    for i, p in enumerate(extra):
        gs = [g[i] for g in grads if g[i] is not None]
        p.grad = None if not gs else (sum(gs[1:], gs[0]).coalesce() * 0.5)
    ref.step()
    for i, p in enumerate(extra):
        assert torch.allclose(ret["extra0"][i], p.detach(), atol=1e-7), i
    assert sorted(ref.state_dict()["state"]) == [0, 1, 3]
    assert torch.equal(ret["extra0"][2], _extra()[2]) and torch.equal(ret["extra0"][3], _extra()[3])

"""FusedSparseAdam's data-parallel step with real NCCL, one process per GPU:

    python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 scripts/check_sparse_ddp.py

Every rank builds the same Code2Vec (both tables sparse, the same seeded weights), takes its shard of one global batch
(padded, then PackedBags), runs forward_loss / backward and FusedSparseAdam(tables, group=WORLD).step().  Checks: the
tables and the optimizer state are bit-identical on every rank, and they match a single-process step on the whole batch,
both judged against an fp64 SparseAdam on the mean of the shards' gradients (`judge`).  Prints PASS on every rank that
passed.  The helpers are shared with tests/test_sparse_ddp_gpu.py, which runs the same check on one GPU with emulated
ranks."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for d in (ROOT, os.path.join(ROOT, "tests")):
    if d not in sys.path:
        sys.path.insert(0, d)
from gpu_util import option_from, random_params     # noqa: E402
from code2vec_b200 import functional as CF          # noqa: E402
from code2vec_b200.distributed import FusedSparseAdam, shard_range   # noqa: E402
from code2vec_b200.model import Code2Vec             # noqa: E402

T, P, C, L = 600, 500, 11, 16
LR, BETAS, EPS = 0.01, (0.9, 0.999), 1e-8


def make_case(seed, dims, B):
    """seeded weights and one global batch of B bags: (params, (starts, paths, ends, label, lengths)) on the host"""
    rng = np.random.default_rng(seed)
    Et, Ep, H = dims
    params = random_params(rng, T, P, C, Et, Ep, H)
    s, p, e = rng.integers(1, 60, (B, L)), rng.integers(1, 50, (B, L)), rng.integers(1, T, (B, L))
    n = rng.integers(1, L + 1, B)
    for b in range(B):
        s[b, n[b]:] = 0; p[b, n[b]:] = 0; e[b, n[b]:] = 0
    lab = rng.integers(0, C, B)
    return params, [torch.from_numpy(np.ascontiguousarray(a, np.int64)) for a in (s, p, e, lab)] + [n]


def make_model(params, dims, dev):
    Et, Ep, H = dims
    m = Code2Vec(option_from({"T": T, "P": P, "C": C, "Et": Et, "Ep": Ep, "H": H}))
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    m = m.to(dev).train()
    m.terminal_embedding.sparse = m.path_embedding.sparse = True
    return m


def inputs(batch, lo, hi, packed, dev):
    """bags [lo, hi) of the batch, padded or as PackedBags -> (starts, paths, ends, label)"""
    s, p, e, lab, n = (x[lo:hi] for x in batch)
    if not packed:
        return s.to(dev), p.to(dev), e.to(dev), lab.to(dev)
    keep = torch.from_numpy(np.arange(L)[None, :] < n[:, None])
    off = np.concatenate([[0], np.cumsum(n)])
    return CF.PackedBags(s[keep].to(dev), p[keep].to(dev), e[keep].to(dev), off, L), None, None, lab.to(dev)


def table_grads(model, args):
    """the two tables' sparse gradients of forward_loss on `args` (coalesced, cloned)"""
    model.zero_grad(set_to_none=True)
    model.forward_loss(*args)[0].backward()
    out = [model.terminal_embedding.weight.grad.clone(), model.path_embedding.weight.grad.clone()]
    model.zero_grad(set_to_none=True)
    assert all(g.is_sparse for g in out)
    return out


def shard_grads(model, batch, world, rank, packed, dev):
    lo, hi = shard_range(len(batch[4]), rank, world)
    return table_grads(model, inputs(batch, lo, hi, packed, dev))


def step_copy(tables, grads):
    """one FusedSparseAdam step of copies of `tables` on `grads`, one process -> (params, optimizer)"""
    ps = [torch.nn.Parameter(t.detach().clone()) for t in tables]
    opt = FusedSparseAdam(ps, lr=LR, betas=BETAS, eps=EPS)
    for p, g in zip(ps, grads):
        p.grad = g
    opt.step()
    return ps, opt


def fp64_sparse_adam(table, shard_grads_of_table):
    """torch's first SparseAdam step in fp64 on the mean of the shards' gradients"""
    g = sum(x.double().to_dense() for x in shard_grads_of_table) / len(shard_grads_of_table)
    rows = torch.unique(torch.cat([x.coalesce().indices()[0] for x in shard_grads_of_table]))
    p = table.detach().double().clone()
    gr = g[rows]
    m = (1 - BETAS[0]) * gr
    v = (1 - BETAS[1]) * gr * gr
    step_size = LR * (1 - BETAS[1]) ** 0.5 / (1 - BETAS[0])
    p[rows] -= step_size * m / (v.sqrt() + EPS)
    return p, rows


def judge(p_dp, p_single, p64, rows):
    """the data-parallel step's error against fp64, in units of lr, next to the single-process step's on the whole batch.
    Both see the mean gradient; the single-process one computes it in one backward, the data-parallel one adds the
    shards' in fp32.  Where a gradient element nearly cancels, Adam's first step (about lr * sign(g)) flips with
    last-bit changes, so the bound is the single-process error, or 1e-3 lr."""
    e_dp = float((p_dp.double() - p64).abs().max()) / LR
    e_single = float((p_single.double() - p64).abs().max()) / LR
    untouched = torch.ones(p64.shape[0], dtype=torch.bool, device=p64.device)
    untouched[rows] = False
    assert torch.equal(p_dp.double()[untouched], p64[untouched]), "a row outside the union moved"
    assert e_dp <= max(e_single, 1e-3), (e_dp, e_single)
    return e_dp, e_single


def main():
    import torch.distributed as dist
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    rank, world = dist.get_rank(), dist.get_world_size()
    ok = True
    try:
        for dims, packed in (((128, 128, 128), False), ((128, 128, 128), True), ((100, 100, 100), False)):
            params, batch = make_case(7 + dims[0], dims, 8 * world)
            model = make_model(params, dims, dev)
            tables = [model.terminal_embedding.weight, model.path_embedding.weight]
            grads = shard_grads(model, batch, world, rank, packed, dev)
            ps = [torch.nn.Parameter(t.detach().clone()) for t in tables]
            opt = FusedSparseAdam(ps, lr=LR, betas=BETAS, eps=EPS, group=dist.group.WORLD)
            for p, g in zip(ps, grads):
                p.grad = g
            opt.step()
            for i, p in enumerate(ps):                          # bit-identical replicas
                st = opt.state[p]
                for t in (p.detach(), st["exp_avg"], st["exp_avg_sq"]):
                    got = [torch.empty_like(t) for _ in range(world)]
                    dist.all_gather(got, t.contiguous())
                    if not all(torch.equal(x, got[0]) for x in got):
                        ok = False
                        print(f"rank {rank}: {dims} packed={packed} table {i}: replicas differ", flush=True)
            # the reference on every rank: every shard's gradient, the single-process step and fp64
            all_shards = [shard_grads(model, batch, world, r, packed, dev) for r in range(world)]
            single, _ = step_copy(tables, table_grads(model, inputs(batch, 0, len(batch[4]), packed, dev)))
            for i in range(2):
                p64, rows = fp64_sparse_adam(tables[i], [s[i] for s in all_shards])
                e_dp, e_single = judge(ps[i].detach(), single[i].detach(), p64, rows)
                if rank == 0:
                    print(f"{dims} packed={packed} table {i}: world {world}, |dp - fp64| = {e_dp:.3g} lr, "
                          f"|single - fp64| = {e_single:.3g} lr", flush=True)
    except AssertionError as e:
        ok = False
        print(f"rank {rank}: FAIL {e}", flush=True)
    finally:
        dist.destroy_process_group()
    if ok:
        print(f"PASS rank {rank}", flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()

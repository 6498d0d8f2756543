"""world_size-2 gloo tests (CPU) of the N>1 host logic: sharding, the single flat-bucket allreduce,
and that N ranks on shards of a global batch produce the single-process gradients / parameters."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn as nn
import torch.nn.functional as F

from code2vec_b200.distributed import (FlatGradBucket, broadcast_parameters, ddp_step, shard_items, shard_range,
                                       sharded_layout)


def test_shard_range_partitions_everything():
    for n in (0, 1, 7, 8, 9, 1000, 14048):
        for w in (1, 2, 4, 8):
            r = [shard_range(n, k, w) for k in range(w)]
            assert r[0][0] == 0 and r[-1][1] == n
            assert all(r[i][1] == r[i + 1][0] for i in range(w - 1))
            sizes = [hi - lo for lo, hi in r]
            assert max(sizes) - min(sizes) <= 1


class TinyBag(nn.Module):
    """CPU stand-in with the same call surface (the CUDA module cannot run here): embedding bag + head."""

    def __init__(self):
        super().__init__()
        self.emb = nn.Embedding(50, 8)
        self.lin = nn.Linear(8, 5)

    def forward(self, starts, paths, ends, label):
        cv = torch.tanh(self.emb(starts) + self.emb(ends)).mean(1)
        return self.lin(cv), cv, None


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close(); return p


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.manual_seed(100 + rank)                       # different init per rank on purpose
        model = TinyBag()
        broadcast_parameters(model, src=0)
        bucket = FlatGradBucket(model.parameters())
        opt = torch.optim.Adam(model.parameters(), lr=0.01)
        g = torch.Generator().manual_seed(7)
        starts = torch.randint(0, 50, (16, 6), generator=g); ends = torch.randint(0, 50, (16, 6), generator=g)
        label = torch.randint(0, 5, (16,), generator=g)
        idx = shard_items(list(range(16)))                  # this rank's bags of the global batch
        loss_fn = lambda out, lab: F.nll_loss(F.log_softmax(out, dim=1), lab)
        ddp_step(model, opt, bucket, starts[idx], starts[idx], ends[idx], label[idx], loss_fn)
        bucket.check_views()
        ret[rank] = {k: v.clone() for k, v in model.state_dict().items()}
        ret[f"g{rank}"] = bucket.flat.clone()
    finally:
        dist.destroy_process_group()


def test_two_rank_step_equals_single_process_step_on_the_global_batch():
    world, port = 2, _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)
    # single-process reference on the whole batch, rank 0's init
    torch.manual_seed(100)
    model = TinyBag()
    opt = torch.optim.Adam(model.parameters(), lr=0.01)
    g = torch.Generator().manual_seed(7)
    starts = torch.randint(0, 50, (16, 6), generator=g); ends = torch.randint(0, 50, (16, 6), generator=g)
    label = torch.randint(0, 5, (16,), generator=g)
    bucket = FlatGradBucket(model.parameters())
    bucket.zero()
    out, _, _ = model.forward(starts, starts, ends, label)
    F.nll_loss(F.log_softmax(out, dim=1), label).backward()
    assert torch.allclose(ret["g0"], bucket.flat, atol=1e-6) and torch.allclose(ret["g1"], bucket.flat, atol=1e-6)
    opt.step()
    for k, v in model.state_dict().items():
        assert torch.allclose(ret[0][k], v, atol=1e-6), k
        assert torch.equal(ret[0][k], ret[1][k]), k         # replicas stay bit-identical


def test_bucket_is_one_buffer_and_detects_broken_views():
    m = TinyBag()
    b = FlatGradBucket(m.parameters())
    assert b.numel == sum(p.numel() for p in m.parameters()) and b.nbytes() == 4 * b.numel
    b.check_views()
    torch.optim.SGD(m.parameters(), lr=0.1).zero_grad(set_to_none=True)
    with pytest.raises(RuntimeError):
        b.check_views()


# ---- sharded optimizer (reduce-scatter -> Adam on the owned slice -> all-gather) --------------------------------
def _torch_adam_slice(self, p_slice, g_slice, zero_grad=False, state=None):
    m_, v_ = state if state is not None else (self.exp_avg, self.exp_avg_sq)
    """CPU stand-in for `c2v_adam_step` (same operation order; the CUDA kernels are checked against an fp64 Adam on the
    GPU by tests/test_adam_gpu.py): TEST INFRASTRUCTURE, patched in below."""
    b1, b2 = self.betas
    g = g_slice * (1.0 / self.world)
    if self.weight_decay:
        g = g + self.weight_decay * p_slice
    m_.lerp_(g, 1 - b1)
    v_.mul_(b2).addcmul_(g, g, value=1 - b2)
    bc1, bc2 = 1 - b1 ** self.t, 1 - b2 ** self.t
    denom = v_.sqrt() / (bc2 ** 0.5) + self.eps
    p_slice.addcdiv_(m_, denom, value=-self.lr / bc1)
    if zero_grad:
        g_slice.zero_()


def _sharded_worker(rank, world, port, ret):
    from code2vec_b200.distributed import ShardedFlatAdam
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        torch.manual_seed(100 + rank)
        model = TinyBag()
        broadcast_parameters(model, src=0)
        ShardedFlatAdam._adam_slice = _torch_adam_slice
        opt = ShardedFlatAdam(model.parameters(), lr=0.01, weight_decay=0.01, early=[model.lin.weight])   # two regions
        assert opt.transport == "nccl" and opt.padded % (4 * world) == 0 and opt.exp_avg.numel() * world == opt.padded
        assert len(opt.regions) == 2 and opt.params[0] is model.lin.weight
        # lin.weight (40) is region 0, emb.weight + lin.bias (405) region 1, both padded to multiples of 4 * world = 8
        assert opt.regions == [(0, 40), (40, 408)] and opt.padded == 448
        assert opt.slices == [(20 * rank, 20, 0), (40 + 204 * rank, 204, 20)] and opt.state_numel == 224
        g = torch.Generator().manual_seed(7)
        loss_fn = lambda out, lab: F.nll_loss(F.log_softmax(out, dim=1), lab)
        for step in range(3):
            starts = torch.randint(0, 50, (16, 6), generator=g); ends = torch.randint(0, 50, (16, 6), generator=g)
            label = torch.randint(0, 5, (16,), generator=g)
            idx = shard_items(list(range(16)))
            ddp_step(model, opt, None, starts[idx], starts[idx], ends[idx], label[idx], loss_fn)
            assert float(opt.buckets[1 - opt.cur].abs().max()) > 0 or step == 0      # last step's bucket is the stale one ...
            assert float(opt.bucket.abs().max()) == 0.0                                # ... and the next one starts zeroed
        ret[rank] = {k: v.clone() for k, v in model.state_dict().items()}
        ret[f"m{rank}"] = opt.exp_avg.clone()
        ret["layout"] = (opt.regions, [s_[1:] for s_ in opt.slices])
    finally:
        dist.destroy_process_group()


def test_sharded_layout_tiles_every_region():
    for n_early, numel in ((0, 1), (0, 445), (40, 445), (3, 4), (5003, 75004)):
        for world in (1, 2, 3, 4, 7, 16):
            per_rank = [sharded_layout(n_early, numel, world, r) for r in range(world)]
            regions = per_rank[0][0]
            assert len(regions) == (2 if n_early else 1)
            assert regions[0][0] == 0 and all(n % (4 * world) == 0 for _, n in regions)
            assert regions[-1][0] + regions[-1][1] - numel < 4 * world * len(regions)
            if n_early:
                assert n_early <= regions[0][1] < n_early + 4 * world and regions[1][0] == regions[0][1]
            for r, (reg, slices, state_numel) in enumerate(per_rank):
                assert reg == regions and state_numel == sum(n for _, n in regions) // world
                o = 0
                for (begin, n), (lo, sl, so) in zip(regions, slices):
                    assert sl == n // world and lo == begin + r * sl and so == o      # slice r of the region, state packed
                    o += sl


def test_sharded_adam_two_ranks_equal_single_process_adam_on_the_global_batch():
    world, port = 2, _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_sharded_worker, args=(world, port, ret), nprocs=world, join=True)
    torch.manual_seed(100)
    model = TinyBag()
    opt = torch.optim.Adam(model.parameters(), lr=0.01, weight_decay=0.01)
    g = torch.Generator().manual_seed(7)
    for step in range(3):
        starts = torch.randint(0, 50, (16, 6), generator=g); ends = torch.randint(0, 50, (16, 6), generator=g)
        label = torch.randint(0, 5, (16,), generator=g)
        opt.zero_grad()
        out, _, _ = model.forward(starts, starts, ends, label)
        F.nll_loss(F.log_softmax(out, dim=1), label).backward()
        opt.step()
    for k, v in model.state_dict().items():
        assert torch.allclose(ret[0][k], v, atol=2e-6), k
        assert torch.equal(ret[0][k], ret[1][k]), k         # replicas stay bit-identical
    # the optimizer state is sharded: the two slices together are the single-process exp_avg
    regions, slices = ret["layout"]                        # region 0 = the early parameter (lin.weight), region 1 = the rest
    early = model.lin.weight
    order = [[early], [p for p in model.parameters() if p is not early]]
    for r, (begin, n) in enumerate(regions):
        sl, so = slices[r]
        got = torch.cat([ret["m0"][so:so + sl], ret["m1"][so:so + sl]])
        full = torch.cat([opt.state[p]["exp_avg"].reshape(-1) for p in order[r]])
        assert torch.allclose(got[:full.numel()], full, atol=2e-6), r
        assert float(got[full.numel():].abs().max()) == 0.0 if got.numel() > full.numel() else True

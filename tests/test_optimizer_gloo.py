"""world_size-2 gloo test (CPU) of ShardedFlatAdam's checkpoints: state_dict() all-gathers the sharded moments into
torch.optim.Adam's full dict on every rank, load_state_dict() keeps this rank's slices, and a checkpoint saved at world
size 2 resumes at world size 2 and at world size 1.  The Adam kernel is replaced by the torch stand-in of
test_distributed_gloo.py."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

from code2vec_b200.distributed import ShardedFlatAdam, broadcast_parameters, ddp_step, shard_items
from test_distributed_gloo import TinyBag, _free_port, _torch_adam_slice

LR, WD, STEPS, MORE = 0.01, 0.01, 3, 2


def _batch(g):
    starts = torch.randint(0, 50, (16, 6), generator=g); ends = torch.randint(0, 50, (16, 6), generator=g)
    return starts, ends, torch.randint(0, 5, (16,), generator=g)


def _loss(out, lab):
    return F.nll_loss(F.log_softmax(out, dim=1), lab)


def _train(model, opt, g, steps):
    for _ in range(steps):
        starts, ends, label = _batch(g)
        idx = shard_items(list(range(16))) if dist.is_initialized() else slice(None)
        ddp_step(model, opt, None, starts[idx], starts[idx], ends[idx], label[idx], _loss)


def _new(seed):
    torch.manual_seed(seed)
    model = TinyBag()
    if dist.is_initialized():
        broadcast_parameters(model, src=0)
    return model, ShardedFlatAdam(model.parameters(), lr=LR, weight_decay=WD, early=[model.lin.weight])


def _params(model):
    return {k: v.clone() for k, v in model.state_dict().items()}


def _worker(rank, world, port, ret):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        ShardedFlatAdam._adam_slice = _torch_adam_slice
        g = torch.Generator().manual_seed(7)
        model, opt = _new(100 + rank)
        _train(model, opt, g, STEPS)
        sd, msd = opt.state_dict(), _params(model)
        ret[f"sd{rank}"] = sd
        ret[f"model{rank}"] = msd
        g_state = g.get_state()
        _train(model, opt, g, MORE)                                # the uninterrupted run
        ret[f"straight{rank}"] = _params(model)
        model2, opt2 = _new(300 + rank)                            # resume in a fresh pair at world size 2
        model2.load_state_dict(msd)
        opt2.load_state_dict(sd)
        assert opt2.t == STEPS
        g.set_state(g_state)
        _train(model2, opt2, g, MORE)
        ret[f"resumed{rank}"] = _params(model2)
        with pytest.raises(NotImplementedError, match="one process"):
            ShardedFlatAdam(TinyBag().parameters(), max_grad_norm=1.0)
    finally:
        dist.destroy_process_group()


def test_sharded_state_dict_is_torch_adams_and_resumes_at_either_world_size(monkeypatch):
    world, port = 2, _free_port()
    ret = mp.Manager().dict()
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)
    # the full dict on both ranks, equal to a single-process torch Adam's on the global batch
    torch.manual_seed(100)
    model = TinyBag()
    ref = torch.optim.Adam(model.parameters(), lr=LR, weight_decay=WD)
    g = torch.Generator().manual_seed(7)
    for _ in range(STEPS):
        starts, ends, label = _batch(g)
        ref.zero_grad()
        _loss(model.forward(starts, starts, ends, label)[0], label).backward()
        ref.step()
    ref_sd, sd0, sd1 = ref.state_dict(), ret["sd0"], ret["sd1"]
    assert sd0["param_groups"] == sd1["param_groups"] and sd0["param_groups"][0]["params"] == [0, 1, 2]
    for i, p in enumerate(model.parameters()):
        assert sorted(sd0["state"][i]) == sorted(ref_sd["state"][i])
        for k, v in ref_sd["state"][i].items():
            assert torch.equal(sd0["state"][i][k], sd1["state"][i][k]), (i, k)
            assert sd0["state"][i][k].shape == v.shape and sd0["state"][i][k].dtype == v.dtype
            assert torch.allclose(sd0["state"][i][k], v, atol=2e-6), (i, k)
    for k, v in ret["straight0"].items():
        assert torch.equal(ret["resumed0"][k], v) and torch.equal(ret["resumed1"][k], v), k
    # the same checkpoint at world size 1 (this process): the gradient of the global batch is the mean of the shards'
    monkeypatch.setattr(ShardedFlatAdam, "_adam_slice", _torch_adam_slice)
    model1, opt1 = _new(500)
    model1.load_state_dict(ret["model0"])
    opt1.load_state_dict(sd0)
    assert opt1.world == 1 and opt1.t == STEPS
    _train(model1, opt1, g, MORE)
    for k, v in ret["straight0"].items():
        assert torch.allclose(model1.state_dict()[k], v, atol=2e-6), k

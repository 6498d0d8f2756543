"""torchrun --nproc-per-node N scripts/check_sharded_adam.py : ShardedFlatAdam (nvls / p2p / nccl transports) against
torch.optim.Adam on the rank-averaged gradients, 4 steps, weight decay on; replicas must stay bit-identical.
Also times the step's communication phase on a cfg2-sized flat buffer (91 M parameters).

Every rank prints one machine-readable line per transport case, whether it ran or not:
  TRANSPORT {"rank": 0, "case": "p2p", "early": false, "ran": true, "transport": "p2p", "max_err": 1e-07, "identical": true}
  TRANSPORT {"rank": 0, "case": "nvls", "early": false, "ran": false, "reason": "RuntimeError: ..."}
A transport that cannot be set up is reported, not failed, here; only a failing run (or an nccl case that cannot run)
fails the script.  tests/test_sharded_adam_multigpu.py decides which missing transports are failures."""
import json, os, sys
R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, R)
import torch, torch.distributed as dist
from code2vec_b200.distributed import ShardedFlatAdam

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local); dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
ok = True
shapes = [(1000, 37), (513,), (64, 129), (7,), (300, 128)]
for transport, use_early in (("nvls", False), ("p2p", False), ("nccl", False), ("nvls", True), ("p2p", True)):
    try:
        g = torch.Generator(device=dev).manual_seed(5)
        params = [torch.nn.Parameter(torch.randn(*s, generator=g, device=dev)) for s in shapes]
        ref = [torch.nn.Parameter(p.detach().clone()) for p in params]
        ropt = torch.optim.Adam(ref, lr=0.01, weight_decay=0.01)
        opt = ShardedFlatAdam(params, lr=0.01, weight_decay=0.01, transport=transport, early=[params[2]] if use_early else ())
        for step in range(4):
            gr = torch.Generator(device=dev).manual_seed(100 * step + rank)
            mine = [torch.randn(*s, generator=gr, device=dev) for s in shapes]
            for p, m in zip(params, mine):
                p.grad.add_(m)                       # backward accumulates into the (zeroed) bucket views
            if use_early:
                opt.early_step()                     # region 0 (params[2]) on the side stream, as from inside the backward
            opt.step()
            allg = []
            for r in range(world):
                gg = torch.Generator(device=dev).manual_seed(100 * step + r)
                allg.append([torch.randn(*s, generator=gg, device=dev) for s in shapes])
            for i, p in enumerate(ref):
                p.grad = sum(a[i] for a in allg) / world
            ropt.step()
            assert float(opt.bucket.abs().max()) == 0.0, "next bucket not zeroed"
        err = max(float((a - b).abs().max()) for a, b in zip(params, ref))
        flat = opt.flat_param.clone()
        ref0 = flat.clone(); dist.broadcast(ref0, 0)
        same = bool(torch.equal(flat, ref0))
        print(f"[rank {rank}] {transport}{' + early region' if use_early else ''}: transport={opt.transport} max|p - torch.Adam| = {err:.2e} replicas identical: {same}", flush=True)
        print("TRANSPORT " + json.dumps(dict(rank=rank, case=transport, early=use_early, ran=True, transport=opt.transport,
                                             max_err=err, identical=same)), flush=True)
        ok &= err < 2e-6 and same
        del opt
    except Exception as ex:
        print(f"[rank {rank}] {transport}: unavailable ({type(ex).__name__}: {ex})", flush=True)
        print("TRANSPORT " + json.dumps(dict(rank=rank, case=transport, early=use_early, ran=False,
                                             reason=f"{type(ex).__name__}: {ex}")), flush=True)
        if transport == "nccl":
            ok = False
# ---- timing on a cfg2-sized buffer ----------------------------------------------------------------------------------
n = 91_144_960
for transport in ("nvls", "p2p", "nccl"):
    try:
        big = [torch.nn.Parameter(torch.zeros(n, device=dev))]
        opt = ShardedFlatAdam(big, lr=0.01, transport=transport)
        for _ in range(3):
            opt.bucket.fill_(0.001); opt.step()
        torch.cuda.synchronize(); dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        iters = 10
        e0.record()
        for _ in range(iters):
            opt.step()
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        t = torch.tensor([ms], device=dev); dist.all_reduce(t, op=dist.ReduceOp.MAX)
        if rank == 0:
            print(f"TIMING {opt.transport}: {t.item():.3f} ms per step for {4 * n / 1e6:.1f} MB of gradients over {world} GPUs "
                  f"(reduction + Adam + broadcast)", flush=True)
        del opt, big
        torch.cuda.empty_cache()
    except Exception as ex:
        if rank == 0:
            print(f"TIMING {transport}: unavailable ({type(ex).__name__}: {ex})", flush=True)
print(f"[rank {rank}] {'PASS' if ok else 'FAIL'}", flush=True)
dist.destroy_process_group()
sys.exit(0 if ok else 1)

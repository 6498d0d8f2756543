"""Data-parallel plumbing for the training loop (BASELINE.json north_star: "training shards the corpus
across the 8 GPUs of one box with a single NCCL allreduce on the gradients per step over NVLink").

The reference has no distributed code at all; this adds
the minimum: bags are independent, so the forward shards with no collective; only the gradients meet.

  shard_range / shard_items : contiguous shard of the methods of the corpus for a rank
  FlatGradBucket            : every parameter's .grad is a view into ONE flat fp32 buffer, so the step
                              needs exactly one all_reduce (NCCL over NVLink/NVSwitch; gloo in the CPU tests)
  ddp_step                  : zero_grad -> forward -> loss -> backward -> allreduce -> optimizer.step,
                              the body of main.py:171-175 with the collective inserted
torch.distributed is only plumbing here (process group, the collective); launch one process per GPU with
`python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 ...`.
"""
import torch
import torch.distributed as dist


def shard_range(n_items, rank, world):
    """[lo, hi) of a contiguous, balanced split of n_items (first n_items % world ranks get one more)."""
    base, rem = divmod(n_items, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_items(items, rank=None, world=None):
    rank = dist.get_rank() if rank is None else rank
    world = dist.get_world_size() if world is None else world
    lo, hi = shard_range(len(items), rank, world)
    return items[lo:hi]


class FlatGradBucket:
    """All gradients of `params` live in one flat buffer; `allreduce()` is the step's single collective."""

    def __init__(self, params):
        self.params = [p for p in params if p.requires_grad]
        if not self.params:
            raise ValueError("no trainable parameters")
        dev, dt = self.params[0].device, self.params[0].dtype
        self.numel = sum(p.numel() for p in self.params)
        self.flat = torch.zeros(self.numel, dtype=dt, device=dev)
        o = 0
        for p in self.params:
            if p.device != dev or p.dtype != dt:
                raise ValueError("parameters must share device and dtype")
            p.grad = self.flat[o:o + p.numel()].view_as(p)     # a view: backward accumulates in place
            o += p.numel()

    def zero(self):
        """optimizer.zero_grad(set_to_none=False) for the whole model in one memset (main.py:171)."""
        self.flat.zero_()

    def check_views(self):
        """.grad must still alias the flat buffer (zero_grad(set_to_none=True) would break that)."""
        o = 0
        for p in self.params:
            if p.grad is None or p.grad.data_ptr() != self.flat.data_ptr() + o * self.flat.element_size():
                raise RuntimeError("a .grad no longer aliases the flat bucket; use bucket.zero(), not "
                                   "optimizer.zero_grad(set_to_none=True)")
            o += p.numel()

    def nbytes(self):
        return self.numel * self.flat.element_size()

    def allreduce(self, average=True):
        """ONE all_reduce(sum) over the flat bucket, then 1/world (mean of per-rank mean losses ==
        mean over the global batch when every rank holds the same number of bags)."""
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            dist.all_reduce(self.flat, op=dist.ReduceOp.SUM)
            if average:
                self.flat.mul_(1.0 / dist.get_world_size())


class FlatAdam:
    """torch.optim.Adam(model.parameters(), lr, betas, weight_decay) (main.py:138) as ONE kernel launch per step
    (`c2v_adam_step`): parameters, like the gradients of `bucket`, become views into one flat buffer; the step reads
    p, g, m, v once, writes p, m, v and leaves the gradient zeroed for the next backward (main.py:171), folding the
    1/world of the data-parallel mean into the read.  Dense, same update rule and operation order as torch's Adam."""

    def __init__(self, bucket, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0):
        self.bucket = bucket
        self.lr, self.betas, self.eps, self.weight_decay = float(lr), (float(betas[0]), float(betas[1])), float(eps), float(weight_decay)
        flat = torch.empty_like(bucket.flat)
        o = 0
        for p in bucket.params:                                  # same order as the gradient bucket
            n = p.numel()
            flat[o:o + n].copy_(p.data.reshape(-1))
            p.data = flat[o:o + n].view_as(p)
            o += n
        self.flat_param = flat
        self.exp_avg = torch.zeros_like(flat)
        self.exp_avg_sq = torch.zeros_like(flat)
        self.t = 0

    def step(self, grad_scale=1.0, zero_grad=True):
        import ctypes
        from . import _lib
        lib = _lib.load()
        self.t += 1
        P = lambda t: ctypes.c_void_p(t.data_ptr())
        dev = self.flat_param.device
        with torch.cuda.device(dev):
            rc = lib.c2v_adam_step(P(self.flat_param), P(self.bucket.flat), P(self.exp_avg), P(self.exp_avg_sq),
                                   self.flat_param.numel(), self.lr, self.betas[0], self.betas[1], self.eps,
                                   self.weight_decay, self.t, float(grad_scale), 1 if zero_grad else 0,
                                   ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        _lib.check(rc, "c2v_adam_step")
        # the kernel wrote through raw pointers: tell autograd (and the weight-image caches of the model, which key on
        # Tensor._version) that every parameter changed, as an in-place torch op would
        for p in self.bucket.params:
            torch.autograd.graph.increment_version(p)

    def zero_grad(self):
        self.bucket.zero()


class ShardedFlatAdam:
    """Data-parallel Adam with the optimizer state sharded over the ranks and the gradient reduction fused into the
    optimizer kernel.  Same update rule, dense, as
    torch.optim.Adam (main.py:138) -- every rank ends a step with bit-identical parameters.

    Layout: parameters live in ONE flat fp32 buffer (views, like FlatAdam), gradients in TWO flat buckets that alternate
    between steps (`.grad` of every parameter is re-pointed after each step).  The flat buffers consist of one or two
    REGIONS, each padded to a multiple of 4 * world; rank r owns slice r of every region (exp_avg / exp_avg_sq exist only
    for the owned slices: 1/world of the state).  With `early=[p, ...]` those parameters form region 0: their gradients
    are complete before the backward ends (path_embedding, once the path sub-vector of dC has run), and `early_step()` --
    called from inside the backward -- reduces / updates / broadcasts region 0 on a side stream while the rest of the
    backward is still computing; `step()` then handles region 1 and joins.

    transport
      "nvls"  buffers are symmetric memory (torch.distributed._symmetric_memory: plumbing only -- allocation, the
              multicast mapping, the cross-GPU barriers); one `c2v_adam_step_sharded` launch per rank and region reduces
              the slice's gradients in the NVSwitch (`multimem.ld_reduce`), runs Adam, and multicasts the new parameters
              (`multimem.st`), zero-filling the other bucket meanwhile.  No NCCL call in the step.
      "p2p"   same kernel, peer pointers instead of the multicast mapping (NVLink loads / stores, rank-ordered sum).
      "nccl"  reduce_scatter -> `c2v_adam_step` on the slice -> all_gather (two NCCL collectives; the fallback when
              symmetric memory is unavailable, and what the gloo CPU tests drive with a stand-in kernel).
      "auto"  nvls or p2p, whichever is faster on this group (timed at construction), else nccl.
    """

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, group=None, transport="auto",
                 early=()):
        params = [p for p in params if p.requires_grad]
        if not params:
            raise ValueError("no trainable parameters")
        early_ids = {id(p) for p in early}
        first = [p for p in params if id(p) in early_ids]
        self.params = first + [p for p in params if id(p) not in early_ids]      # flat order: early region first
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if self.world > 1 else 0
        self.lr, self.betas, self.eps, self.weight_decay = float(lr), (float(betas[0]), float(betas[1])), float(eps), float(weight_decay)
        dev, dt = self.params[0].device, self.params[0].dtype
        if dt != torch.float32:
            raise TypeError("parameters must be fp32")
        self.numel = sum(p.numel() for p in self.params)
        q = 4 * self.world
        pad = lambda n: (n + q - 1) // q * q
        n_early = sum(p.numel() for p in first)
        # regions: (begin, length) in the flat buffers; region 0 = the early parameters (absent when there are none)
        self.regions = ([(0, pad(n_early))] if n_early else []) + \
            [(pad(n_early) if n_early else 0, pad(self.numel - n_early))]
        self.padded = sum(n for _, n in self.regions)
        # this rank's slice of every region, and where its optimizer state sits in exp_avg / exp_avg_sq
        self.slices, o = [], 0
        for begin, n in self.regions:
            sl = n // self.world
            self.slices.append((begin + self.rank * sl, sl, o))
            o += sl
        self.state_numel = o
        self._auto = transport == "auto"
        self.transport, self._hdl = self._allocate(transport, dev)
        self._grad_views = ([], [])
        self.flat_param.zero_()
        pos = {}
        o = 0
        for i, p in enumerate(self.params):
            if p.device != dev or p.dtype != dt:
                raise ValueError("parameters must share device and dtype")
            if n_early and i == len(first):
                o = self.regions[1][0]                           # region 1 starts after region 0's padding
            pos[i] = o
            o += p.numel()
        for i, p in enumerate(self.params):
            n, o = p.numel(), pos[i]
            self.flat_param[o:o + n].copy_(p.data.reshape(-1))
            p.data = self.flat_param[o:o + n].view_as(p)
            for k in (0, 1):
                self._grad_views[k].append(self.buckets[k][o:o + n].view_as(p))
        self.exp_avg = torch.zeros(self.state_numel, dtype=dt, device=dev)
        self.exp_avg_sq = torch.zeros(self.state_numel, dtype=dt, device=dev)
        self.t, self.cur = 0, 0
        self._early_done = False
        self._side = torch.cuda.Stream(dev) if (dev.type == "cuda" and len(self.regions) > 1) else None
        self._point_grads(0)
        if self.world > 1:
            dist.barrier(group)
        self.calibration = None
        if self._auto and self.transport == "nvls":
            self._calibrate()

    def _calibrate(self):
        """transport="auto" with a multicast mapping available: time the fused kernel both ways on the real buffers
        (zero gradients, zero optimizer state, lr = 0: nothing changes) and keep the faster: which one wins depends on the
        number of GPUs and the fabric."""
        dev = self.flat_param.device
        res = {}
        saved = (self.lr, self.weight_decay)
        self.lr, self.weight_decay = 0.0, 0.0
        try:
            for tr in ("nvls", "p2p"):
                self.transport = tr
                for i in range(6):
                    if i == 2:
                        torch.cuda.synchronize(dev)
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                    self.t = 0
                    self.step()
                e1.record()
                torch.cuda.synchronize(dev)
                t = torch.tensor([e0.elapsed_time(e1) / 4], dtype=torch.float64, device=dev)
                dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.group)
                res[tr] = float(t.item())
        finally:
            self.lr, self.weight_decay = saved
            self.t = 0
        self.transport = min(res, key=res.get)
        self.calibration = res

    # ---- buffers ------------------------------------------------------------------------------------------------------
    def _allocate(self, transport, dev):
        n = self.padded
        want = transport
        if self.world > 1 and want in ("auto", "nvls", "p2p") and dev.type == "cuda":
            try:
                import torch.distributed._symmetric_memory as symm
                g = self.group if self.group is not None else dist.group.WORLD
                bufs = [symm.empty(n, dtype=torch.float32, device=dev) for _ in range(3)]
                hdls = [symm.rendezvous(b, g) for b in bufs]
                for b in bufs:
                    b.zero_()
                self.flat_param, self.buckets = bufs[0], (bufs[1], bufs[2])
                mc = all(int(h.multicast_ptr) != 0 for h in hdls)
                if want == "nvls" and not mc:
                    raise RuntimeError("this process group has no NVSwitch multicast support")
                return ("nvls" if (mc and want != "p2p") else "p2p"), hdls
            except Exception:
                if want in ("nvls", "p2p"):
                    raise
        if want in ("nvls", "p2p") and self.world > 1:
            raise RuntimeError(f"transport {want!r} needs CUDA symmetric memory")
        self.flat_param = torch.empty(n, dtype=torch.float32, device=dev)
        self.buckets = (torch.zeros(n, dtype=torch.float32, device=dev), torch.zeros(n, dtype=torch.float32, device=dev))
        return "nccl", None

    def _point_grads(self, k):
        for p, v in zip(self.params, self._grad_views[k]):
            p.grad = v
        self.cur = k

    @property
    def bucket(self):
        """the flat gradient bucket the next backward accumulates into"""
        return self.buckets[self.cur]

    def state_bytes(self):
        return 4 * (2 * self.state_numel)

    def zero_grad(self):
        self.buckets[self.cur].zero_()

    # ---- the step -----------------------------------------------------------------------------------------------------
    def _adam_slice(self, p_slice, g_slice, zero_grad=False, state=None):
        """c2v_adam_step on an owned slice (the gloo CPU tests replace this method with a torch stand-in)"""
        import ctypes
        from . import _lib
        lib = _lib.load()
        P = lambda t: ctypes.c_void_p(t.data_ptr())
        m, v = state if state is not None else (self.exp_avg, self.exp_avg_sq)
        dev = p_slice.device
        with torch.cuda.device(dev):
            rc = lib.c2v_adam_step(P(p_slice), P(g_slice), P(m), P(v), p_slice.numel(), self.lr,
                                   self.betas[0], self.betas[1], self.eps, self.weight_decay, self.t, 1.0 / self.world,
                                   1 if zero_grad else 0, ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        _lib.check(rc, "c2v_adam_step")

    def _reduce_scatter(self, out, full):
        try:
            dist.reduce_scatter_tensor(out, full, op=dist.ReduceOp.SUM, group=self.group)
        except (RuntimeError, NotImplementedError):          # gloo (CPU tests) has no reduce_scatter
            tmp = full.clone()
            dist.all_reduce(tmp, op=dist.ReduceOp.SUM, group=self.group)
            sl = full.numel() // self.world
            out.copy_(tmp[self.rank * sl:(self.rank + 1) * sl])

    def _bulk_region(self, r, cur):
        """barrier -> c2v_adam_step_sharded_bulk (one warp + 28 KB of shared memory per CTA: fits beside the persistent
        backward kernels) on this rank's slice of region r -> barrier, on the current (side) stream.  No zero-fill."""
        import ctypes
        from . import _lib
        lib = _lib.load()
        hp, hg = self._hdl[0], self._hdl[1 + cur]
        dev = self.flat_param.device
        V = ctypes.c_void_p
        pp = (V * self.world)(*[int(x) for x in hp.buffer_ptrs])
        gp = (V * self.world)(*[int(x) for x in hg.buffer_ptrs])
        lo, n, so = self.slices[r]
        with torch.cuda.device(dev):
            hg.barrier(channel=2 * r)
            rc = lib.c2v_adam_step_sharded_bulk(
                V(self.flat_param.data_ptr()), pp, gp, self.world, V(self.exp_avg.data_ptr() + 4 * so),
                V(self.exp_avg_sq.data_ptr() + 4 * so), lo, n, self.lr, self.betas[0], self.betas[1], self.eps,
                self.weight_decay, self.t, 1.0 / self.world, 0, V(torch.cuda.current_stream(dev).cuda_stream))
            _lib.check(rc, "c2v_adam_step_sharded_bulk")
            hp.barrier(channel=2 * r + 1)

    def _fused_region(self, r, cur, nxt, zero_all=False):
        """barrier -> c2v_adam_step_sharded on this rank's slice of region r -> barrier, on the current stream"""
        import ctypes
        from . import _lib
        lib = _lib.load()
        hp, hg = self._hdl[0], self._hdl[1 + cur]
        dev = self.flat_param.device
        V = ctypes.c_void_p
        use_mc = self.transport == "nvls"
        pp = (V * self.world)(*[int(x) for x in hp.buffer_ptrs])
        gp = (V * self.world)(*[int(x) for x in hg.buffer_ptrs])
        lo, n, so = self.slices[r]
        rb, rn = (0, self.padded) if zero_all else self.regions[r]     # which part of the OTHER bucket this launch zero-fills
        with torch.cuda.device(dev):
            hg.barrier(channel=2 * r)                        # every rank's backward has finished writing this region
            rc = lib.c2v_adam_step_sharded(
                V(self.flat_param.data_ptr()), V(int(hp.multicast_ptr)) if use_mc else None,
                V(int(hg.multicast_ptr)) if use_mc else None, pp, gp, self.world, V(self.exp_avg.data_ptr() + 4 * so),
                V(self.exp_avg_sq.data_ptr() + 4 * so), lo, n, V(self.buckets[nxt].data_ptr() + 4 * rb), rn, self.lr,
                self.betas[0], self.betas[1], self.eps, self.weight_decay, self.t, 1.0 / self.world,
                V(torch.cuda.current_stream(dev).cuda_stream))
            _lib.check(rc, "c2v_adam_step_sharded")
            hp.barrier(channel=2 * r + 1)                    # every rank's parameter stores of this region have landed here

    def early_step(self):
        """Called from inside the backward once the early parameters' gradients are complete (Code2Vec.on_path_grads_ready):
        reduce + Adam + broadcast of region 0 on a side stream, overlapping the rest of the backward."""
        if self.world == 1 or self.transport == "nccl" or len(self.regions) < 2 or self._early_done:
            return
        dev = self.flat_param.device
        self.t += 1
        self._side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(self._side):
            self._bulk_region(0, self.cur)
        self._early_done = True

    def step(self):
        """reduce this step's gradients over the ranks (mean), Adam, parameters identical everywhere afterwards; the
        other bucket is left zeroed and becomes the target of the next backward (main.py:171 + :175)."""
        cur, nxt = self.cur, 1 - self.cur
        if not self._early_done:
            self.t += 1
        if self.world == 1:                                      # one launch, gradient zeroed in the same pass, no swap
            self._adam_slice(self.flat_param, self.buckets[cur], zero_grad=True)
            for p in self.params:
                torch.autograd.graph.increment_version(p)
            return
        if self.transport == "nccl":
            dev = self.flat_param.device
            for r, (rb, rn) in enumerate(self.regions):
                lo, n, so = self.slices[r]
                g_slice = torch.empty(n, dtype=torch.float32, device=dev)
                self._reduce_scatter(g_slice, self.buckets[cur][rb:rb + rn])
                self._adam_slice(self.flat_param[lo:lo + n], g_slice, state=(self.exp_avg[so:so + n], self.exp_avg_sq[so:so + n]))
                dist.all_gather_into_tensor(self.flat_param[rb:rb + rn], self.flat_param[lo:lo + n].clone(), group=self.group)
            self.buckets[nxt].zero_()
        else:
            first = 1 if self._early_done else 0
            for r in range(first, len(self.regions)):
                self._fused_region(r, cur, nxt, zero_all=self._early_done)   # (the bulk kernel of region 0 does not zero-fill)
            if self._early_done:
                torch.cuda.current_stream(self.flat_param.device).wait_stream(self._side)
        self._early_done = False
        self._point_grads(nxt)
        for p in self.params:                                    # raw-pointer writes: bump the version counters
            torch.autograd.graph.increment_version(p)


def ddp_step(model, optimizer, bucket, starts, paths, ends, label, loss_fn):
    """One training step of main.py:171-175 on this rank's shard of the global batch."""
    if isinstance(optimizer, (ShardedFlatAdam, FlatAdam)) and hasattr(model, "fuse_grad_accumulation"):
        model.fuse_grad_accumulation = True                  # .grad are persistent views into a flat bucket: accumulate in place
        if isinstance(optimizer, ShardedFlatAdam) and len(optimizer.regions) > 1 and optimizer.world > 1 and \
                optimizer.transport != "nccl":
            model.on_path_grads_ready = optimizer.early_step # region 0 is reduced while the backward is still running
    if isinstance(optimizer, ShardedFlatAdam):               # reduction + optimizer + broadcast are one kernel per rank
        if loss_fn is None:                                  # fused loss: the [b, C] logits are never written
            loss = model.forward_loss(starts, paths, ends, label)[0]
        else:
            outputs, code_vector, attention = model.forward(starts, paths, ends, label)
            loss = loss_fn(outputs, label)
        loss.backward()
        optimizer.step()
        return loss
    fused = isinstance(optimizer, FlatAdam)
    if not fused:
        bucket.zero()                       # (FlatAdam leaves the bucket zeroed at the end of its step)
    outputs, code_vector, attention = model.forward(starts, paths, ends, label)
    loss = loss_fn(outputs, label)
    loss.backward()
    if fused:
        bucket.allreduce(average=False)     # plain sum; the 1/world is folded into the optimizer's gradient read
        world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        optimizer.step(grad_scale=1.0 / world)
    else:
        bucket.allreduce()
        optimizer.step()
    return loss


def broadcast_parameters(model, src=0):
    """Same initial weights everywhere (the reference seeds one process; here rank `src` wins)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        for t in list(model.parameters()) + list(model.buffers()):
            dist.broadcast(t.data, src)
            # a write through .data does not bump Tensor._version, which the model's cached weight images
            # (functional.PrepCache) are keyed on: bump it so the next forward rebuilds them
            torch.autograd.graph.increment_version(t)


class FusedSparseAdam(torch.optim.SparseAdam):
    """torch.optim.SparseAdam whose step is one kernel per parameter (`c2v_sparse_adam_step`): for the rows of the
    coalesced sparse gradient it reads g, p, exp_avg and exp_avg_sq once and writes p, exp_avg and exp_avg_sq, with torch's
    operation order and rounding, so parameters and state stay bit-identical to torch.optim.SparseAdam's.  Only step() is
    overridden: parameter groups, hyper-parameter checks and state_dict are torch's and interchange with
    torch.optim.SparseAdam in both directions.  For the embedding tables of a Code2Vec whose `.sparse` is set (see
    INTEGRATION.md, "Sparse embedding gradients").  Lazy Adam: rows a batch does not touch keep their moments and do not
    move, unlike the dense torch.optim.Adam of the reference.  Single process only: a data-parallel reduction of sparse
    gradients is not implemented, and without one the replicas would drift apart."""

    @torch.no_grad()
    def step(self, closure=None):
        from . import functional as CF
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            raise NotImplementedError("FusedSparseAdam: sparse gradients are not reduced across processes "
                                      f"(world size {dist.get_world_size()}); use one process or dense gradients")
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            maximize = group.get("maximize", False)
            lr = group["lr"]
            lr = float(lr.item()) if isinstance(lr, torch.Tensor) else float(lr)
            for p in group["params"]:
                if p.grad is None:
                    continue
                grad = p.grad
                if not grad.is_sparse:
                    raise RuntimeError("SparseAdam does not support dense gradients, please consider Adam instead")
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = 0
                    state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["step"] += 1
                if maximize:
                    grad = -grad
                if not grad.is_coalesced():
                    grad = grad.coalesce()
                if grad.sparse_dim() != 1:
                    raise NotImplementedError("FusedSparseAdam: gradients must be sparse in the first dimension only "
                                              "(row-sparse, as nn.Embedding(sparse=True) produces)")
                values = grad._values()
                if values.numel() == 0:                          # torch skips an empty gradient (the step still counts)
                    continue
                CF.sparse_adam_step(p, state["exp_avg"], state["exp_avg_sq"], values, grad._indices()[0], lr, beta1,
                                    beta2, group["eps"], state["step"])
                torch.autograd.graph.increment_version(p)        # raw-pointer writes: bump the version counter
        return loss

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
import warnings

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


# the parameter-group keys of FlatAdam / ShardedFlatAdam; torch.optim.Adam's amsgrad and maximize are accepted as False
_GROUP_KEYS = ("params", "lr", "betas", "eps", "weight_decay", "decoupled_weight_decay", "max_grad_norm", "capturable")
_FALSE_KEYS = ("amsgrad", "maximize")
# settings of the whole optimizer: one global norm for clipping, one place for the step count
_WHOLE_KEYS = ("max_grad_norm", "capturable")


class _FlatAdamBase(torch.optim.Optimizer):
    """What FlatAdam and ShardedFlatAdam share as torch.optim.Optimizers: parameter groups that are the source of truth
    for lr, betas, eps, weight_decay, decoupled_weight_decay (per group) and max_grad_norm (the same in every group: one
    global norm), so that the torch.optim.lr_scheduler classes drive them (a group's `capturable` records the `capturable`
    attribute, which is fixed at construction); state_dict() / load_state_dict() in torch.optim.Adam's format; and the flat
    launch itself.  The groups are fixed at construction: the flat layout is.  One group without decoupled weight decay
    launches the one-group kernels; otherwise the grouped ones (c2v_adam_step_groups), whose segment table maps the flat
    buffers to the groups.  Subclasses provide `_flat_offsets` (parameter in group order -> offset in the flat buffers),
    call `_layout_groups`, and provide `_gather_state()` and `_scatter_state()`."""

    def _init_optimizer(self, params, dev, lr, betas, eps, weight_decay, max_grad_norm, capturable,
                        decoupled_weight_decay=False):
        if max_grad_norm is not None and not float(max_grad_norm) > 0.0:
            raise ValueError(f"max_grad_norm must be None or > 0, got {max_grad_norm}")
        self.capturable = bool(capturable)               # fixed at construction: it decides where the step count lives
        self._dev = dev
        self._building = True
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay,
                                      decoupled_weight_decay=decoupled_weight_decay, max_grad_norm=max_grad_norm,
                                      capturable=capturable))
        self._building = False
        for group in self.param_groups:
            self._check_group(group)
        for k in _WHOLE_KEYS:
            self._whole(k)
        self._ordered = [p for g in self.param_groups for p in g["params"]]     # state_dict()'s numbering
        if len({id(p) for p in self._ordered}) != len(self._ordered):
            raise ValueError(f"{type(self).__name__}: a parameter appears more than once in the parameter groups")
        # {norm, coef} of the last clipped step (c2v_grad_clip_coef) and the per-CTA partials of its norm pass
        self._norm_coef = torch.zeros(2, dtype=torch.float32, device=dev)
        self._norm_ws = torch.empty(1024, dtype=torch.float32, device=dev)

    def _check_group(self, group):
        name = type(self).__name__
        for k in group:
            if k in _FALSE_KEYS:
                if group[k]:
                    raise ValueError(f"{name}: {k}=True is not this optimizer's update rule")
            elif k not in _GROUP_KEYS:
                raise ValueError(f"{name}: unknown parameter-group key {k!r} (the keys are {', '.join(_GROUP_KEYS)})")
        lr = group["lr"]
        if isinstance(lr, torch.Tensor):
            if not self.capturable:
                raise ValueError("a tensor lr is read by the captured step-count kernel: it needs capturable=True")
            if lr.device != self._dev or lr.dtype != torch.float32 or lr.numel() != 1:
                raise ValueError(f"a tensor lr must be a one-element fp32 tensor on {self._dev}, got {lr.dtype} "
                                 f"{tuple(lr.shape)} on {lr.device}")
        else:
            group["lr"] = float(lr)
        mgn = group["max_grad_norm"]
        if mgn is not None and not float(mgn) > 0.0:
            raise ValueError(f"max_grad_norm must be None or > 0, got {mgn}")
        group.update(betas=(float(group["betas"][0]), float(group["betas"][1])), eps=float(group["eps"]),
                     weight_decay=float(group["weight_decay"]),
                     decoupled_weight_decay=bool(group["decoupled_weight_decay"]),
                     max_grad_norm=None if mgn is None else float(mgn), capturable=bool(group["capturable"]))
        if group["capturable"] != self.capturable:
            raise ValueError(f"{name}: capturable is a setting of the whole optimizer, a group has "
                             f"capturable={group['capturable']}")

    def _whole(self, key):
        """the value of a setting of the whole optimizer; ValueError when the groups disagree"""
        values = [g[key] for g in self.param_groups]
        if any(v != values[0] for v in values):
            raise ValueError(f"{type(self).__name__}: {key} is a setting of the whole optimizer (clipping uses one "
                             f"global norm, the step count is shared), but the parameter groups have {values}")
        return values[0]

    def _layout_groups(self, flat_params, offsets):
        """the segment table: maximal runs of one group over `flat_params` (flat order, at `offsets`), as
        [(first flat element, group)], the first at 0"""
        gid = {id(p): k for k, g in enumerate(self.param_groups) for p in g["params"]}
        segs = []
        for p, o in zip(flat_params, offsets):
            if p.numel() and (not segs or segs[-1][1] != gid[id(p)]):
                segs.append((o, gid[id(p)]))
        segs = [(0, segs[0][1] if segs else 0)] + segs[1:]
        from . import _lib
        if len(self.param_groups) > _lib.ADAM_MAX_GROUPS or len(segs) > _lib.ADAM_MAX_SEGMENTS:
            raise ValueError(f"{type(self).__name__}: {len(self.param_groups)} parameter groups in {len(segs)} runs of "
                             f"the flat buffers; the grouped kernels take up to {_lib.ADAM_MAX_GROUPS} groups and "
                             f"{_lib.ADAM_MAX_SEGMENTS} runs")
        self._segments = segs

    def _patch_step_function(self):
        # torch wraps the class's step() with the step hooks when the first instance is built; wrap this instance's
        # instead, so that the class keeps the plain function whether or not an instance exists
        self._zero_grad_profile_name = f"Optimizer.zero_grad#{type(self).__name__}.zero_grad"
        self.step = torch.optim.Optimizer.profile_hook_step(type(self).step).__get__(self)

    def add_param_group(self, param_group):
        if not self._building:
            if len(self.param_groups) == 1:
                raise ValueError(f"{type(self).__name__} has one parameter group: one flat launch has one set of "
                                 "hyper-parameters")
            raise ValueError(f"{type(self).__name__}: the parameter groups are fixed at construction, where the flat "
                             "buffers are laid out")
        super().add_param_group(param_group)

    def _group_value(name):
        def one(self):
            if len(self.param_groups) > 1:
                raise AttributeError(f"{type(self).__name__} has {len(self.param_groups)} parameter groups: "
                                     f"use param_groups[k][{name!r}]")
            return self.param_groups[0]

        def get(self):
            return one(self)[name]

        def put(self, value):
            g = one(self)
            if name == "lr" and isinstance(g["lr"], torch.Tensor):
                g["lr"].fill_(float(value))              # a captured graph reads this address
            else:
                g[name] = value
        return property(get, put)

    lr, betas, eps, weight_decay = _group_value("lr"), _group_value("betas"), _group_value("eps"), _group_value("weight_decay")
    del _group_value

    @property
    def max_grad_norm(self):
        return self._whole("max_grad_norm")

    @max_grad_norm.setter
    def max_grad_norm(self, value):
        for g in self.param_groups:
            g["max_grad_norm"] = value

    def _grouped(self):
        """whether the step takes the grouped kernels: more than one group, or decoupled weight decay"""
        return len(self.param_groups) > 1 or self.param_groups[0]["decoupled_weight_decay"]

    def step_count(self):
        """the number of steps taken (synchronises in capturable mode)"""
        return int(self.step_state[0]) if self.capturable else self.t

    @property
    def grad_norm(self):
        """one-element fp32 device tensor: the global L2 norm of the last step's gradient (after grad_scale, before
        the clip: what clip_grad_norm_ returns); written only by steps with max_grad_norm set.  No synchronise."""
        return self._norm_coef[:1]

    def _group_table(self, lo=0, n=None):
        """the groups (c2v_adam_group[]) and the segments that meet flat elements [lo, lo + n), rebased to lo:
        (groups, n_groups, seg_begin, seg_group, n_segments) for the *_groups entry points"""
        import ctypes
        from . import _lib
        groups = (_lib.AdamGroup * len(self.param_groups))()
        for a, g in zip(groups, self.param_groups):
            lr = g["lr"]
            a.lr, a.lr_dev = (0.0, lr.data_ptr()) if isinstance(lr, torch.Tensor) else (float(lr), None)
            a.beta1, a.beta2 = g["betas"]
            a.eps, a.weight_decay, a.decoupled = g["eps"], g["weight_decay"], 1 if g["decoupled_weight_decay"] else 0
        segs = self._segments
        if lo:
            hi = lo + n
            segs = [(max(b - lo, 0), k) for i, (b, k) in enumerate(segs)
                    if b < hi and (i + 1 == len(segs) or segs[i + 1][0] > lo)]
        begin = (ctypes.c_int64 * len(segs))(*[b for b, _ in segs])
        group = (ctypes.c_int32 * len(segs))(*[k for _, k in segs])
        return groups, len(groups), begin, group, len(segs)

    def _launch(self, p, g, m, v, step, grad_scale, zero_grad, lo=0):
        """c2v_adam_step_ex on flat fp32 buffers with the group's hyper-parameters, behind c2v_grad_clip_coef on the same
        gradient when max_grad_norm is set.  With max_grad_norm None and a float lr it is c2v_adam_step /
        c2v_adam_step_capturable: same kernels, same launch parameters.  With parameter groups (or decoupled weight
        decay) c2v_adam_step_groups; p begins at flat element `lo`."""
        import ctypes
        from . import _lib
        lib = _lib.load()
        P = lambda t: ctypes.c_void_p(t.data_ptr())
        max_norm = self.max_grad_norm
        dev = p.device
        with torch.cuda.device(dev):
            stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            coef_dev = None
            if max_norm is not None:
                rc = lib.c2v_grad_clip_coef(P(g), g.numel(), float(grad_scale), float(max_norm), P(self._norm_coef),
                                            P(self._norm_ws), 4 * self._norm_ws.numel(), stream)
                _lib.check(rc, "c2v_grad_clip_coef")
                coef_dev = ctypes.c_void_p(self._norm_coef.data_ptr() + 4)
            state = P(self.step_state) if self.capturable else None
            if self._grouped():
                rc = lib.c2v_adam_step_groups(P(p), P(g), P(m), P(v), p.numel(), *self._group_table(lo, p.numel()), step,
                                              state, float(grad_scale), 1 if zero_grad else 0, coef_dev, stream)
                _lib.check(rc, "c2v_adam_step_groups")
                return
            group = self.param_groups[0]
            lr, (beta1, beta2) = group["lr"], group["betas"]
            lr_dev = P(lr) if isinstance(lr, torch.Tensor) else None
            rc = lib.c2v_adam_step_ex(P(p), P(g), P(m), P(v), p.numel(), 0.0 if lr_dev else float(lr), beta1, beta2,
                                      group["eps"], group["weight_decay"], step, state, float(grad_scale),
                                      1 if zero_grad else 0, lr_dev, coef_dev, stream)
        _lib.check(rc, "c2v_adam_step_ex")

    # ---- checkpoints ---------------------------------------------------------------------------------------------------
    def state_dict(self):
        """torch.optim.Adam's (or, with decoupled_weight_decay, torch.optim.AdamW's) state_dict for the same parameter
        groups: state[i] = {"step", "exp_avg", "exp_avg_sq"} for the parameters numbered across the groups in order
        (copies shaped like parameter i; step a tensor as in torch: on the device and without a host read when
        capturable, a CPU fp32 scalar otherwise) and one dict per group with integer `params`, plus the key
        max_grad_norm.  torch.optim.Adam / AdamW load it and continue.  ShardedFlatAdam at world size > 1: a collective,
        every rank returns the full dict."""
        exp_avg, exp_avg_sq = self._gather_state()
        if self.capturable:
            step = self.step_state[0].to(torch.float32)
        else:
            step = torch.tensor(float(self.t), dtype=torch.float32)
        state = {}
        for i, (p, o) in enumerate(zip(self._ordered, self._flat_offsets)):
            n = p.numel()
            state[i] = {"step": step.clone(), "exp_avg": exp_avg[o:o + n].view_as(p).clone(),
                        "exp_avg_sq": exp_avg_sq[o:o + n].view_as(p).clone()}
        groups, i = [], 0
        for g in self.param_groups:
            group = {k: (v.clone() if isinstance(v, torch.Tensor) else v) for k, v in g.items() if k != "params"}
            group["params"] = list(range(i, i + len(g["params"])))
            i += len(g["params"])
            groups.append(group)
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, state_dict):
        """Loads state_dict()'s output, torch.optim.Adam's or torch.optim.AdamW's for the same parameter groups (the
        same count, with the same number of parameters each).  Each group's hyper-parameters are taken over (a tensor
        lr is filled in place, capturable stays as constructed, decoupled_weight_decay defaults to False and
        max_grad_norm to None), the moments are copied into the flat buffers (at world size > 1: this rank's slices of
        them) and the step count is set.  Parameters without state load as zeros and step 0; per-parameter steps that
        differ raise ValueError: the flat kernel has one step count."""
        saved_groups, mine = state_dict["param_groups"], self.param_groups
        if len(saved_groups) != len(mine) or any(len(s["params"]) != len(g["params"])
                                                 for s, g in zip(saved_groups, mine)):
            want = (f"one parameter group of {len(mine[0]['params'])} parameters" if len(mine) == 1 else
                    f"{len(mine)} parameter groups of {[len(g['params']) for g in mine]} parameters")
            raise ValueError(f"{type(self).__name__}.load_state_dict: expected {want}, got "
                             f"{[len(g['params']) for g in saved_groups]}")
        for saved in saved_groups:
            for k in _FALSE_KEYS:
                if saved.get(k):
                    raise ValueError(f"{type(self).__name__}.load_state_dict: {k}=True is not this optimizer's update "
                                     "rule")
        state, steps = state_dict["state"], set()
        exp_avg, exp_avg_sq = (torch.zeros(self._flat_numel, dtype=torch.float32, device=self._norm_coef.device)
                               for _ in range(2))
        keys = [key for saved in saved_groups for key in saved["params"]]
        for i, (p, o, key) in enumerate(zip(self._ordered, self._flat_offsets, keys)):
            st = state.get(key)
            if not st:
                steps.add(0)
                continue
            if tuple(st["exp_avg"].shape) != tuple(p.shape) or tuple(st["exp_avg_sq"].shape) != tuple(p.shape):
                raise ValueError(f"{type(self).__name__}.load_state_dict: state {i} has shape "
                                 f"{tuple(st['exp_avg'].shape)}, the parameter {tuple(p.shape)}")
            n = p.numel()
            exp_avg[o:o + n].copy_(st["exp_avg"].reshape(-1))
            exp_avg_sq[o:o + n].copy_(st["exp_avg_sq"].reshape(-1))
            steps.add(int(st["step"]))
        if len(steps) != 1:
            raise ValueError(f"{type(self).__name__}.load_state_dict: the parameters have different step counts "
                             f"{sorted(steps)}; the flat kernel has one")
        for group, saved in zip(mine, saved_groups):
            for k, v in saved.items():
                if k in ("params", "capturable", "foreach", "differentiable", "fused") + _FALSE_KEYS:
                    continue                             # ours, or torch.optim.Adam's switches
                if k == "lr":
                    if isinstance(group["lr"], torch.Tensor):
                        group["lr"].fill_(float(v))
                    else:
                        group["lr"] = float(v)
                elif k == "betas":
                    group[k] = (float(v[0]), float(v[1]))
                else:
                    group[k] = v.clone() if isinstance(v, torch.Tensor) else v
            group["decoupled_weight_decay"] = bool(saved.get("decoupled_weight_decay", False))
            group["max_grad_norm"] = saved.get("max_grad_norm")
        self._whole("max_grad_norm")
        self._scatter_state(exp_avg, exp_avg_sq)
        if self.capturable:
            self.step_state[0] = steps.pop()
        else:
            self.t = steps.pop()


class FlatAdam(_FlatAdamBase):
    """torch.optim.Adam(model.parameters(), lr, betas, weight_decay) (main.py:138) as ONE kernel launch per step
    (`c2v_adam_step`): parameters, like the gradients of `bucket`, become views into one flat buffer; the step reads
    p, g, m, v once, writes p, m, v and leaves the gradient zeroed for the next backward (main.py:171), folding the
    1/world of the data-parallel mean into the read.  Dense, same update rule and operation order as torch's Adam.

    A torch.optim.Optimizer: the torch.optim.lr_scheduler classes drive `lr` (and OneCycleLR `betas[0]`), and
    state_dict() / load_state_dict() interchange with torch.optim.Adam's and torch.optim.AdamW's.

    groups: None (one group of bucket.params) or torch's parameter-group dicts {"params": [...], "lr", "betas", "eps",
    "weight_decay", "decoupled_weight_decay", "max_grad_norm"}, a missing key taking the constructor's value.  Their
    parameters must be bucket.params, each once, in any grouping (the flat layout stays bucket.params' order, so groups
    may interleave).  lr (a float, or a tensor with capturable=True), betas, eps, weight_decay and
    decoupled_weight_decay are per group; max_grad_norm and capturable are for the whole optimizer.  All groups share
    one step count, each group's bias corrections use its betas.  decoupled_weight_decay=True is torch.optim.AdamW's
    rule: p *= 1 - lr * weight_decay before the moments.  Still one launch per step (c2v_adam_step_groups).

    capturable=True (torch.optim.Adam's flag): the step count lives on the device (`step_state`, see
    c2v_adam_step_capturable) and every step, eager or inside a CUDA graph, runs the capturable kernels; `t` is then not
    kept (read `step_count()`).  With capturable=False a step cannot be captured.  With capturable=True `lr` may be a
    one-element fp32 device tensor, torch's convention: the step reads it on the device, so the replays of a captured
    step follow a scheduler (which fills the tensor in place).  betas stay launch parameters, fixed at capture.

    max_grad_norm: clip the gradient by its global L2 norm inside the step, as
    torch.nn.utils.clip_grad_norm_(params, max_grad_norm) between the backward and the step would: the norm of
    g * grad_scale over the whole bucket (after `bucket.allreduce` at world size > 1 every rank computes the same one),
    coef = min(1, max_grad_norm / (norm + 1e-6)), Adam reads g * (grad_scale * coef), weight decay is added after the
    clip.  One extra read of the bucket; no host read, so it is capturable.  A NaN or inf gradient gives NaN parameters,
    as in torch.  `grad_norm` holds the last norm."""

    def __init__(self, bucket, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, capturable=False,
                 max_grad_norm=None, decoupled_weight_decay=False, groups=None):
        self.bucket = bucket
        self._init_optimizer(bucket.params if groups is None else groups, bucket.flat.device, lr, betas, eps, weight_decay,
                             max_grad_norm, capturable, decoupled_weight_decay)
        if {id(p) for p in self._ordered} != {id(p) for p in bucket.params} or len(self._ordered) != len(bucket.params):
            raise ValueError("FlatAdam: the parameter groups must hold exactly the bucket's parameters, each once")
        flat = torch.empty_like(bucket.flat)
        o, offsets = 0, []
        for p in bucket.params:                                  # same order as the gradient bucket
            n = p.numel()
            flat[o:o + n].copy_(p.data.reshape(-1))
            p.data = flat[o:o + n].view_as(p)
            offsets.append(o)
            o += n
        self._layout_groups(bucket.params, offsets)
        at = {id(p): o for p, o in zip(bucket.params, offsets)}
        self._flat_offsets = [at[id(p)] for p in self._ordered]
        self._flat_numel = o
        self.flat_param = flat
        self.exp_avg = torch.zeros_like(flat)
        self.exp_avg_sq = torch.zeros_like(flat)
        self.t = 0
        self.step_state = _step_state(flat.device, len(self.param_groups)) if self.capturable else None

    def step(self, grad_scale=1.0, zero_grad=True):
        _check_capturable(self.capturable, "FlatAdam")
        if not self.capturable:
            self.t += 1
        self._launch(self.flat_param, self.bucket.flat, self.exp_avg, self.exp_avg_sq, self.t, grad_scale, zero_grad)
        # the kernel wrote through raw pointers: tell autograd (and the weight-image caches of the model, which key on
        # Tensor._version) that every parameter changed, as an in-place torch op would
        for p in self.bucket.params:
            torch.autograd.graph.increment_version(p)

    def zero_grad(self, set_to_none=False):
        """zeroes the bucket; `.grad` stays a view of it whatever set_to_none says"""
        self.bucket.zero()

    def _gather_state(self):
        return self.exp_avg, self.exp_avg_sq

    def _scatter_state(self, exp_avg, exp_avg_sq):
        self.exp_avg.copy_(exp_avg)
        self.exp_avg_sq.copy_(exp_avg_sq)


def _step_state(device, n_groups):
    """the device step-state, step 0: {int64 step; float s[3 * n_groups]} (c2v_adam_step_groups), which begins with the
    one of c2v_adam_step_capturable, {int64 step; float step_size; float inv_sqrt_bc2}"""
    return torch.zeros(1 + (3 * n_groups + 1) // 2, dtype=torch.int64, device=device)


def _check_capturable(capturable, name):
    from .functional import capturing
    if capturing() and not capturable:
        raise RuntimeError(f"{name}.step() is being captured into a CUDA graph, but the optimizer keeps its step count on "
                           f"the host, so every replay would repeat the captured step: construct it with capturable=True")


def sharded_layout(n_early, numel, world, rank):
    """The flat-buffer layout of ShardedFlatAdam for `numel` parameters of which the first `n_early` form the early
    region (0: no early region).  -> (regions, slices, state_numel):
      regions      [(begin, length)] in the flat buffers, each length padded to a multiple of 4 * world
      slices       [(begin, length, state_offset)] of this rank per region: the owned part of the flat buffers and where
                   its exp_avg / exp_avg_sq sit in the rank's state buffers
      state_numel  elements of the rank's exp_avg (and of its exp_avg_sq)"""
    q = 4 * world
    pad = lambda n: (n + q - 1) // q * q
    regions = ([(0, pad(n_early))] if n_early else []) + [(pad(n_early) if n_early else 0, pad(numel - n_early))]
    slices, o = [], 0
    for begin, n in regions:
        sl = n // world
        slices.append((begin + rank * sl, sl, o))
        o += sl
    return regions, slices, o


def nvls_allowed(transport, world):
    """Whether ShardedFlatAdam's transport="auto" may pick "nvls" for a group of `world` ranks.  Under
    torch.use_deterministic_algorithms(True) at world size > 1 it may not: the in-switch reduction (multimem.ld_reduce)
    has no documented summation order.  An explicit "nvls" then raises RuntimeError, or warns (UserWarning) with
    warn_only=True and stays.  "p2p" sums the ranks in a fixed order and "nccl" is left to NCCL: both are unchanged."""
    if world <= 1 or not torch.are_deterministic_algorithms_enabled():
        return True
    if transport == "nvls":
        msg = ('ShardedFlatAdam: transport "nvls" reduces the gradients in the NVSwitch in no documented order, so it is '
               'not deterministic; torch.use_deterministic_algorithms(True) is set: use transport="p2p" (or "auto")')
        if not torch.is_deterministic_algorithms_warn_only_enabled():
            raise RuntimeError(msg)
        warnings.warn(msg, UserWarning)
    return False


class ShardedFlatAdam(_FlatAdamBase):
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

    A torch.optim.Optimizer like FlatAdam: parameter groups (`params` in torch's forms: parameters or group dicts, a
    missing key taking the constructor's value), lr schedulers, and state_dict() / load_state_dict() in
    torch.optim.Adam's / AdamW's format.  The flat order is the groups' parameters in order, the early ones first; with
    more than one group every parameter starts at a multiple of 4 elements.  At world size > 1 state_dict() is a collective (it all-gathers the
    owned slices) that returns the full dict on every rank, and load_state_dict() keeps this rank's slices of the full
    dict: a checkpoint saved at one world size loads at another.  At world size 1 a tensor `lr` (capturable=True) and
    `max_grad_norm` work as in FlatAdam.  max_grad_norm at world size > 1 raises NotImplementedError: the fused kernel
    reduces the gradient and applies Adam in one pass, so the norm of the reduced gradient does not exist before the
    update; clipping there would be a two-phase kernel.
    """

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, group=None, transport="auto",
                 early=(), capturable=False, max_grad_norm=None, decoupled_weight_decay=False):
        params = list(params)
        if params and isinstance(params[0], dict):               # parameter groups: their trainable parameters
            groups = [dict(g, params=[p for p in ([g["params"]] if isinstance(g["params"], torch.Tensor) else g["params"])
                                      if p.requires_grad]) for g in params]
            params = [p for g in groups for p in g["params"]]
        else:
            params = groups = [p for p in params if p.requires_grad]
        if not params:
            raise ValueError("no trainable parameters")
        early_ids = {id(p) for p in early}
        first = [p for p in params if id(p) in early_ids]
        self.params = first + [p for p in params if id(p) not in early_ids]      # flat order: early region first
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if self.world > 1 else 0
        if capturable and self.world > 1:
            raise NotImplementedError("ShardedFlatAdam(capturable=True) supports one process only: the data-parallel step "
                                      f"uses cross-GPU barriers and a side stream (world size {self.world})")
        if max_grad_norm is not None and self.world > 1:
            raise NotImplementedError("ShardedFlatAdam(max_grad_norm=...) supports one process only: the data-parallel "
                                      "step reduces the gradient and applies Adam in one pass, so the norm of the reduced "
                                      f"gradient does not exist before the update (world size {self.world})")
        dev, dt = self.params[0].device, self.params[0].dtype
        if dt != torch.float32:
            raise TypeError("parameters must be fp32")
        self._init_optimizer(groups, dev, lr, betas, eps, weight_decay, max_grad_norm, capturable, decoupled_weight_decay)
        self.numel = sum(p.numel() for p in self.params)
        # with several groups the flat order is the groups', and a parameter whose size is not a multiple of 4 (the
        # output bias at C = 195,299) may come before an embedding table, which the model's kernels read 16 bytes at a
        # time: there every parameter starts at a multiple of 4 elements (the gaps are zero and stay zero)
        span = (lambda p: (p.numel() + 3) // 4 * 4) if len(self.param_groups) > 1 else (lambda p: p.numel())
        n_early = sum(span(p) for p in first)
        # regions: (begin, length) in the flat buffers; region 0 = the early parameters (absent when there are none);
        # this rank's slice of every region, and where its optimizer state sits in exp_avg / exp_avg_sq
        self.regions, self.slices, self.state_numel = sharded_layout(n_early, sum(span(p) for p in self.params),
                                                                     self.world, self.rank)
        self.padded = sum(n for _, n in self.regions)
        self._auto = transport == "auto"
        self._auto_nvls = nvls_allowed(transport, self.world)
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
            o += span(p)
        flat_pos = {id(p): pos[i] for i, p in enumerate(self.params)}
        self._flat_offsets = [flat_pos[id(p)] for p in self._ordered]      # in the caller's order, which state_dict() keeps
        self._layout_groups(self.params, [pos[i] for i in range(len(self.params))])
        self._flat_numel = self.padded
        for i, p in enumerate(self.params):
            n, o = p.numel(), pos[i]
            self.flat_param[o:o + n].copy_(p.data.reshape(-1))
            p.data = self.flat_param[o:o + n].view_as(p)
            for k in (0, 1):
                self._grad_views[k].append(self.buckets[k][o:o + n].view_as(p))
        self.exp_avg = torch.zeros(self.state_numel, dtype=dt, device=dev)
        self.exp_avg_sq = torch.zeros(self.state_numel, dtype=dt, device=dev)
        self.t, self.cur = 0, 0
        self.step_state = _step_state(dev, len(self.param_groups)) if self.capturable else None
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
        saved = [(g["lr"], g["weight_decay"]) for g in self.param_groups]
        for g in self.param_groups:
            g["lr"], g["weight_decay"] = 0.0, 0.0
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
            for g, (lr, wd) in zip(self.param_groups, saved):
                g["lr"], g["weight_decay"] = lr, wd
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
                return ("nvls" if (mc and (want == "nvls" or (want == "auto" and self._auto_nvls))) else "p2p"), hdls
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

    def zero_grad(self, set_to_none=False):
        """zeroes the current bucket; `.grad` stays a view of it whatever set_to_none says"""
        self.buckets[self.cur].zero_()

    def _gather_state(self):
        """the full flat exp_avg / exp_avg_sq [padded]: at world size > 1 every region's slices, all-gathered"""
        if self.world == 1:
            return self.exp_avg, self.exp_avg_sq
        full = []
        for own in (self.exp_avg, self.exp_avg_sq):
            out = torch.empty(self.padded, dtype=own.dtype, device=own.device)
            for (rb, rn), (lo, n, so) in zip(self.regions, self.slices):
                dist.all_gather_into_tensor(out[rb:rb + rn], own[so:so + n].clone(), group=self.group)
            full.append(out)
        return full

    def _scatter_state(self, exp_avg, exp_avg_sq):
        for lo, n, so in self.slices:
            self.exp_avg[so:so + n].copy_(exp_avg[lo:lo + n])
            self.exp_avg_sq[so:so + n].copy_(exp_avg_sq[lo:lo + n])

    # ---- the step -----------------------------------------------------------------------------------------------------
    def _adam_slice(self, p_slice, g_slice, zero_grad=False, state=None):
        """the flat step on an owned slice (the gloo CPU tests replace this method with a torch stand-in)"""
        m, v = state if state is not None else (self.exp_avg, self.exp_avg_sq)
        lo = (p_slice.data_ptr() - self.flat_param.data_ptr()) // p_slice.element_size()   # where the slice begins
        self._launch(p_slice, g_slice, m, v, self.t, 1.0 / self.world, zero_grad, lo=lo)

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
            stream = V(torch.cuda.current_stream(dev).cuda_stream)
            if self._grouped():
                rc = lib.c2v_adam_step_sharded_bulk_groups(
                    V(self.flat_param.data_ptr()), pp, gp, self.world, V(self.exp_avg.data_ptr() + 4 * so),
                    V(self.exp_avg_sq.data_ptr() + 4 * so), lo, n, *self._group_table(), self.t, 1.0 / self.world, 0,
                    stream)
            else:
                rc = lib.c2v_adam_step_sharded_bulk(
                    V(self.flat_param.data_ptr()), pp, gp, self.world, V(self.exp_avg.data_ptr() + 4 * so),
                    V(self.exp_avg_sq.data_ptr() + 4 * so), lo, n, self.lr, self.betas[0], self.betas[1], self.eps,
                    self.weight_decay, self.t, 1.0 / self.world, 0, stream)
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
            head = (V(self.flat_param.data_ptr()), V(int(hp.multicast_ptr)) if use_mc else None,
                    V(int(hg.multicast_ptr)) if use_mc else None, pp, gp, self.world, V(self.exp_avg.data_ptr() + 4 * so),
                    V(self.exp_avg_sq.data_ptr() + 4 * so), lo, n, V(self.buckets[nxt].data_ptr() + 4 * rb), rn)
            stream = V(torch.cuda.current_stream(dev).cuda_stream)
            if self._grouped():
                rc = lib.c2v_adam_step_sharded_groups(*head, *self._group_table(), self.t, 1.0 / self.world, stream)
            else:
                rc = lib.c2v_adam_step_sharded(*head, self.lr, self.betas[0], self.betas[1], self.eps, self.weight_decay,
                                               self.t, 1.0 / self.world, stream)
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
        _check_capturable(self.capturable, "ShardedFlatAdam")
        if self.transport == "nvls":             # the switch may have been turned on after the construction chose "nvls"
            nvls_allowed("nvls", self.world)
        if self.world > 1 and self.max_grad_norm is not None:
            raise NotImplementedError("ShardedFlatAdam: max_grad_norm supports one process only")
        cur, nxt = self.cur, 1 - self.cur
        if not self._early_done and not self.capturable:
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


def _forward_loss(model, starts, paths, ends, label, criterion, sampler=None):
    # criterion None: the call without it, for any forward_loss of the (starts, paths, ends, label) form
    if sampler is not None:
        return model.forward_sampled_loss(starts, paths, ends, label, sampler)[0]
    if criterion is None:
        return model.forward_loss(starts, paths, ends, label)[0]
    return model.forward_loss(starts, paths, ends, label, criterion=criterion)[0]


def ddp_step(model, optimizer, bucket, starts, paths, ends, label, loss_fn, criterion=None, sampler=None):
    """One training step of main.py:171-175 on this rank's shard of the global batch.  loss_fn None: the fused loss of
    Code2Vec.forward_loss with `criterion` (None, nn.NLLLoss or nn.CrossEntropyLoss; a mean is this rank's own, as with
    DDP); else forward() and loss_fn(outputs, label).  sampler (a functional.SampledSoftmax): the step's loss is
    Code2Vec.forward_sampled_loss(...)[0] instead, its candidates drawn from this rank's own generator; it takes neither
    loss_fn nor criterion (ValueError)."""
    if sampler is not None and (loss_fn is not None or criterion is not None):
        raise ValueError("ddp_step: sampler= replaces the loss; pass loss_fn=None and no criterion with it")
    if isinstance(optimizer, (ShardedFlatAdam, FlatAdam)) and hasattr(model, "fuse_grad_accumulation"):
        model.fuse_grad_accumulation = True                  # .grad are persistent views into a flat bucket: accumulate in place
        if isinstance(optimizer, ShardedFlatAdam) and len(optimizer.regions) > 1 and optimizer.world > 1 and \
                optimizer.transport != "nccl":
            model.on_path_grads_ready = optimizer.early_step # region 0 is reduced while the backward is still running
    if isinstance(optimizer, ShardedFlatAdam):               # reduction + optimizer + broadcast are one kernel per rank
        if loss_fn is None:                                  # fused loss: the [b, C] logits are never written
            loss = _forward_loss(model, starts, paths, ends, label, criterion, sampler)
        else:
            outputs, code_vector, attention = model.forward(starts, paths, ends, label)
            loss = loss_fn(outputs, label)
        loss.backward()
        optimizer.step()
        return loss
    fused = isinstance(optimizer, FlatAdam)
    if not fused:
        bucket.zero()                       # (FlatAdam leaves the bucket zeroed at the end of its step)
    if loss_fn is None:                     # fused loss (Code2Vec.forward_loss)
        loss = _forward_loss(model, starts, paths, ends, label, criterion, sampler)
    else:
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
    move, unlike the dense torch.optim.Adam of the reference.

    Data-parallel training (`group`: the process group, default the world; an attribute, not a group default, so
    state_dict() is unchanged): at world size > 1 step() first reduces each parameter's sparse gradient over the group
    and then takes one SparseAdam step on the result, the same on every rank, so parameters and state stay replicated
    bit for bit.  The reduced gradient holds the union of the ranks' rows, ascending, each the fp32 sum of the ranks that
    touched it, in rank order, times the fp32 1/W (the mean, as for the dense parameters).  A parameter whose gradient is
    None on every rank is skipped; one with a gradient on some ranks is stepped on all, a None gradient counting as an
    empty one.  One all-gather of every parameter's row count (read on the host, to size the buffers), then per
    parameter an all-gather of its rows and of its values, each padded to the largest count, and
    `c2v_sparse_union_rows` + `c2v_sparse_adam_step_merged`, which merge the lists inside the update."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, maximize=False, group=None):
        super().__init__(params, lr=lr, betas=betas, eps=eps, maximize=maximize)
        self.group = group

    def _world_size(self):
        return dist.get_world_size(self.group) if dist.is_available() and dist.is_initialized() else 1

    def _all_gather(self, t):
        """[W, *t.shape]: every rank's `t` in rank order (the collective of the data-parallel step; the one-GPU tests
        replace this method)"""
        world = self._world_size()
        out = t.new_empty(world * t.numel())
        dist.all_gather_into_tensor(out, t.contiguous().reshape(-1), group=self.group)
        return out.view((world,) + tuple(t.shape))

    def _merged_step(self, p, state, rows, values, counts, lr, beta1, beta2, eps, scale):
        """the union of the gathered row lists and the merged SparseAdam step on it, on the device (the gloo CPU tests
        replace this method with a torch restatement)"""
        from . import functional as CF
        union, count = CF.sparse_union_rows(rows, counts, p.shape[0])
        CF.sparse_adam_step_merged(p, state["exp_avg"], state["exp_avg_sq"], values, rows, counts, union, count, lr,
                                   beta1, beta2, eps, state["step"], scale)

    def _step_data_parallel(self, world):
        entries, local = [], []
        for group in self.param_groups:
            for p in group["params"]:
                grad = p.grad
                if grad is not None:
                    if not grad.is_sparse:
                        raise RuntimeError("SparseAdam does not support dense gradients, please consider Adam instead")
                    if not grad.is_coalesced():
                        grad = grad.coalesce()
                    if grad.sparse_dim() != 1:
                        raise NotImplementedError("FusedSparseAdam: gradients must be sparse in the first dimension "
                                                  "only (row-sparse, as nn.Embedding(sparse=True) produces)")
                entries.append((group, p, grad))
                local.append(-1 if grad is None else grad._nnz())
        if not entries:
            return
        counts = self._all_gather(torch.tensor(local, dtype=torch.int64, device=entries[0][1].device))
        host = counts.cpu()                                  # the step's one host wait: it sizes the exchange buffers
        inv_world = float(torch.tensor(1.0 / world, dtype=torch.float32))
        for i, (group, p, grad) in enumerate(entries):
            col = host[:, i]
            if bool((col < 0).all()):                        # None on every rank: skipped, as torch skips it
                continue
            state = self.state[p]
            if len(state) == 0:
                state["step"] = 0
                state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            state["step"] += 1
            u_max = int(col.max())
            if u_max == 0:                                   # an empty union: the step still counts
                continue
            E = p[0].numel()
            rows = torch.zeros(u_max, dtype=torch.int64, device=p.device)
            values = torch.zeros((u_max, E), dtype=p.dtype, device=p.device)
            n = int(local[i]) if grad is not None else 0
            if n:
                rows[:n] = grad._indices()[0]
                values[:n] = grad._values().reshape(n, E)
            lr = group["lr"]
            lr = float(lr.item()) if isinstance(lr, torch.Tensor) else float(lr)
            beta1, beta2 = group["betas"]
            scale = -inv_world if group.get("maximize", False) else inv_world
            self._merged_step(p, state, self._all_gather(rows), self._all_gather(values), counts[:, i].contiguous(), lr,
                              beta1, beta2, group["eps"], scale)
            torch.autograd.graph.increment_version(p)        # raw-pointer writes: bump the version counter

    @torch.no_grad()
    def step(self, closure=None):
        from . import functional as CF
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        world = self._world_size()
        if world > 1:
            self._step_data_parallel(world)
            return loss
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

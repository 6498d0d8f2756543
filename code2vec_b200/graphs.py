"""CUDA-graph capture of the training step and of prediction.

At small batches (the reference trains at batch 32) the GPU work of a step is small, and the host -- autograd nodes, one
ctypes call per library entry point, the allocations around them -- can set the step time.  A CUDA graph replays the
whole step's kernels with one launch.  These helpers apply torch's capture recipe (warm-up on real batches, capture on
static inputs, copy in and replay) to a Code2Vec step:

    GraphedTrainStep(model, optimizer, batch_size, max_path_length, loss_fn=None, criterion=None)(starts, paths, ends,
                     label) -> loss
    GraphedPredict(model, batch_size, max_path_length, k=None)(starts, paths, ends) -> predict() / predict_topk(k)

What a captured step needs (checked, each with a clear error): dropout keys drawn on the device
(Code2Vec.use_device_rng), an optimizer whose step count lives on the device (FlatAdam / ShardedFlatAdam with
capturable=True at world size 1, or torch.optim.Adam(capturable=True)), dense embedding gradients and padded [B, L]
batches.  Hyper-parameters, model.training and torch's TF32 matmul switch are fixed at capture.  See INTEGRATION.md, "CUDA graphs".
"""
import torch

from .distributed import FlatAdam, ShardedFlatAdam, _forward_loss, ddp_step
from .functional import torch_matmul_tf32

__all__ = ["GraphedTrainStep", "GraphedPredict"]


def _bump_versions(model):
    # a replay writes the parameters through raw pointers without bumping Tensor._version; bump it as an eager step would
    for p in model.parameters():
        torch.autograd.graph.increment_version(p)


class _Graphed:
    """warm-up -> capture -> replay of `self._run(*static inputs)` for inputs of one shape; other shapes run eagerly"""

    WARMUP = 2

    def __init__(self, model, shapes):
        self.model, self.shapes = model, shapes
        self.graph, self.static_in, self.static_out = None, None, None
        self.warmed = 0
        self._frozen = None

    def _settings(self):
        # the matmul precision selects other kernels than the captured ones
        return (self.model.training, torch_matmul_tf32())

    def _call(self, *inputs):
        self.model._enc_cache.raise_deferred()           # an out-of-range index in an earlier replay
        if not all(isinstance(t, torch.Tensor) for t in inputs):
            raise TypeError(f"{type(self).__name__}: takes padded [B, L] batches; PackedBags batches change their context "
                            "count from batch to batch and cannot be captured (call the model directly)")
        if tuple(tuple(t.shape) for t in inputs) != self.shapes:
            return self._run(*inputs)                    # e.g. the ragged last batch of an epoch: eagerly
        if self.graph is not None:
            if self._settings() != self._frozen:
                raise RuntimeError(f"{type(self).__name__}: hyper-parameters, the criterion, model.training, "
                                   "torch.are_deterministic_algorithms_enabled() or the TF32 matmul switch "
                                   "(torch.backends.cuda.matmul.fp32_precision) changed since the capture "
                                   f"({self._frozen} -> {self._settings()}); build a new {type(self).__name__}")
            for s, t in zip(self.static_in, inputs):
                s.copy_(t, non_blocking=True)
            self.graph.replay()
            return self.static_out
        cur = torch.cuda.current_stream()
        if self.warmed < self.WARMUP:                    # warm-up on real batches, on a side stream (torch's recipe)
            self.warmed += 1
            side = torch.cuda.Stream()
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                out = self._run(*inputs)
            cur.wait_stream(side)
            return out
        self.static_in = tuple(t.clone() for t in inputs)
        self._frozen = self._settings()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self.static_out = self._run(*self.static_in)
        self.graph = graph
        graph.replay()
        return self.static_out


class GraphedTrainStep(_Graphed):
    """One training step of main.py:171-175, captured into a CUDA graph.  Calling it with (starts, paths, ends, label)
    runs the step and returns the loss as a fresh device tensor:
      FlatAdam / ShardedFlatAdam (capturable=True): ddp_step (gradients accumulated in the flat bucket);
      any torch optimizer, e.g. torch.optim.Adam(capturable=True): zero_grad(set_to_none=False) + forward + backward +
      step().
    loss_fn None: the fused loss of Code2Vec.forward_loss with `criterion` (None, nn.NLLLoss or nn.CrossEntropyLoss);
    else forward() and loss_fn(outputs, label).  The criterion's type, ignore_index, label_smoothing, reduction and its
    weight tensor (address and shape) are fixed at capture like the hyper-parameters; the replays read the weight's
    values, so an in-place change to them (weight.copy_, weight.mul_) takes effect at the next replay.
    The first two [batch_size, max_path_length] calls run eagerly (warm-up on real batches: no extra optimizer step), the
    third captures and replays, later ones copy into the static inputs and replay.  Other shapes run eagerly.  After each
    replay the parameters' version counters are bumped."""

    def __init__(self, model, optimizer, batch_size, max_path_length, loss_fn=None, criterion=None):
        B, L = int(batch_size), int(max_path_length)
        super().__init__(model, ((B, L), (B, L), (B, L), (B,)))
        if isinstance(optimizer, ShardedFlatAdam) and optimizer.world > 1:
            raise NotImplementedError("GraphedTrainStep: ShardedFlatAdam at world size > 1 uses cross-GPU barriers and a "
                                      "side stream and cannot be captured")
        if isinstance(optimizer, (FlatAdam, ShardedFlatAdam)) and not optimizer.capturable:
            raise ValueError(f"GraphedTrainStep: construct {type(optimizer).__name__} with capturable=True")
        if model.terminal_embedding.sparse or model.path_embedding.sparse:
            raise NotImplementedError("GraphedTrainStep: sparse embedding gradients cannot be captured")
        if model.training and model.input_dropout is not None and model._rng_base is None:
            raise RuntimeError("GraphedTrainStep: dropout needs device-drawn keys: call model.use_device_rng() first")
        self.optimizer, self.loss_fn, self.criterion = optimizer, loss_fn, criterion

    def _settings(self):
        o = self.optimizer
        if isinstance(o, (FlatAdam, ShardedFlatAdam)):
            hyper = (o.lr, o.betas, o.eps, o.weight_decay)
        else:
            hyper = tuple(tuple((k, v) for k, v in sorted(g.items()) if k != "params" and not isinstance(v, torch.Tensor))
                          for g in o.param_groups)
        c = self.criterion
        crit = None if c is None else (type(c), c.ignore_index, getattr(c, "label_smoothing", 0.0), c.reduction,
                                       None if c.weight is None else (c.weight.data_ptr(), tuple(c.weight.shape)))
        # the deterministic mode selects other kernels and workspace sizes than the captured ones, the matmul precision
        # other kernels
        return (self.model.training, torch.are_deterministic_algorithms_enabled(), torch_matmul_tf32(), hyper, crit)

    def _run(self, starts, paths, ends, label):
        model, opt = self.model, self.optimizer
        if isinstance(opt, FlatAdam):
            loss = ddp_step(model, opt, opt.bucket, starts, paths, ends, label, self.loss_fn, self.criterion)
        elif isinstance(opt, ShardedFlatAdam):
            loss = ddp_step(model, opt, None, starts, paths, ends, label, self.loss_fn, self.criterion)
        else:
            opt.zero_grad(set_to_none=False)
            if self.loss_fn is None:
                loss = _forward_loss(model, starts, paths, ends, label, self.criterion)
            else:
                loss = self.loss_fn(model(starts, paths, ends, label)[0], label)
            loss.backward()
            opt.step()
        return loss.detach()

    def __call__(self, starts, paths, ends, label):
        loss = self._call(starts, paths, ends, label)
        if loss is self.static_out:
            _bump_versions(self.model)
            return loss.clone()
        return loss


class GraphedPredict(_Graphed):
    """Code2Vec.predict() (k None) or predict_topk(k) on [batch_size, max_path_length] batches, captured into a CUDA
    graph after one eager warm-up call; returns fresh tensors, the same values as the eager call.  Other shapes run
    eagerly.  model.training is fixed at capture."""

    WARMUP = 1

    def __init__(self, model, batch_size, max_path_length, k=None):
        B, L = int(batch_size), int(max_path_length)
        super().__init__(model, ((B, L), (B, L), (B, L)))
        self.k = None if k is None else int(k)

    def _run(self, starts, paths, ends):
        if self.k is None:
            return self.model.predict(starts, paths, ends)
        return self.model.predict_topk(starts, paths, ends, k=self.k)

    def __call__(self, starts, paths, ends):
        out = self._call(starts, paths, ends)
        if out is self.static_out:
            return tuple(t.clone() if t is not None else None for t in out)
        return out

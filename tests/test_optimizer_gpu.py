"""-m gpu, one H100: FlatAdam / ShardedFlatAdam as torch optimizers: gradient clipping by global norm inside the step
(grad_sumsq_kernel, grad_norm_finalize_kernel, the DEV_COEF instantiations of adam_step_kernel), learning-rate schedules
eager and under CUDA-graph capture (a tensor lr read by adam_step_count_kernel), and checkpoints.

Every optimizer of a comparison is fed the SAME recorded gradients: those of a cfg2-shaped Code2Vec (E = H = 128, L = 200,
B = 256, small vocabularies) on ten batches, so that the backward's atomics do not blur it.  The judge is torch.optim.Adam
(+ clip_grad_norm_) on fp64 copies; fp32 torch.optim.Adam on the same gradients gives the error a correct fp32
implementation makes, and ours must stay within a small factor of it."""
import contextlib
import ctypes

import numpy as np
import pytest
import torch
import torch.nn as nn
from torch.optim import lr_scheduler as LS

from gpu_util import cuda, option_from, random_batch, random_params
from code2vec_b200 import _lib
from code2vec_b200.distributed import FlatAdam, FlatGradBucket, ShardedFlatAdam, ddp_step
from code2vec_b200.graphs import GraphedTrainStep
from code2vec_b200.model import Code2Vec

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
T, P, C, E, L, B = 3001, 2003, 301, 128, 200, 256         # odd vocabularies: the flat size is not a multiple of 4
CFG2_NUMEL = 90_000_000                                     # about cfg2's parameter count (360 MB of gradients)
KINDS = ["flat", "sharded", "sharded-early"]
PATH = 1                                                    # index of path_embedding.weight in model.parameters()


def _model(seed=0, T=T, P=P, C=C):
    o = {"T": T, "P": P, "C": C, "Et": E, "Ep": E, "H": E}
    m = Code2Vec(option_from(o, 0.0))
    m.load_state_dict({k: torch.from_numpy(v) for k, v in random_params(np.random.default_rng(seed), T, P, C, E, E, E).items()})
    return m.to(DEV)


def _batches(n, B=B, L=L, T=T, P=P, C=C, seed=1):
    rng = np.random.default_rng(seed)
    return [tuple(cuda(a) for a in random_batch(rng, B, L, T, P, C)) for _ in range(n)]


@pytest.fixture(scope="module")
def recorded():
    """(initial parameters, 12 lists of per-parameter gradients) of the cfg2-shaped model"""
    m = _model()
    grads = []
    for s, p, e, y in _batches(12):
        m.zero_grad(set_to_none=True)
        m.forward_loss(s, p, e, y)[0].backward()
        grads.append([q.grad.detach().clone() for q in m.parameters()])
    init = [q.detach().clone() for q in m.parameters()]
    assert sum(q.numel() for q in init) % 4 != 0
    return init, grads


def _ours(kind, init, **kw):
    params = [nn.Parameter(q.clone()) for q in init]
    if kind == "flat":
        return params, FlatAdam(FlatGradBucket(params), **kw)
    return params, ShardedFlatAdam(params, early=[params[PATH]] if kind == "sharded-early" else (), **kw)


def _feed(params, grads):
    for p, g in zip(params, grads):
        p.grad.copy_(g)


def _run_ours(kind, init, grads, sched=None, **kw):
    params, opt = _ours(kind, init, **kw)
    sch = sched(opt) if sched else None
    norms = []
    for g in grads:
        _feed(params, g)
        opt.step()
        norms.append(opt.grad_norm.clone())
        if sch:
            sch.step()
    return params, opt, torch.cat(norms)


def _run_torch(init, grads, dtype, max_norm=None, sched=None, **kw):
    params = [nn.Parameter(q.to(dtype).clone()) for q in init]
    opt = torch.optim.Adam(params, **kw)
    sch = sched(opt) if sched else None
    norms = []
    for g in grads:
        for p, x in zip(params, g):
            p.grad = x.to(dtype).clone()
        if max_norm is not None:
            norms.append(torch.nn.utils.clip_grad_norm_(params, max_norm).reshape(1))
        opt.step()
        if sch:
            sch.step()
    return params, opt, (torch.cat(norms) if norms else None)


def _err(params, ref64):
    return max(float((p.detach().double() - r.detach()).abs().max()) for p, r in zip(params, ref64))


def _assert_within_torch(what, ours, ref32, ref64, factor=4.0, floor=1e-7):
    e_ours, e_torch = _err(ours, ref64), _err(ref32, ref64)
    print(f"{what}: max |p - fp64 Adam|: ours {e_ours:.3e}, fp32 torch.optim.Adam {e_torch:.3e}")
    assert e_ours <= factor * e_torch + floor, (what, e_ours, e_torch)


def _bits_equal(a, b):
    return torch.equal(a.detach().contiguous().view(torch.int32), b.detach().contiguous().view(torch.int32))


# ---- the norm ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 3, 5, 255, 1023, 1027, 4 * 256 * 1024 + 6, CFG2_NUMEL + 3])
def test_norm_matches_fp64_and_is_reproducible(n):
    lib = _lib.load()
    V = ctypes.c_void_p
    gen = torch.Generator(device=DEV).manual_seed(n % 1000)
    g = torch.randn(n, device=DEV, generator=gen) * torch.pow(10.0, torch.empty(n, device=DEV).uniform_(-4, 1, generator=gen))
    ws = torch.empty(lib.c2v_grad_norm_workspace_bytes(n) // 4, device=DEV)
    keep = g.clone()
    outs = []
    for gs, max_norm in ((1.0, 1e30), (1.0 / 3.0, 0.5), (1.0 / 3.0, 0.5)):
        ws.fill_(float("nan"))                               # the workspace needs no initialisation
        out = torch.full((2,), -1.0, device=DEV)
        rc = lib.c2v_grad_clip_coef(V(g.data_ptr()), n, gs, max_norm, V(out.data_ptr()), V(ws.data_ptr()), 4 * ws.numel(),
                                    V(torch.cuda.current_stream().cuda_stream))
        _lib.check(rc, "c2v_grad_clip_coef")
        outs.append(out)
        ref = float(g.double().square().sum().sqrt()) * gs
        norm, coef = (float(x) for x in out)
        assert abs(norm - ref) <= 1e-6 * ref, (n, norm, ref)
        expect = min(1.0, max_norm / (ref + 1e-6))
        assert coef == 1.0 if expect == 1.0 else abs(coef - expect) <= 4e-6 * expect, (n, coef, expect)
    assert _bits_equal(outs[1], outs[2]) and _bits_equal(g, keep)


def test_launch_count_counts_the_norm_kernels():
    lib = _lib.load()
    params, opt = _ours("flat", [torch.randn(1000, device=DEV)], max_grad_norm=1.0)
    before = lib.c2v_launch_count()
    opt.step()
    assert lib.c2v_launch_count() - before == 3              # grad_sumsq_kernel, grad_norm_finalize_kernel, adam_step_kernel


# ---- clipping -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("capturable", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_inactive_clip_changes_no_bit(recorded, kind, capturable):
    init, grads = recorded
    a, oa, _ = _run_ours(kind, init, grads[:5], weight_decay=0.01, capturable=capturable)
    b, ob, norms = _run_ours(kind, init, grads[:5], weight_decay=0.01, capturable=capturable, max_grad_norm=1e6)
    assert float(ob._norm_coef[1]) == 1.0 and float(norms.min()) > 0.0
    assert all(_bits_equal(x, y) for x, y in zip(a, b))
    assert _bits_equal(oa.exp_avg, ob.exp_avg) and _bits_equal(oa.exp_avg_sq, ob.exp_avg_sq)


@pytest.mark.parametrize("capturable", [False, True])
@pytest.mark.parametrize("wd", [0.0, 0.01])
@pytest.mark.parametrize("kind", ["flat", "sharded-early"])
def test_active_clip_matches_clip_grad_norm(recorded, kind, wd, capturable):
    init, grads = recorded
    grads = grads[:10]
    typical = float(torch.cat([g.reshape(-1) for g in grads[0]]).double().norm())
    max_norm = typical / 3.0
    ours, opt, norms = _run_ours(kind, init, grads, lr=1e-3, weight_decay=wd, capturable=capturable, max_grad_norm=max_norm)
    ref32, _, norms32 = _run_torch(init, grads, torch.float32, max_norm, lr=1e-3, weight_decay=wd)
    ref64, _, norms64 = _run_torch(init, grads, torch.float64, max_norm, lr=1e-3, weight_decay=wd)
    assert float(norms64.min()) > max_norm                                      # every step was clipped
    assert float(((norms.double() - norms64) / norms64).abs().max()) <= 1e-6
    assert float(opt._norm_coef[1]) < 0.5
    _assert_within_torch(f"clip {kind} wd={wd} capturable={capturable}", ours, ref32, ref64)
    assert opt.step_count() == 10


@pytest.mark.parametrize("kind", ["flat", "sharded"])
@pytest.mark.parametrize("bad", [float("nan"), float("inf")])
def test_nonfinite_gradient_is_not_hidden(recorded, kind, bad):
    init, grads = recorded
    g = [x.clone() for x in grads[0]]
    g[2].view(-1)[7] = bad
    ours, opt, norms = _run_ours(kind, init, [g], max_grad_norm=1.0)
    ref, _, norms32 = _run_torch(init, [g], torch.float32, 1.0)
    if bad != bad:
        assert bool(norms.isnan().all()) and bool(norms32.isnan().all())
        assert all(bool(p.isnan().all()) for p in ours) and all(bool(p.isnan().all()) for p in ref)
    else:
        assert bool(norms.isinf().all()) and bool(norms32.isinf().all())
        assert bool(ours[2].view(-1)[7].isnan()) and bool(ref[2].view(-1)[7].isnan())     # inf * 0


# ---- schedules ----------------------------------------------------------------------------------------------------------
def _warmup_cosine(opt):
    warm = LS.LambdaLR(opt, lambda e: min(1.0, (e + 1) / 5.0))
    return LS.SequentialLR(opt, [warm, LS.CosineAnnealingLR(opt, T_max=15)], milestones=[5])


@pytest.mark.filterwarnings("ignore:The epoch parameter")
@pytest.mark.parametrize("kind", KINDS)
def test_eager_schedule_follows_torch_adam(recorded, kind):
    init, grads = recorded
    grads = (grads + grads)[:20]
    ours, opt, _ = _run_ours(kind, init, grads, sched=_warmup_cosine, lr=2e-3, weight_decay=0.01)
    ref32, t32, _ = _run_torch(init, grads, torch.float32, sched=_warmup_cosine, lr=2e-3, weight_decay=0.01)
    ref64, _, _ = _run_torch(init, grads, torch.float64, sched=_warmup_cosine, lr=2e-3, weight_decay=0.01)
    assert opt.lr == t32.param_groups[0]["lr"] and opt.lr < 2e-3 * 0.05
    _assert_within_torch(f"schedule {kind}", ours, ref32, ref64)


def test_one_cycle_moves_beta1(recorded):
    init, grads = recorded
    sched = lambda o: LS.OneCycleLR(o, max_lr=5e-3, total_steps=13)
    ours, opt, _ = _run_ours("flat", init, grads, sched=sched, lr=1e-3)
    ref32, t32, _ = _run_torch(init, grads, torch.float32, sched=sched, lr=1e-3)
    ref64, _, _ = _run_torch(init, grads, torch.float64, sched=sched, lr=1e-3)
    assert opt.betas == t32.param_groups[0]["betas"] and opt.betas[0] != 0.9
    _assert_within_torch("OneCycleLR", ours, ref32, ref64)


@contextlib.contextmanager
def _deterministic():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


def _sched_run(graphed, batches, kind="flat"):
    m = _model(seed=3, T=300, P=200, C=17).train()
    lr = torch.tensor(2e-3, device=DEV)
    if kind == "flat":
        opt = FlatAdam(FlatGradBucket(m.parameters()), lr=lr, capturable=True, max_grad_norm=0.01, weight_decay=0.01)
        bucket = opt.bucket
    else:
        opt = ShardedFlatAdam(m.parameters(), lr=lr, capturable=True, max_grad_norm=0.01, weight_decay=0.01)
        bucket = None
    sch = LS.LambdaLR(opt, lambda e: min(1.0, (e + 1) / 4.0) * 0.9 ** e)
    step = GraphedTrainStep(m, opt, 32, 40) if graphed else None
    losses, launches = [], []
    lib = _lib.load()
    with _deterministic():
        for b in batches:
            before = lib.c2v_launch_count()
            loss = step(*b) if graphed else ddp_step(m, opt, bucket, *b, None)
            launches.append(lib.c2v_launch_count() - before)
            losses.append(loss.detach().clone())
            sch.step()
    torch.cuda.synchronize()
    return m, opt, torch.stack(losses), launches, step


@pytest.mark.parametrize("kind", ["flat", "sharded"])
def test_captured_schedule_equals_eager(kind):
    batches = _batches(12, B=32, L=40, T=300, P=200, C=17, seed=5)
    me, oe, le, _, _ = _sched_run(False, batches, kind)
    mg, og, lg, launches, step = _sched_run(True, batches, kind)
    assert step.graph is not None and launches[0] > 0 and launches[3:] == [0] * 9      # replays launch through the graph
    assert _bits_equal(le, lg)
    for a, b in zip(me.parameters(), mg.parameters()):
        assert _bits_equal(a, b)
    assert _bits_equal(oe.exp_avg, og.exp_avg) and _bits_equal(oe.grad_norm, og.grad_norm)
    assert oe.step_count() == og.step_count() == 12 and float(og.lr) == float(oe.lr) < 2e-3
    assert float(og._norm_coef[1]) < 1.0                                                # the clip was active
    og.eps = 1e-6                                                                       # a launch parameter: frozen
    with pytest.raises(RuntimeError, match="changed since the capture"):
        step(*batches[0])


def test_float_lr_changed_after_capture_still_raises():
    batches = _batches(4, B=32, L=40, T=300, P=200, C=17, seed=6)
    m = _model(seed=3, T=300, P=200, C=17).train()
    opt = FlatAdam(FlatGradBucket(m.parameters()), lr=1e-3, capturable=True)
    step = GraphedTrainStep(m, opt, 32, 40)
    sch = LS.StepLR(opt, step_size=1, gamma=0.5)
    for b in batches[:3]:
        step(*b)
    sch.step()
    with pytest.raises(RuntimeError, match="changed since the capture"):
        step(*batches[3])


# ---- checkpoints ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("capturable", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_resume_is_bit_identical(recorded, kind, capturable):
    init, grads = recorded
    # (a tensor lr belongs to one optimizer: its scheduler fills it in place)
    kw = lambda lr: dict(lr=torch.tensor(lr, device=DEV) if capturable else lr, weight_decay=0.01, capturable=capturable,
                         max_grad_norm=0.1)
    sched = lambda o: LS.StepLR(o, step_size=4, gamma=0.5)
    straight, so, _ = _run_ours(kind, init, grads, sched=sched, **kw(1e-3))
    half, ho, _ = _run_ours(kind, init, grads[:6], sched=sched, **kw(1e-3))
    sd = ho.state_dict()
    assert sd["state"][0]["step"].device.type == ("cuda" if capturable else "cpu") and float(sd["state"][0]["step"]) == 6.0
    assert sd["state"][PATH]["exp_avg"].shape == init[PATH].shape
    params, opt = _ours(kind, [p.detach() for p in half], **kw(7.0))         # the checkpoint's lr wins
    opt.load_state_dict(sd)
    assert opt.step_count() == 6 and float(opt.lr) == pytest.approx(5e-4) and opt.max_grad_norm == 0.1
    sch = sched(opt)
    sch.last_epoch = 6
    for g in grads[6:]:
        _feed(params, g)
        opt.step()
        sch.step()
    assert all(_bits_equal(a, b) for a, b in zip(params, straight))
    assert _bits_equal(opt.exp_avg, so.exp_avg) and _bits_equal(opt.exp_avg_sq, so.exp_avg_sq)
    assert opt.step_count() == 12 and float(opt.lr) == float(so.lr)


@pytest.mark.parametrize("capturable", [False, True])
def test_cross_load_with_torch_adam(recorded, capturable):
    """FlatAdam -> torch.optim.Adam -> FlatAdam, one step each side, against torch's Adam alone"""
    init, grads = recorded
    ref32, _, _ = _run_torch(init, grads[:3], torch.float32, lr=1e-3, weight_decay=0.01)
    ref64, _, _ = _run_torch(init, grads[:3], torch.float64, lr=1e-3, weight_decay=0.01)
    a, oa, _ = _run_ours("flat", init, grads[:1], lr=1e-3, weight_decay=0.01, capturable=capturable)
    mid = [nn.Parameter(p.detach().clone()) for p in a]
    t = torch.optim.Adam(mid, lr=0.5, capturable=capturable)
    t.load_state_dict(oa.state_dict())
    assert t.param_groups[0]["lr"] == 1e-3 and t.param_groups[0]["weight_decay"] == 0.01
    for p, g in zip(mid, grads[1]):
        p.grad = g.clone()
    t.step()
    params, opt = _ours("flat", [p.detach() for p in mid], capturable=capturable)
    opt.load_state_dict(t.state_dict())
    assert opt.step_count() == 2 and opt.weight_decay == 0.01
    _feed(params, grads[2])
    opt.step()
    _assert_within_torch(f"cross-load capturable={capturable}", params, ref32, ref64)

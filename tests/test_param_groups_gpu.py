"""-m gpu, one H100: parameter groups in FlatAdam / ShardedFlatAdam (the AdamGroups instantiations of adam_step_kernel,
adam_step_sharded_kernel and adam_step_bulk_kernel, and adam_step_count_groups_kernel) against torch.optim.Adam / AdamW
with the same groups.

Every optimizer of a comparison is fed the SAME recorded gradients (those of a cfg2-shaped Code2Vec, or random ones for
small parameter sets), as in test_optimizer_gpu.py.  The judge is torch's optimizer on fp64 copies; fp32 torch on the same
gradients gives the error a correct fp32 implementation makes, and ours must stay within a small factor of it.  The
grouped sharded kernels are also run on one GPU with emulated ranks (as test_adam_gpu.py runs today's), against an fp64
Adam / AdamW element by element."""
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
KINDS = ["flat", "sharded", "sharded-early"]
NAMES = [n for n, _ in Code2Vec(option_from({"T": 5, "P": 5, "C": 3, "Et": 4, "Ep": 4, "H": 4}, 0.0)).named_parameters()]
# the usual recipe: weight decay on the embedding tables, input_linear and output_linear.weight, none on LayerNorm's weight
# and bias, attention_parameter and the output bias (interleaved in the model's parameter order)
DECAY = [i for i, n in enumerate(NAMES) if n.endswith("embedding.weight") or n in ("input_linear.weight",
                                                                                   "output_linear.weight")]
NO_DECAY = [i for i in range(len(NAMES)) if i not in DECAY]
PATH = NAMES.index("path_embedding.weight")


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
    """(initial parameters, 10 lists of per-parameter gradients) of the cfg2-shaped model"""
    m = _model()
    grads = []
    for s, p, e, y in _batches(10):
        m.zero_grad(set_to_none=True)
        m.forward_loss(s, p, e, y)[0].backward()
        grads.append([q.grad.detach().clone() for q in m.parameters()])
    return [q.detach().clone() for q in m.parameters()], grads


def _spec(params, spec):
    """[{"idx": [...], **hyper}] -> torch's group dicts over `params`"""
    return [dict({k: v for k, v in g.items() if k != "idx"}, params=[params[i] for i in g["idx"]]) for g in spec]


def _ours(kind, init, spec, early=PATH, **kw):
    params = [nn.Parameter(q.clone()) for q in init]
    groups = _spec(params, spec)
    if kind == "flat":
        return params, FlatAdam(FlatGradBucket(params), groups=groups, **kw)
    return params, ShardedFlatAdam(groups, early=[params[early]] if kind == "sharded-early" else (), **kw)


def _run_ours(kind, init, grads, spec, sched=None, early=PATH, **kw):
    params, opt = _ours(kind, init, spec, early, **kw)
    sch = sched(opt) if sched else None
    for g in grads:
        for p, x in zip(params, g):
            p.grad.copy_(x)
        opt.step()
        if sch:
            sch.step()
    return params, opt


def _run_torch(init, grads, spec, dtype, max_norm=None, sched=None, **kw):
    params = [nn.Parameter(q.to(dtype).clone()) for q in init]
    opt = torch.optim.Adam(_spec(params, spec), **kw)
    sch = sched(opt) if sched else None
    for g in grads:
        for p, x in zip(params, g):
            p.grad = x.to(dtype).clone()
        if max_norm is not None:
            torch.nn.utils.clip_grad_norm_(params, max_norm)
        opt.step()
        if sch:
            sch.step()
    return params, opt


def _err(params, ref64):
    return max(float((p.detach().double() - r.detach()).abs().max()) for p, r in zip(params, ref64))


def _assert_within_torch(what, ours, ref32, ref64, factor=4.0, floor=1e-7):
    e_ours, e_torch = _err(ours, ref64), _err(ref32, ref64)
    print(f"{what}: max |p - fp64 Adam|: ours {e_ours:.3e}, fp32 torch.optim.Adam {e_torch:.3e}")
    assert e_ours <= factor * e_torch + floor, (what, e_ours, e_torch)


def _bits_equal(a, b):
    return torch.equal(a.detach().contiguous().view(torch.int32), b.detach().contiguous().view(torch.int32))


def _kernels(fn):
    """names of the c2v kernels `fn` launches"""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.name for e in prof.events() if "c2v::" in e.name}


RECIPE = [{"idx": DECAY, "weight_decay": 0.01}, {"idx": NO_DECAY, "weight_decay": 0.0}]


# ---- the no-decay recipe -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("decoupled", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_no_decay_recipe_matches_torch(recorded, kind, decoupled):
    init, grads = recorded
    grads = (grads + grads)[:20]
    kw = dict(lr=2e-3, decoupled_weight_decay=decoupled)
    ours, opt = _run_ours(kind, init, grads, RECIPE, **kw)
    ref32, _ = _run_torch(init, grads, RECIPE, torch.float32, **kw)
    ref64, _ = _run_torch(init, grads, RECIPE, torch.float64, **kw)
    _assert_within_torch(f"recipe {kind} decoupled={decoupled}", ours, ref32, ref64)
    assert opt.step_count() == 20
    names = _kernels(lambda: opt.step())
    assert any("adam_step_kernel" in n and "AdamGroups" in n for n in names), names


def test_one_adamw_group_takes_the_grouped_kernel_and_one_adam_group_todays(recorded):
    init, grads = recorded
    for decoupled in (False, True):
        params, opt = _ours("flat", init, [{"idx": list(range(len(init)))}], decoupled_weight_decay=decoupled,
                            weight_decay=0.1)
        names = _kernels(lambda: opt.step())
        assert any("adam_step_kernel" in n and ("AdamGroups" in n) == decoupled for n in names), (decoupled, names)


# ---- interleaved groups, boundaries at odd offsets -----------------------------------------------------------------------
SIZES = [5, 1, 7, 3, 100_003, 13, 1, 9, 2, 11, 4 * 256 * 1024 + 6]
INTERLEAVED = [
    {"idx": [0, 3, 5, 8, 10], "lr": 3e-3, "betas": (0.9, 0.999), "weight_decay": 0.02, "decoupled_weight_decay": True},
    {"idx": [1], "lr": 1e-2, "betas": (0.5, 0.9), "eps": 1e-6},                          # one element, a group of its own
    {"idx": [2, 4, 6, 7, 9], "lr": 1e-3, "betas": (0.8, 0.99), "weight_decay": 0.05},
]


def _random_grads(n_steps, seed=7):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    init = [torch.randn(n, generator=gen, device=DEV) for n in SIZES]
    grads = [[torch.randn(n, generator=gen, device=DEV) * 10.0 ** float(torch.empty(1).uniform_(-3, 1)) for n in SIZES]
             for _ in range(n_steps)]
    return init, grads


@pytest.mark.parametrize("kind", KINDS)
def test_three_interleaved_groups_match_torch(kind):
    init, grads = _random_grads(20)
    ours, opt = _run_ours(kind, init, grads, INTERLEAVED, early=4)
    # FlatAdam keeps the bucket's order, so the groups interleave; ShardedFlatAdam lays out the groups in order, the
    # early parameter first
    assert len(opt._segments) == {"flat": 10, "sharded": 3, "sharded-early": 4}[kind], opt._segments
    ref32, _ = _run_torch(init, grads, INTERLEAVED, torch.float32)
    ref64, _ = _run_torch(init, grads, INTERLEAVED, torch.float64)
    _assert_within_torch(f"interleaved {kind}", ours, ref32, ref64)


# ---- schedules -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sched", ["lambda", "onecycle"])
@pytest.mark.parametrize("kind", KINDS)
def test_per_group_schedules_follow_torch(recorded, kind, sched):
    init, grads = recorded
    spec = [dict(RECIPE[0], lr=2e-3), dict(RECIPE[1], lr=5e-4)]
    if sched == "lambda":
        mk = lambda o: LS.LambdaLR(o, [lambda e: min(1.0, (e + 1) / 4.0), lambda e: 0.8 ** e])
    else:
        mk = lambda o: LS.OneCycleLR(o, max_lr=[5e-3, 1e-3], total_steps=11)
    ours, opt = _run_ours(kind, init, grads, spec, sched=mk, decoupled_weight_decay=True)
    ref32, t32 = _run_torch(init, grads, spec, torch.float32, sched=mk, decoupled_weight_decay=True)
    ref64, _ = _run_torch(init, grads, spec, torch.float64, sched=mk, decoupled_weight_decay=True)
    for a, b in zip(opt.param_groups, t32.param_groups):
        assert a["lr"] == b["lr"] and a["betas"] == b["betas"]
    assert opt.param_groups[0]["lr"] != opt.param_groups[1]["lr"]
    _assert_within_torch(f"schedule {sched} {kind}", ours, ref32, ref64)


def _sched_run(graphed, batches, kind):
    m = _model(seed=3, T=300, P=200, C=17).train()
    params = list(m.parameters())
    lrs = [torch.tensor(2e-3, device=DEV), torch.tensor(1e-3, device=DEV)]
    groups = [{"params": [params[i] for i in DECAY], "lr": lrs[0], "weight_decay": 0.01, "decoupled_weight_decay": True},
              {"params": [params[i] for i in NO_DECAY], "lr": lrs[1], "betas": (0.8, 0.99)}]
    if kind == "flat":
        opt = FlatAdam(FlatGradBucket(params), groups=groups, capturable=True, max_grad_norm=0.01)
        bucket = opt.bucket
    else:
        opt = ShardedFlatAdam(groups, capturable=True, max_grad_norm=0.01)
        bucket = None
    sch = LS.LambdaLR(opt, [lambda e: min(1.0, (e + 1) / 4.0) * 0.9 ** e, lambda e: 0.7 ** e])
    step = GraphedTrainStep(m, opt, 32, 40) if graphed else None
    losses, launches = [], []
    lib = _lib.load()
    for b in batches:
        before = lib.c2v_launch_count()
        loss = step(*b) if graphed else ddp_step(m, opt, bucket, *b, None)
        launches.append(lib.c2v_launch_count() - before)
        losses.append(loss.detach().clone())
        sch.step()
    torch.cuda.synchronize()
    return m, opt, torch.stack(losses), launches, step


@pytest.mark.parametrize("kind", ["flat", "sharded"])
def test_captured_group_schedules_equal_eager(kind):
    torch.use_deterministic_algorithms(True)
    try:
        batches = _batches(12, B=32, L=40, T=300, P=200, C=17, seed=5)
        me, oe, le, _, _ = _sched_run(False, batches, kind)
        mg, og, lg, launches, step = _sched_run(True, batches, kind)
    finally:
        torch.use_deterministic_algorithms(False)
    assert step.graph is not None and launches[3:] == [0] * 9
    assert _bits_equal(le, lg)
    for a, b in zip(me.parameters(), mg.parameters()):
        assert _bits_equal(a, b)
    assert _bits_equal(oe.exp_avg, og.exp_avg) and _bits_equal(oe.exp_avg_sq, og.exp_avg_sq)
    assert oe.step_count() == og.step_count() == 12
    assert [float(g["lr"]) for g in og.param_groups] == [float(g["lr"]) for g in oe.param_groups]
    og.param_groups[1]["betas"] = (0.9, 0.999)                    # a launch parameter of group 1: frozen at capture
    with pytest.raises(RuntimeError, match="changed since the capture"):
        step(*batches[0])


# ---- clipping ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("capturable", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_clip_with_groups_is_clip_grad_norm_then_the_grouped_step(recorded, kind, capturable):
    init, grads = recorded
    max_norm = float(torch.cat([g.reshape(-1) for g in grads[0]]).double().norm()) / 3.0
    kw = dict(lr=1e-3, decoupled_weight_decay=True)
    ours, opt = _run_ours(kind, init, grads, RECIPE, max_grad_norm=max_norm, capturable=capturable, **kw)
    ref32, _ = _run_torch(init, grads, RECIPE, torch.float32, max_norm, **kw)
    ref64, _ = _run_torch(init, grads, RECIPE, torch.float64, max_norm, **kw)
    assert float(opt._norm_coef[1]) < 0.5
    _assert_within_torch(f"clip {kind} capturable={capturable}", ours, ref32, ref64)


# ---- checkpoints ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("capturable", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_grouped_resume_is_bit_identical(recorded, kind, capturable):
    init, grads = recorded
    spec = [dict(RECIPE[0], lr=torch.tensor(2e-3, device=DEV) if capturable else 2e-3), dict(RECIPE[1])]
    kw = dict(capturable=capturable, decoupled_weight_decay=True, lr=1e-3)
    sched = lambda o: LS.StepLR(o, step_size=3, gamma=0.5)
    fresh = lambda: [dict(g, lr=g["lr"].clone()) if isinstance(g.get("lr"), torch.Tensor) else dict(g) for g in spec]
    straight, so = _run_ours(kind, init, grads, fresh(), sched=sched, **kw)
    half, ho = _run_ours(kind, init, grads[:5], fresh(), sched=sched, **kw)
    sd = ho.state_dict()
    assert [g["params"] for g in sd["param_groups"]] == [list(range(len(DECAY))),
                                                         list(range(len(DECAY), len(init)))]
    params, opt = _ours(kind, [p.detach() for p in half], fresh(), **kw)
    opt.load_state_dict(sd)
    assert opt.step_count() == 5
    sch = sched(opt)
    sch.last_epoch = 5
    for g in grads[5:]:
        for p, x in zip(params, g):
            p.grad.copy_(x)
        opt.step()
        sch.step()
    assert all(_bits_equal(a, b) for a, b in zip(params, straight))
    assert _bits_equal(opt.exp_avg, so.exp_avg) and _bits_equal(opt.exp_avg_sq, so.exp_avg_sq)


@pytest.mark.parametrize("decoupled", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_cross_load_with_torch_groups(recorded, kind, decoupled):
    """ours -> torch.optim.Adam / AdamW -> ours, against torch alone over the same three steps"""
    init, grads = recorded
    cls = torch.optim.AdamW if decoupled else torch.optim.Adam
    kw = dict(lr=1e-3, decoupled_weight_decay=decoupled)
    ref32, _ = _run_torch(init, grads[:3], RECIPE, torch.float32, **kw)
    ref64, _ = _run_torch(init, grads[:3], RECIPE, torch.float64, **kw)
    a, oa = _run_ours(kind, init, grads[:1], RECIPE, **kw)
    mid = [nn.Parameter(p.detach().clone()) for p in a]
    t = cls(_spec(mid, [{"idx": g["idx"]} for g in RECIPE]), lr=0.5)
    t.load_state_dict(oa.state_dict())
    assert [g["weight_decay"] for g in t.param_groups] == [0.01, 0.0]
    assert all(g["decoupled_weight_decay"] == decoupled for g in t.param_groups)
    for p, g in zip(mid, grads[1]):
        p.grad = g.clone()
    t.step()
    params, opt = _ours(kind, [p.detach() for p in mid], [{"idx": g["idx"]} for g in RECIPE])
    opt.load_state_dict(t.state_dict())
    assert opt.step_count() == 2 and [g["decoupled_weight_decay"] for g in opt.param_groups] == [decoupled] * 2
    for p, x in zip(params, grads[2]):
        p.grad.copy_(x)
    opt.step()
    _assert_within_torch(f"cross-load {kind} decoupled={decoupled}", params, ref32, ref64)


# ---- the grouped sharded kernels with emulated ranks ----------------------------------------------------------------------
V = ctypes.c_void_p
GROUP_HYPER = [(1e-3, 0.9, 0.999, 1e-8, 0.01, 0), (3e-3, 0.8, 0.99, 1e-6, 0.05, 1), (2e-2, 0.5, 0.9, 1e-7, 0.0, 0)]
SLICE_BEGIN = 36                 # rank 0's slice begins here, inside segment 0


def _table(seg_begin, seg_group):
    groups = (_lib.AdamGroup * len(GROUP_HYPER))()
    for a, (lr, b1, b2, eps, wd, dec) in zip(groups, GROUP_HYPER):
        a.lr, a.beta1, a.beta2, a.eps, a.weight_decay, a.decoupled, a.lr_dev = lr, b1, b2, eps, wd, dec, None
    return (groups, len(groups), (ctypes.c_int64 * len(seg_begin))(*seg_begin),
            (ctypes.c_int32 * len(seg_group))(*seg_group), len(seg_begin))


def _f32(x):
    return float(np.float32(x))


def _judge(where, gidx, p, s, m, v, new_p, new_m, new_v, t, gs):
    """fp64 Adam / AdamW, element by element with its group's hyper-parameters (as the fp32 values the kernel gets);
    AdamW's p * (1 - lr * wd) is a rounded fp32 product, as in torch's param.mul_"""
    h = torch.tensor([[_f32(x) for x in g[:5]] + [g[5]] for g in GROUP_HYPER], dtype=torch.float64, device=DEV)[gidx]
    lr, b1, b2, eps, wd, dec = h.unbind(1)
    p, s, m, v = (x.double() for x in (p, s, m, v))
    decay = (1.0 - lr * wd).float()
    p = torch.where(dec > 0, (p.float() * decay).double(), p)
    gr = s * _f32(gs) + torch.where(dec > 0, 0.0, wd) * p
    m64 = b1 * m + (1.0 - b1) * gr
    v64 = b2 * v + (1.0 - b2) * gr * gr
    p64 = p - (lr / (1.0 - b1 ** t)) * m64 / (torch.sqrt(v64) / torch.sqrt(1.0 - b2 ** t) + eps)
    ulp = torch.ldexp(torch.ones_like(p64), (torch.frexp(p64.float())[1] - 24).double())
    # the update itself carries a few fp32 roundings (m, v, sqrt, the quotient, step_size): with b2 = 0.9 and lr = 2e-2
    # its error can exceed lr * 2^-20, so the bound also scales with it
    upd = (p64 - p).abs()
    for name, got, ref, bound in (("param", new_p, p64, 3.0 * ulp + lr * 2.0 ** -20 + upd * 2.0 ** -19),
                                  ("exp_avg", new_m, m64, 8 * 2.0 ** -24 * (b1 * m.abs() + (1 - b1) * gr.abs())),
                                  ("exp_avg_sq", new_v, v64, 8 * 2.0 ** -24 * (b2 * v + (1 - b2) * gr * gr))):
        bad = ~((got.double() - ref).abs() <= bound)
        if int(bad.sum()):
            i = int(bad.nonzero()[0, 0])
            raise AssertionError(f"{where}: {name}: {int(bad.sum())} elements off, first {i} (group {int(gidx[i])}): "
                                 f"got {float(got[i])!r}, fp64 {float(ref[i])!r}, bound {float(bound[i]):.3e}")


@pytest.mark.parametrize("path", ["peer", "bulk"])
@pytest.mark.parametrize("W", [1, 2, 4])
def test_grouped_sharded_kernels_match_fp64(W, path):
    """W ranks' buffers on one device; rank r owns [SLICE_BEGIN + r * sn, +sn); segments begin at odd elements, one
    inside rank 0's slice, and a one-element segment; every rank's launch reads all ranks' gradients"""
    lib = _lib.load()
    sn = 4 * 3001 if path == "peer" else 4 * 1000
    hi = SLICE_BEGIN + W * sn
    seg_begin = [0, SLICE_BEGIN + 7, SLICE_BEGIN + 8, SLICE_BEGIN + 1001, hi // 2 + 3, hi - 5]
    seg_group = [0, 2, 1, 0, 2, 1]
    gidx = torch.zeros(hi, dtype=torch.int64, device=DEV)
    for b, k in zip(seg_begin, seg_group):
        gidx[b:] = k
    gen = torch.Generator(device=DEV).manual_seed(97 * W + len(path))
    for t in (1, 7):
        p0 = torch.randn(hi, generator=gen, device=DEV)
        g = torch.randn(W, hi, generator=gen, device=DEV) * 0.1
        m0 = torch.randn(hi, generator=gen, device=DEV) * 0.01 if t > 1 else torch.zeros(hi, device=DEV)
        v0 = torch.rand(hi, generator=gen, device=DEV) * 1e-4 if t > 1 else torch.zeros(hi, device=DEV)
        param = [p0.clone() for _ in range(W)]
        grad = [g[r].clone() for r in range(W)]
        m = [m0[SLICE_BEGIN + r * sn:SLICE_BEGIN + (r + 1) * sn].clone() for r in range(W)]
        v = [v0[SLICE_BEGIN + r * sn:SLICE_BEGIN + (r + 1) * sn].clone() for r in range(W)]
        ptab = (V * W)(*[V(x.data_ptr()) for x in param])
        gtab = (V * W)(*[V(x.data_ptr()) for x in grad])
        stream = V(torch.cuda.current_stream().cuda_stream)
        for r in range(W):
            args = (V(param[r].data_ptr()),)
            if path == "peer":
                rc = lib.c2v_adam_step_sharded_groups(*args, None, None, ptab, gtab, W, V(m[r].data_ptr()),
                                                      V(v[r].data_ptr()), SLICE_BEGIN + r * sn, sn, None, 0,
                                                      *_table(seg_begin, seg_group), t, 1.0 / W, stream)
            else:
                rc = lib.c2v_adam_step_sharded_bulk_groups(*args, ptab, gtab, W, V(m[r].data_ptr()), V(v[r].data_ptr()),
                                                           SLICE_BEGIN + r * sn, sn, *_table(seg_begin, seg_group), t,
                                                           1.0 / W, 3, stream)
            assert rc == _lib.C2V_OK, lib.c2v_last_error()
        torch.cuda.synchronize()
        for r in range(W):
            assert _bits_equal(param[r], param[0])
            assert _bits_equal(param[r][:SLICE_BEGIN], p0[:SLICE_BEGIN])           # outside every slice: untouched
        s = torch.zeros(hi, device=DEV)
        for r in range(W):
            s = s + g[r]
        lo = SLICE_BEGIN
        _judge(f"{path} W={W} t={t}", gidx[lo:], p0[lo:], s[lo:], m0[lo:], v0[lo:], param[0][lo:], torch.cat(m),
               torch.cat(v), t, 1.0 / W)


def test_grouped_flat_kernel_matches_fp64_across_the_grid():
    """c2v_adam_step_groups over more than one grid-stride iteration, with a tail of 3 and host / device step counts"""
    lib = _lib.load()
    n = 2 * torch.cuda.get_device_properties(DEV).multi_processor_count * 16 * 256 * 4 + 4 * 37 + 3
    seg_begin = [0, 3, 4, 5, 1_000_001, n - 2]
    seg_group = [1, 0, 2, 1, 0, 2]
    gidx = torch.zeros(n, dtype=torch.int64, device=DEV)
    for b, k in zip(seg_begin, seg_group):
        gidx[b:] = k
    gen = torch.Generator(device=DEV).manual_seed(11)
    for device_step in (False, True):
        p0, g0 = torch.randn(n, generator=gen, device=DEV), torch.randn(n, generator=gen, device=DEV)
        m0, v0 = torch.randn(n, generator=gen, device=DEV) * 0.01, torch.rand(n, generator=gen, device=DEV) * 1e-4
        p, g, m, v = p0.clone(), g0.clone(), m0.clone(), v0.clone()
        state = torch.tensor([6, 0, 0, 0, 0, 0], dtype=torch.int64, device=DEV) if device_step else None
        rc = lib.c2v_adam_step_groups(*(V(x.data_ptr()) for x in (p, g, m, v)), n, *_table(seg_begin, seg_group),
                                      7, V(state.data_ptr()) if device_step else None, 0.5, 1, None,
                                      V(torch.cuda.current_stream().cuda_stream))
        assert rc == _lib.C2V_OK, lib.c2v_last_error()
        torch.cuda.synchronize()
        assert int((g != 0).sum()) == 0
        _judge(f"flat device_step={device_step}", gidx, p0, g0, m0, v0, p, m, v, 7, 0.5)
        if device_step:
            assert int(state[0]) == 7


def test_sharded_groups_keep_the_tables_16_byte_aligned():
    """the no-decay group first: the output bias (C = 17 elements) comes before the embedding tables in the flat order;
    every parameter still starts at a multiple of 4 elements, and training steps run and match FlatAdam's"""
    batches = _batches(3, B=64, L=40, T=300, P=200, C=17, seed=9)
    out = []
    for kind in ("flat", "sharded"):
        m = _model(seed=4, T=300, P=200, C=17).train()
        params = list(m.parameters())
        groups = [{"params": [params[i] for i in NO_DECAY], "weight_decay": 0.0},
                  {"params": [params[i] for i in DECAY], "weight_decay": 0.01}]
        if kind == "flat":
            opt = FlatAdam(FlatGradBucket(params), groups=groups, decoupled_weight_decay=True)
            bucket = opt.bucket
        else:
            opt = ShardedFlatAdam(groups, decoupled_weight_decay=True)
            bucket = None
            assert all(o % 4 == 0 for o in opt._flat_offsets)
            assert all(p.data_ptr() % 16 == 0 and p.grad.data_ptr() % 16 == 0 for p in params)
        losses = [ddp_step(m, opt, bucket, *b, None).detach().clone() for b in batches]
        torch.cuda.synchronize()
        out.append((torch.stack(losses), [p.detach().clone() for p in m.parameters()]))
    (la, pa), (lb, pb) = out
    assert bool(torch.isfinite(la).all()) and torch.allclose(la, lb, rtol=1e-5, atol=1e-6)
    assert all(torch.allclose(a, b, rtol=1e-4, atol=1e-6) for a, b in zip(pa, pb))

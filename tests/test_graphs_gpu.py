"""-m gpu: CUDA-graph capture of the training step and of prediction (code2vec_b200.graphs): dropout keys read from
device memory, the capturable Adam, dropout parity at a replayed step, the reference loop through GraphedTrainStep,
GraphedPredict, the stale-image guard, the deferred IndexError and steady-state memory."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gpu_util import option_from, random_params, random_batch, cuda
from philox_ref import dropout_mask
from test_graphs_abi import splitmix64
from code2vec_b200 import _lib
from code2vec_b200 import functional as CF
from code2vec_b200.distributed import FlatAdam, FlatGradBucket
from code2vec_b200.graphs import GraphedPredict, GraphedTrainStep
from code2vec_b200.model import Code2Vec

pytestmark = pytest.mark.gpu

# tensor-core shapes and a CUDA-core one (Et != Ep, not multiples of 4)
SHAPES = {"tc128": dict(Et=128, Ep=128, H=128), "tc100": dict(Et=100, Ep=100, H=100), "odd": dict(Et=12, Ep=10, H=20)}


def _model(shape, T=300, P=200, C=17, dropout=0.0, seed=0, angular=False):
    o = {"T": T, "P": P, "C": C, "angular": int(angular), **shape}
    m = Code2Vec(option_from(o, dropout))
    rng = np.random.default_rng(seed)
    params = random_params(rng, T, P, C, shape["Et"], shape["Ep"], shape["H"])
    if angular:
        params.pop("output_linear.bias")
        params["output_linear"] = params.pop("output_linear.weight")
    m.load_state_dict({k: torch.from_numpy(v) for k, v in params.items()})
    return m.to("cuda:0"), params


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("name", list(SHAPES))
def test_key_by_value_and_by_address_agree(name, packed):
    shape = SHAPES[name]
    m, _ = _model(shape, dropout=0.3)
    T, P, C, B, L = 300, 200, 17, 24, 40
    s, p, e, _ = (cuda(a) for a in random_batch(np.random.default_rng(1), B, L, T, P, C))
    dims = m._dims()
    params = CF.make_params(m.terminal_embedding.weight, m.path_embedding.weight, m.input_linear.weight,
                            m.input_layer_norm.weight, m.input_layer_norm.bias, m.attention_parameter)
    shapes = {k: t.shape for k, t in (("terminal_embedding", m.terminal_embedding.weight),
                                      ("path_embedding", m.path_embedding.weight), ("input_linear", m.input_linear.weight),
                                      ("ln_weight", m.input_layer_norm.weight), ("ln_bias", m.input_layer_norm.bias),
                                      ("attention", m.attention_parameter))}
    key_value = 0x1234_5678_9ABC_DEF1
    key_dev = torch.tensor([key_value], dtype=torch.int64, device="cuda:0")
    bags = None
    if packed:
        n = (s > 0).sum(1).clamp(min=1).cpu().numpy()
        off = np.concatenate([[0], np.cumsum(n)])
        keep = torch.arange(L, device="cuda:0")[None, :] < torch.from_numpy(n).to("cuda:0")[:, None]
        bags = CF.PackedBags(s[keep], p[keep], e[keep], off, L)
    res = []
    for seed in (key_value, key_dev):
        if packed:
            cv, att, xs = CF.encode_forward_packed(dims, params, bags, 0.3, True, seed, stash=True)
        else:
            cv, att, xs = CF.encode_forward(dims, params, s, p, e, 0.3, True, seed, stash=True)
        d_cv = torch.linspace(-1, 1, cv.numel(), device="cuda:0").view_as(cv)
        if packed:
            g = CF.encode_backward_packed(dims, params, bags, cv, att, d_cv, None, shapes, 0.3, True, seed, x_stash=xs)
        else:
            g = CF.encode_backward(dims, params, s, p, e, cv, att, d_cv, None, shapes, 0.3, True, seed, x_stash=xs)
        res.append((cv, att, xs, g))
    torch.cuda.synchronize()
    (cv0, att0, xs0, g0), (cv1, att1, xs1, g1) = res
    assert torch.equal(cv0, cv1) and torch.equal(att0, att1) and torch.equal(xs0, xs1)
    for k in g0:      # LayerNorm / attention gradients are summed with cross-CTA atomics: run-to-run order differs
        torch.testing.assert_close(g0[k], g1[k], rtol=1e-5, atol=1e-6)


def test_capturable_adam():
    lib = _lib.load()
    n = 1003
    gen = torch.Generator(device="cuda:0").manual_seed(0)
    p0 = torch.randn(n, device="cuda:0", generator=gen)
    g = torch.randn(n, device="cuda:0", generator=gen)
    bufs = {k: [p0.clone(), g.clone(), torch.zeros(n, device="cuda:0"), torch.zeros(n, device="cuda:0")] for k in "ab"}
    state = torch.zeros(2, dtype=torch.int64, device="cuda:0")
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    def host_scalars(t, lr, b1, b2):
        lr, b1, b2 = (float(np.float32(x)) for x in (lr, b1, b2))
        return np.array([lr / (1.0 - b1 ** t), 1.0 / np.sqrt(1.0 - b2 ** t)]).astype(np.float32)

    same = 0
    for t in range(1, 21):    # given identical scalars the update is bit-identical to c2v_adam_step's
        a, b = bufs["a"], bufs["b"]
        for x, y in zip(b, a):
            x.copy_(y)
        a[1].copy_(g); b[1].copy_(g)
        _lib.check(lib.c2v_adam_step(*map(P, a), n, 1e-2, 0.9, 0.999, 1e-8, 0.01, t, 1.0, 0, None), "c2v_adam_step")
        _lib.check(lib.c2v_adam_step_capturable(*map(P, b), n, 1e-2, 0.9, 0.999, 1e-8, 0.01, P(state), 1.0, 0, None),
                   "c2v_adam_step_capturable")
        torch.cuda.synchronize()
        dev = state[1:].cpu().numpy().view(np.float32)
        if (dev == host_scalars(t, 1e-2, 0.9, 0.999)).all():
            same += 1
            for x, y in zip(a, b):
                assert torch.equal(x, y), t
    print(f"capturable Adam: {same} of 20 steps with scalars identical to the host formula, all bit-identical")
    assert same >= 1 and int(state[0]) == 20

    # device scalars against the host formula for t = 1 .. 10^5
    steps = 100_000
    dummy = [torch.zeros(4, device="cuda:0") for _ in range(4)]
    report = {}
    for betas in ((0.9, 0.999), (0.5, 0.9), (0.99, 0.9999)):
        st = torch.zeros(2, dtype=torch.int64, device="cuda:0")
        rec = torch.empty(steps, 2, dtype=torch.int64, device="cuda:0")
        for t in range(steps):
            lib.c2v_adam_step_capturable(*map(P, dummy), 4, 1e-3, betas[0], betas[1], 1e-8, 0.0, P(st), 1.0, 0, None)
            rec[t].copy_(st)
        r = rec.cpu().numpy()
        assert (r[:, 0] == np.arange(1, steps + 1)).all()
        dev = r[:, 1].copy().view(np.float32).reshape(steps, 2)
        tt = np.arange(1, steps + 1, dtype=np.float64)
        b1, b2, lr = float(np.float32(betas[0])), float(np.float32(betas[1])), float(np.float32(1e-3))
        host = np.stack([(lr / (1.0 - b1 ** tt)).astype(np.float32), (1.0 / np.sqrt(1.0 - b2 ** tt)).astype(np.float32)], 1)
        ulp = np.abs(dev.view(np.int32).astype(np.int64) - host.view(np.int32).astype(np.int64))
        assert ulp.max() <= 1, (betas, ulp.max())
        report[betas] = int((ulp > 0).sum())
    print("capturable Adam: scalars differing from the host formula (of 2 x 10^5 per betas):", report)

    # the counter advances once per call, eager or replayed
    st = torch.zeros(2, dtype=torch.int64, device="cuda:0")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        lib.c2v_adam_step_capturable(*map(P, dummy), 4, 1e-3, 0.9, 0.999, 1e-8, 0.0, P(st), 1.0, 0,
                                     ctypes.c_void_p(s.cuda_stream))
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        lib.c2v_adam_step_capturable(*map(P, dummy), 4, 1e-3, 0.9, 0.999, 1e-8, 0.0, P(st), 1.0, 0,
                                     ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    assert int(st[0]) == 1                      # capture launches nothing
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    assert int(st[0]) == 4


@pytest.mark.parametrize("name", ["tc128", "odd"])
def test_dropout_parity_at_replayed_step(name):
    """lr = 0: the parameters do not move, so replay j must reproduce oracle.torch_forward with the mask of key
    splitmix64(base + 2 + j) (two eager warm-up forwards drew keys 0 and 1)."""
    from oracle import oracle
    shape = SHAPES[name]
    drop = 0.25
    m, params = _model(shape, dropout=drop)
    m.train().use_device_rng(seed=1234)
    opt = torch.optim.SGD(m.parameters(), lr=0.0)
    T, P, C, B, L = 300, 200, 17, 16, 30
    step = GraphedTrainStep(m, opt, B, L, loss_fn=lambda o, y: F.nll_loss(F.log_softmax(o, dim=1), y))
    rng = np.random.default_rng(5)
    for j in range(5):
        batch = random_batch(rng, B, L, T, P, C)
        loss = step(*(cuda(a) for a in batch))
        if j < 2:
            continue
        key = splitmix64(1234 + j)
        mask = torch.from_numpy(dropout_mask(key, B * L, shape["H"], drop).reshape(B, L, shape["H"]).astype(np.float32))
        ref = {k: torch.from_numpy(v).clone().requires_grad_(True) for k, v in params.items()}
        out, cv, att = oracle.torch_forward(ref, *(torch.from_numpy(a) for a in batch), dropmask=mask)
        rl = F.nll_loss(F.log_softmax(out, dim=1), torch.from_numpy(batch[3]))
        rl.backward()
        torch.cuda.synchronize()
        assert abs(float(loss) - float(rl)) <= 1e-5 * max(1.0, abs(float(rl))), (j, float(loss), float(rl))
        got = dict(m.named_parameters())
        for k, v in ref.items():
            torch.testing.assert_close(got[k].grad.cpu(), v.grad, rtol=1e-3, atol=2e-5, msg=f"{k} at step {j}")


def _items(rng, n, L, T, P, C):
    s = rng.integers(1, T, (n, L)); p = rng.integers(1, P, (n, L)); e = rng.integers(1, T, (n, L))
    cnt = rng.integers(1, L + 1, n)
    for i in range(n):
        s[i, cnt[i]:] = 0; p[i, cnt[i]:] = 0; e[i, cnt[i]:] = 0
    lab = (s[:, 0] + p[:, 0]) % C
    return [torch.tensor(a, dtype=torch.long) for a in (s, p, e, lab)]


@pytest.mark.parametrize("angular", [False, True])
@pytest.mark.parametrize("way", ["torch_adam", "flat_adam", "forward_nll"])
def test_reference_loop_graphed(way, angular):
    """test_dropin_loop_gpu's 25-step loop (batch 32, ragged last batch) through GraphedTrainStep"""
    from oracle import oracle
    E = H = 128
    T, P, C, L, n, bs = 300, 200, 17, 40, 150, 32
    rng = np.random.default_rng(E)
    data = _items(rng, n, L, T, P, C)
    m, params = _model(dict(Et=E, Ep=E, H=H), T, P, C, angular=angular)
    m.train()
    ang = {"margin": 0.5, "inverse_temp": 30.0} if angular else None
    nll = lambda o, y: F.nll_loss(F.log_softmax(o, dim=1), y)
    if way == "flat_adam":
        opt = FlatAdam(FlatGradBucket(m.parameters()), lr=0.01, capturable=True)
        step = GraphedTrainStep(m, opt, bs, L)
    else:
        opt = torch.optim.Adam(m.parameters(), lr=0.01, capturable=True)
        step = GraphedTrainStep(m, opt, bs, L, loss_fn=nll if way == "forward_nll" else None)
    ref = {k: torch.from_numpy(v).clone().requires_grad_(True) for k, v in params.items()}
    ref_opt = torch.optim.Adam(list(ref.values()), lr=0.01)
    losses, ref_losses = [], []
    for epoch in range(5):
        perm = torch.randperm(n, generator=torch.Generator().manual_seed(epoch))
        for i in range(0, n, bs):
            idx = perm[i:i + bs]
            batch = [t[idx] for t in data]
            losses.append(step(*(t.to("cuda:0") for t in batch)))
            ref_opt.zero_grad()
            rp, _, _ = oracle.torch_forward(ref, *batch, angular=ang)
            rl = nll(rp, batch[3])
            rl.backward()
            ref_opt.step()
            ref_losses.append(rl.item())
    losses = [float(x) for x in losses]
    assert len(losses) == 25 and step.graph is not None
    assert np.abs(np.array(losses[:5]) - np.array(ref_losses[:5])).max() <= 2e-4, (losses[:5], ref_losses[:5])
    assert np.abs(np.array(losses) - np.array(ref_losses)).max() <= 2e-2, (losses, ref_losses)


def test_graphed_predict_and_stale_image_guard():
    T, P, C, B, L = 300, 200, 17, 32, 40
    m, _ = _model(SHAPES["tc128"], T, P, C, dropout=0.25)
    rng = np.random.default_rng(3)
    m.eval()
    for k in (None, 5):
        gp = GraphedPredict(m, B, L, k=k)
        for _ in range(4):
            s, p, e, _ = (cuda(a) for a in random_batch(rng, B, L, T, P, C))
            got = gp(s, p, e)
            want = m.predict(s, p, e) if k is None else m.predict_topk(s, p, e, k=k)
            for x, y in zip(got, want):
                assert (x is None and y is None) or torch.equal(x, y)
        assert gp.graph is not None
    # graphed training, then eager predict() must see the new weights
    m.train().use_device_rng(seed=9)
    opt = FlatAdam(FlatGradBucket(m.parameters()), lr=0.05, capturable=True)
    step = GraphedTrainStep(m, opt, B, L)
    for _ in range(6):
        step(*(cuda(a) for a in random_batch(rng, B, L, T, P, C)))
    m.eval()
    s, p, e, _ = (cuda(a) for a in random_batch(rng, B, L, T, P, C))
    got = m.predict(s, p, e)
    fresh = Code2Vec(m.option).to("cuda:0")
    fresh.load_state_dict(m.state_dict())
    want = fresh.eval().predict(s, p, e)
    for x, y in zip(got, want):
        assert torch.equal(x, y)
    assert opt.step_count() == 6


def test_deferred_index_error_after_replay():
    T, P, C, B, L = 300, 200, 17, 16, 20
    m, _ = _model(SHAPES["tc128"], T, P, C)
    m.train()
    opt = FlatAdam(FlatGradBucket(m.parameters()), lr=0.0, capturable=True)
    step = GraphedTrainStep(m, opt, B, L)
    rng = np.random.default_rng(4)
    for _ in range(4):
        step(*(cuda(a) for a in random_batch(rng, B, L, T, P, C)))
    bad = [cuda(a) for a in random_batch(rng, B, L, T, P, C)]
    bad[0][3, 0] = T + 11                           # clamped to row 0 and counted by the replayed finalize kernel
    step(*bad)
    torch.cuda.synchronize()
    with pytest.raises(IndexError):
        step(*(cuda(a) for a in random_batch(rng, B, L, T, P, C)))
    step(*(cuda(a) for a in random_batch(rng, B, L, T, P, C)))      # consumed


def test_capture_errors_and_steady_state_memory():
    T, P, C, B, L = 300, 200, 17, 16, 20
    m, _ = _model(SHAPES["tc100"], T, P, C, dropout=0.25)
    m.train()
    rng = np.random.default_rng(6)
    batch = [cuda(a) for a in random_batch(rng, B, L, T, P, C)]
    # dropout without device keys, and a non-capturable FlatAdam, refuse to be captured
    m.forward_loss(*batch)
    g = torch.cuda.CUDAGraph()
    with pytest.raises(RuntimeError, match="use_device_rng"):
        with torch.cuda.graph(g):
            m.forward_loss(*batch)
    opt = FlatAdam(FlatGradBucket(m.parameters()))
    opt.step()
    with pytest.raises(RuntimeError, match="capturable=True"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            opt.step()
    with pytest.raises(RuntimeError, match="check_indices"):
        with torch.cuda.graph(torch.cuda.CUDAGraph()):
            m.check_indices()
    torch.cuda.synchronize()

    m2, _ = _model(SHAPES["tc100"], T, P, C, dropout=0.25)
    m2.train().use_device_rng(seed=1)
    step = GraphedTrainStep(m2, FlatAdam(FlatGradBucket(m2.parameters()), lr=1e-3, capturable=True), B, L)
    for _ in range(4):
        step(*batch)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    for _ in range(20):
        step(*batch)
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == before
    step.optimizer.lr = 2e-3
    with pytest.raises(RuntimeError, match="changed since the capture"):
        step(*batch)

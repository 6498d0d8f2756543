"""CPU-side checks of the CUDA-graph support: the argument errors of C2V_DROPOUT_SEED_ON_DEVICE, c2v_next_dropout_key and
c2v_adam_step_capturable return C2V_EINVAL before any CUDA call (without a GPU a CUDA call would return C2V_ECUDA), a
numpy restatement of the key sequence, and the Python-side errors that need no device."""
import ctypes

import numpy as np
import pytest
import torch

from code2vec_b200 import _lib
from code2vec_b200 import functional as CF
from code2vec_b200.distributed import FlatAdam, FlatGradBucket, ShardedFlatAdam
from code2vec_b200.graphs import GraphedPredict, GraphedTrainStep
from code2vec_b200.model import Code2Vec

V = ctypes.c_void_p
FAKE = V(0x1000)          # never dereferenced: every call below fails its argument checks first
ODD = V(0x1004)           # 4-byte aligned, not 8-byte aligned
M64 = (1 << 64) - 1


def splitmix64(x):
    """the key c2v_next_dropout_key writes for the state {base, counter}: splitmix64(base + counter), numpy uint64"""
    with np.errstate(over="ignore"):
        z = np.uint64(x) + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return int(z ^ (z >> np.uint64(31)))


def _splitmix64_int(x):
    z = (x + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def test_splitmix64_restatement():
    # the first output of SplitMix64 seeded with 0 (the published reference value)
    assert splitmix64(0) == 0xE220A8397B1DCDAF
    rng = np.random.default_rng(7)
    for x in [1, 2 ** 62 - 1, M64, M64 - 5] + [int(v) for v in rng.integers(0, 2 ** 63, 50, dtype=np.int64)]:
        assert splitmix64(x) == _splitmix64_int(x)


def _expect_einval(rc, name):
    assert rc == _lib.C2V_EINVAL
    msg = _lib.load().c2v_last_error()
    assert msg and name.encode() in msg, msg


def _dims():
    return CF.make_dims(100, 100, 10, 16, 16, 128)


def _params():
    return _lib.Params(*([FAKE] * 8))


DROP_BAD = {"device key, NULL address": (3, 0), "device key, flag only, NULL": (2, 0),
            "device key, misaligned": (3, 0x1004), "unknown bit 2": (5, 7), "unknown high bit": (1 | (1 << 30), 7),
            "negative": (-1, 7)}


@pytest.mark.parametrize("case", list(DROP_BAD))
@pytest.mark.parametrize("entry", ["forward", "forward_packed", "backward", "backward_packed", "backward_sparse"])
def test_dropout_flags_rejected(case, entry):
    training, seed = DROP_BAD[case]
    lib = _lib.load()
    d, p = _dims(), _params()
    drop = _lib.Dropout(0.25, training, seed)
    B, L, N = 4, 8, 20
    grads = _lib.Grads(*([FAKE] * 6))
    slots = _lib.RowSlots(None, None)
    bd, bp, bdr, bg = ctypes.byref(d), ctypes.byref(p), ctypes.byref(drop), ctypes.byref(grads)
    if entry == "forward":
        rc = lib.c2v_encode_forward_stash(bd, bp, FAKE, FAKE, FAKE, B, L, bdr, FAKE, FAKE, None, FAKE, 1 << 40, 0, None)
        name = "c2v_encode_forward"
    elif entry == "forward_packed":
        rc = lib.c2v_encode_forward_packed(bd, bp, FAKE, FAKE, FAKE, FAKE, B, N, L, bdr, FAKE, FAKE, None, FAKE, 1 << 40, 0,
                                           None)
        name = "c2v_encode_forward_packed"
    elif entry == "backward":
        rc = lib.c2v_encode_backward_phased(bd, bp, FAKE, FAKE, FAKE, B, L, bdr, FAKE, FAKE, None, FAKE, None, bg, FAKE,
                                            1 << 40, 0, None)
        name = "c2v_encode_backward"
    elif entry == "backward_packed":
        rc = lib.c2v_encode_backward_packed(bd, bp, FAKE, FAKE, FAKE, FAKE, B, N, L, bdr, FAKE, FAKE, None, FAKE, None, bg,
                                            FAKE, 1 << 40, 0, None)
        name = "c2v_encode_backward"
    else:
        rc = lib.c2v_encode_backward_sparse(bd, bp, FAKE, FAKE, FAKE, B, L, bdr, FAKE, FAKE, None, FAKE, None, bg,
                                            ctypes.byref(slots), FAKE, 1 << 40, 0, None)
        name = "c2v_encode_backward"
    _expect_einval(rc, name)


@pytest.mark.parametrize("state,key", [(None, FAKE), (FAKE, None), (ODD, FAKE), (FAKE, ODD)])
def test_next_dropout_key_rejects_bad_pointers(state, key):
    _expect_einval(_lib.load().c2v_next_dropout_key(state, key, None), "c2v_next_dropout_key")


def _capturable(p=FAKE, g=FAKE, m=FAKE, v=FAKE, n=100, state=FAKE):
    return _lib.load().c2v_adam_step_capturable(p, g, m, v, n, 1e-3, 0.9, 0.999, 1e-8, 0.0, state, 1.0, 1, None)


CAPTURABLE_BAD = {"param": dict(p=None), "grad": dict(g=None), "exp_avg": dict(m=None), "exp_avg_sq": dict(v=None),
                  "n<1": dict(n=0), "misaligned param": dict(p=V(0x1008)), "misaligned exp_avg_sq": dict(v=V(0x1004)),
                  "NULL step_state": dict(state=None), "misaligned step_state": dict(state=ODD),
                  "step_state off by 1": dict(state=V(0x1001))}


@pytest.mark.parametrize("case", list(CAPTURABLE_BAD))
def test_adam_step_capturable_rejects_bad_arguments(case):
    _expect_einval(_capturable(**CAPTURABLE_BAD[case]), "c2v_adam_step_capturable")


# ---- Python-side errors -------------------------------------------------------------------------------------------------
class _Opt:
    terminal_count, path_count, label_count = 50, 60, 7
    terminal_embed_size = path_embed_size = 8
    encode_size = 16
    dropout_prob = 0.25
    angular_margin_loss = False
    angular_margin, inverse_temp = 0.5, 30.0


def _model(dropout=0.25):
    o = _Opt()
    o.dropout_prob = dropout
    return Code2Vec(o)


def test_graphed_step_needs_capturable_flat_adam():
    m = _model(0.0)
    opt = FlatAdam(FlatGradBucket(m.parameters()))
    with pytest.raises(ValueError, match="capturable=True"):
        GraphedTrainStep(m, opt, 4, 8)


def test_graphed_step_needs_device_rng_with_dropout():
    m = _model(0.25).train()
    opt = FlatAdam(FlatGradBucket(m.parameters()))
    opt.capturable = True            # (a device step state is not needed to reach the check)
    with pytest.raises(RuntimeError, match="use_device_rng"):
        GraphedTrainStep(m, opt, 4, 8)
    m.use_device_rng(seed=5)
    GraphedTrainStep(m, opt, 4, 8)
    GraphedTrainStep(_model(0.25).eval(), torch.optim.Adam(m.parameters()), 4, 8)   # eval: no dropout, no key


def test_graphed_step_rejects_sparse_tables():
    m = _model(0.0)
    m.terminal_embedding.sparse = True
    with pytest.raises(NotImplementedError, match="sparse"):
        GraphedTrainStep(m, torch.optim.Adam(m.parameters()), 4, 8)


def test_graphed_calls_reject_packed_bags():
    m = _model(0.0)
    z = torch.zeros(5, dtype=torch.int64)
    bags = CF.PackedBags(z, z, z, [0, 2, 5], 8)
    with pytest.raises(TypeError, match="PackedBags"):
        GraphedTrainStep(m, torch.optim.Adam(m.parameters()), 2, 8)(bags, None, None, torch.zeros(2, dtype=torch.int64))
    with pytest.raises(TypeError, match="PackedBags"):
        GraphedPredict(m, 2, 8)(bags, None, None)


def test_sharded_capturable_needs_world_one(monkeypatch):
    import torch.distributed as dist
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
    monkeypatch.setattr(dist, "get_rank", lambda group=None: 0)
    m = _model(0.0)
    with pytest.raises(NotImplementedError, match="one process"):
        ShardedFlatAdam(m.parameters(), capturable=True)


def test_use_device_rng_base_from_torch_generator():
    torch.manual_seed(3)
    a = _model().use_device_rng()._rng_base
    torch.manual_seed(3)
    b = _model().use_device_rng()._rng_base
    assert a == b and _model().use_device_rng(seed=11)._rng_base == 11

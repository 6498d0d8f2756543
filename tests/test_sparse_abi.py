"""CPU-side checks of the sparse embedding gradients (c2v_sparse_rows, c2v_encode_backward_sparse,
c2v_encode_backward_packed_sparse, c2v_sparse_adam_step, distributed.FusedSparseAdam): every argument error returns its
code and message before any CUDA call, the workspace sizes, and FusedSparseAdam's state_dict interchanging with
torch.optim.SparseAdam's."""
import ctypes

import pytest
import torch

from code2vec_b200 import _lib
from code2vec_b200 import functional as CF
from code2vec_b200.distributed import FusedSparseAdam

V = ctypes.c_void_p
FAKE = V(0x1000)          # never dereferenced: every call below fails its argument checks first
BIG = 1 << 40


def _expect(rc, code, name):
    assert rc == code
    msg = _lib.load().c2v_last_error()
    assert msg and name.encode() in msg, msg


def _rows(ia=FAKE, na=10, ib=FAKE, nb=10, vocab=1000, slot=FAKE, rows=FAKE, count=FAKE, ws=FAKE, ws_bytes=BIG):
    return _lib.load().c2v_sparse_rows(ia, na, ib, nb, vocab, slot, rows, count, ws, ws_bytes, None)


ROWS_BAD = {"vocab<1": dict(vocab=0), "vocab>=2^31": dict(vocab=1 << 31), "n_a<0": dict(na=-1), "n_b<0": dict(nb=-1),
            "idx_a": dict(ia=None), "idx_b": dict(ib=None), "slot": dict(slot=None), "rows": dict(rows=None),
            "count": dict(count=None), "workspace": dict(ws=None), "misaligned idx": dict(ia=V(0x1004)),
            "misaligned slot": dict(slot=V(0x1002)), "misaligned rows": dict(rows=V(0x1004)),
            "misaligned count": dict(count=V(0x1004)), "misaligned workspace": dict(ws=V(0x1008))}


@pytest.mark.parametrize("case", list(ROWS_BAD))
def test_sparse_rows_rejects_bad_arguments(case):
    _expect(_rows(**ROWS_BAD[case]), _lib.C2V_EINVAL, "c2v_sparse_rows")


def test_sparse_rows_workspace():
    lib = _lib.load()
    assert lib.c2v_sparse_rows_workspace_bytes(0) == 0
    assert lib.c2v_sparse_rows_workspace_bytes(1 << 31) == 0
    assert lib.c2v_sparse_rows_workspace_bytes(1) == 8192 + 256                    # one chunk of flags + its count
    assert lib.c2v_sparse_rows_workspace_bytes(8192) == 8192 + 256
    assert lib.c2v_sparse_rows_workspace_bytes(8193) == 2 * 8192 + 256
    n = (1 << 31) - 1
    chunks = (n + 8191) // 8192
    assert lib.c2v_sparse_rows_workspace_bytes(n) == chunks * 8192 + (chunks * 8 + 255) // 256 * 256
    need = lib.c2v_sparse_rows_workspace_bytes(1000)
    _expect(_rows(ws_bytes=need - 1), _lib.C2V_EWORKSPACE, "c2v_sparse_rows")
    # empty index lists need no index or rows pointers (the call then fails only on its workspace, before any CUDA call)
    _expect(_rows(ia=None, na=0, ib=None, nb=0, rows=None, ws_bytes=need - 1), _lib.C2V_EWORKSPACE, "c2v_sparse_rows")


def test_sparse_rows_wrapper_rejects_bad_inputs():
    with pytest.raises(TypeError):
        CF.sparse_rows([torch.zeros(3, dtype=torch.int32)], 10)
    with pytest.raises(ValueError):
        CF.sparse_rows([], 10)


def _dims(T=1000, P=900, C=10, E=128, H=128):
    return CF.make_dims(T, P, C, E, E, H)


def _backward(packed, dims=None, slots=None, grads=None, **kw):
    lib = _lib.load()
    d = dims or _dims()
    p = _lib.Params(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE, None, None)
    g = grads or _lib.Grads(FAKE, FAKE, FAKE, FAKE, FAKE, FAKE)
    sl = slots if slots is not None else _lib.RowSlots(FAKE, None)
    sl_arg = None if kw.get("null_slots") else ctypes.byref(sl)
    drop = _lib.Dropout(0.0, 0, 0)
    B, L, N = kw.get("B", 4), kw.get("L", 8), kw.get("N", 20)
    ws, ws_bytes, phase = kw.get("ws", FAKE), kw.get("ws_bytes", BIG), kw.get("phase", 0)
    if packed:
        return lib.c2v_encode_backward_packed_sparse(ctypes.byref(d), ctypes.byref(p), FAKE, FAKE, FAKE, FAKE, B, N, L,
                                                     ctypes.byref(drop), FAKE, FAKE, None, FAKE, None, ctypes.byref(g),
                                                     sl_arg, ws, ws_bytes, phase, None)
    return lib.c2v_encode_backward_sparse(ctypes.byref(d), ctypes.byref(p), FAKE, FAKE, FAKE, B, L, ctypes.byref(drop),
                                          FAKE, FAKE, None, FAKE, None, ctypes.byref(g), sl_arg, ws, ws_bytes, phase, None)


BACKWARD_BAD = {"phase": dict(phase=3), "B<1": dict(B=0), "workspace": dict(ws=None), "slots NULL": dict(null_slots=True),
                "misaligned slot": dict(slots=_lib.RowSlots(V(0x1002), None)),
                "misaligned values": dict(grads=_lib.Grads(V(0x1008), FAKE, FAKE, FAKE, FAKE, FAKE))}


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("case", list(BACKWARD_BAD))
def test_encode_backward_sparse_rejects_bad_arguments(packed, case):
    name = "c2v_encode_backward_packed_sparse" if packed else "c2v_encode_backward_sparse"
    _expect(_backward(packed, **BACKWARD_BAD[case]), _lib.C2V_EINVAL, name)


@pytest.mark.parametrize("packed", [False, True])
def test_encode_backward_sparse_checks_shapes_and_workspace(packed):
    lib = _lib.load()
    assert _backward(packed, dims=_dims(T=0)) == _lib.C2V_EINVAL                   # dims_ok
    if packed:
        _expect(_backward(True, N=2), _lib.C2V_EINVAL, "c2v_encode_backward_packed_sparse")       # N < B
    # a dense table (NULL slot map) may have any alignment: only the compact buffers are checked
    sl = _lib.RowSlots(None, FAKE)
    g = _lib.Grads(V(0x1004), FAKE, FAKE, FAKE, FAKE, FAKE)
    d = _dims()
    need = (lib.c2v_encode_backward_packed_workspace_bytes(ctypes.byref(d), 4, 20) if packed
            else lib.c2v_encode_backward_workspace_bytes(ctypes.byref(d), 4, 8))
    assert need > 0
    rc = _backward(packed, slots=sl, grads=g, ws_bytes=need - 1)
    assert rc == _lib.C2V_EWORKSPACE, _lib.load().c2v_last_error()


def _adam(p=FAKE, m=FAKE, v=FAKE, g=FAKE, rows=FAKE, U=10, n=100, E=128, lr=1e-3, b1=0.9, b2=0.999, eps=1e-8, step=1):
    return _lib.load().c2v_sparse_adam_step(p, m, v, g, rows, U, n, E, lr, b1, b2, eps, step, None)


ADAM_BAD = {"U<0": dict(U=-1), "n_rows<1": dict(n=0), "E<1": dict(E=0), "E>65536": dict(E=65537), "step<1": dict(step=0),
            "param": dict(p=None), "exp_avg": dict(m=None), "exp_avg_sq": dict(v=None), "values": dict(g=None),
            "rows": dict(rows=None), "misaligned param": dict(p=V(0x1001)), "misaligned rows": dict(rows=V(0x1004))}


@pytest.mark.parametrize("case", list(ADAM_BAD))
def test_sparse_adam_step_rejects_bad_arguments(case):
    _expect(_adam(**ADAM_BAD[case]), _lib.C2V_EINVAL, "c2v_sparse_adam_step")


def test_sparse_adam_step_empty_gradient_is_a_no_op():
    assert _adam(g=None, rows=None, U=0) == _lib.C2V_OK                    # nothing to do: no CUDA call either


def test_fused_sparse_adam_state_dict_interchanges_with_torch():
    torch.manual_seed(0)
    w = [torch.nn.Parameter(torch.randn(6, 3)), torch.nn.Parameter(torch.randn(5, 2))]
    kw = dict(lr=3e-3, betas=(0.8, 0.99), eps=1e-6)
    ref = torch.optim.SparseAdam(w, **kw)
    for p in w:                                        # one torch step on the CPU: state with step, exp_avg, exp_avg_sq
        p.grad = torch.sparse_coo_tensor(torch.tensor([[0, 2]]), torch.randn(2, p.shape[1]), p.shape)
    ref.step()
    fused = FusedSparseAdam(w, lr=1.0)
    fused.load_state_dict(ref.state_dict())
    sd, rd = fused.state_dict(), ref.state_dict()
    assert sd["param_groups"] == rd["param_groups"]
    for k in rd["state"]:
        assert sd["state"][k]["step"] == rd["state"][k]["step"] == 1
        for name in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(sd["state"][k][name], rd["state"][k][name])
    back = torch.optim.SparseAdam(w, lr=1.0)
    back.load_state_dict(fused.state_dict())
    assert back.state_dict()["param_groups"] == rd["param_groups"]
    assert isinstance(fused, torch.optim.SparseAdam)


def test_fused_sparse_adam_validation_is_torchs():
    p = torch.nn.Parameter(torch.randn(4, 2))
    with pytest.raises(ValueError):
        FusedSparseAdam([p], lr=-1.0)
    with pytest.raises(ValueError):
        FusedSparseAdam([p], betas=(1.0, 0.9))
    opt = FusedSparseAdam([p])
    p.grad = torch.randn(4, 2)
    with pytest.raises(RuntimeError, match="dense gradients"):
        opt.step()

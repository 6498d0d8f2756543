"""CPU-side checks of the data-parallel sparse step's entry points (c2v_sparse_union_rows, c2v_sparse_adam_step_merged):
every argument error returns its code and message before any CUDA call, and the workspace sizes."""
import ctypes

import pytest
import torch

from code2vec_b200 import _lib
from code2vec_b200 import functional as CF

V = ctypes.c_void_p
FAKE = V(0x1000)          # never dereferenced: every call below fails its argument checks first
BIG = 1 << 40


def _expect(rc, code, name):
    assert rc == code
    msg = _lib.load().c2v_last_error()
    assert msg and name.encode() in msg, msg


def _union(rows=FAKE, counts=FAKE, world=4, u_max=10, vocab=1000, out=FAKE, count=FAKE, ws=FAKE, ws_bytes=BIG):
    return _lib.load().c2v_sparse_union_rows(rows, counts, world, u_max, vocab, out, count, ws, ws_bytes, None)


UNION_BAD = {"vocab<1": dict(vocab=0), "vocab>=2^31": dict(vocab=1 << 31), "world<1": dict(world=0),
             "world>1024": dict(world=1025), "u_max<0": dict(u_max=-1), "u_max>vocab": dict(u_max=1001),
             "rows": dict(rows=None), "counts": dict(counts=None), "union_rows": dict(out=None),
             "union_count": dict(count=None), "workspace": dict(ws=None), "misaligned rows": dict(rows=V(0x1004)),
             "misaligned counts": dict(counts=V(0x1004)), "misaligned union_rows": dict(out=V(0x1004)),
             "misaligned union_count": dict(count=V(0x1002)), "misaligned workspace": dict(ws=V(0x1008))}


@pytest.mark.parametrize("case", list(UNION_BAD))
def test_sparse_union_rows_rejects_bad_arguments(case):
    _expect(_union(**UNION_BAD[case]), _lib.C2V_EINVAL, "c2v_sparse_union_rows")


def test_sparse_union_rows_workspace():
    lib = _lib.load()
    assert lib.c2v_sparse_union_rows_workspace_bytes(0) == 0
    assert lib.c2v_sparse_union_rows_workspace_bytes(1 << 31) == 0
    for vocab in (1, 8192, 8193, 2 * 10**6, (1 << 31) - 1):
        # the workspace of c2v_sparse_rows, then the slot map [vocab] int32 that its compact pass writes
        slot = (4 * vocab + 255) // 256 * 256
        assert lib.c2v_sparse_union_rows_workspace_bytes(vocab) == lib.c2v_sparse_rows_workspace_bytes(vocab) + slot
    need = lib.c2v_sparse_union_rows_workspace_bytes(1000)
    _expect(_union(ws_bytes=need - 1), _lib.C2V_EWORKSPACE, "c2v_sparse_union_rows")
    # empty lists (u_max 0) need no rows or union_rows pointers
    _expect(_union(rows=None, u_max=0, out=None, ws_bytes=need - 1), _lib.C2V_EWORKSPACE, "c2v_sparse_union_rows")


def _merged(p=FAKE, m=FAKE, v=FAKE, g=FAKE, rows=FAKE, counts=FAKE, world=4, u_max=10, union=FAKE, count=FAKE, n=100,
            E=128, scale=0.25, lr=1e-3, b1=0.9, b2=0.999, eps=1e-8, step=1):
    return _lib.load().c2v_sparse_adam_step_merged(p, m, v, g, rows, counts, world, u_max, union, count, n, E, scale, lr, b1,
                                                   b2, eps, step, None)


MERGED_BAD = {"world<1": dict(world=0), "world>1024": dict(world=1025), "u_max<0": dict(u_max=-1),
              "u_max>n_rows": dict(u_max=101), "n_rows<1": dict(n=0, u_max=0), "n_rows>=2^31": dict(n=1 << 31),
              "E<1": dict(E=0), "E>65536": dict(E=65537), "step<1": dict(step=0), "param": dict(p=None),
              "exp_avg": dict(m=None), "exp_avg_sq": dict(v=None), "values": dict(g=None), "rows": dict(rows=None),
              "counts": dict(counts=None), "union_rows": dict(union=None), "union_count": dict(count=None),
              "misaligned param": dict(p=V(0x1001)), "misaligned values": dict(g=V(0x1002)),
              "misaligned rows": dict(rows=V(0x1004)), "misaligned counts": dict(counts=V(0x1004)),
              "misaligned union_rows": dict(union=V(0x1004)), "misaligned union_count": dict(count=V(0x1004))}


@pytest.mark.parametrize("case", list(MERGED_BAD))
def test_sparse_adam_step_merged_rejects_bad_arguments(case):
    _expect(_merged(**MERGED_BAD[case]), _lib.C2V_EINVAL, "c2v_sparse_adam_step_merged")


def test_sparse_adam_step_merged_with_empty_lists_is_a_no_op():
    # u_max 0: nothing to merge, no CUDA call; the lists' pointers may be NULL
    assert _merged(g=None, rows=None, union=None, u_max=0) == _lib.C2V_OK


def test_wrappers_reject_bad_inputs():
    rows, counts = torch.zeros(2, 3, dtype=torch.int64), torch.zeros(2, dtype=torch.int64)
    with pytest.raises(TypeError):
        CF.sparse_union_rows(rows.int(), counts, 10)
    with pytest.raises(ValueError):
        CF.sparse_union_rows(rows, torch.zeros(3, dtype=torch.int64), 10)
    with pytest.raises(ValueError):
        CF.sparse_union_rows(rows[0], counts, 10)
    with pytest.raises(_lib.C2VError, match="CUDA"):            # no CPU fallback
        CF.sparse_union_rows(rows, counts, 10)

"""CPU-side checks of the dense Adam entry points (c2v_adam_step, c2v_adam_step_sharded, c2v_adam_step_sharded_bulk):
every argument error returns C2V_EINVAL with the function's name in c2v_last_error() before any CUDA call (on a machine
without a GPU a CUDA call would return C2V_ECUDA instead), and an empty bulk slice is a no-op."""
import ctypes

import pytest
import torch

from code2vec_b200 import _lib

V = ctypes.c_void_p
FAKE = V(0x1000)          # never dereferenced: every call below fails its argument checks first
ODD = V(0x1004)           # 4-byte aligned, not 16-byte aligned
WORLD = 4


def _expect_einval(rc, name):
    assert rc == _lib.C2V_EINVAL
    msg = _lib.load().c2v_last_error()
    assert msg and name.encode() in msg, msg


def _table(entries, size=17):
    """a peer pointer table with room for 17 entries, so that a world the checks should have refused reads nothing
    beyond it"""
    t = (V * size)(*([FAKE] * size))
    for i, e in entries.items():
        t[i] = e
    return t


def _flat(p=FAKE, g=FAKE, m=FAKE, v=FAKE, n=100, step=1):
    return _lib.load().c2v_adam_step(p, g, m, v, n, 1e-3, 0.9, 0.999, 1e-8, 0.0, step, 1.0, 1, None)


FLAT_BAD = {"param": dict(p=None), "grad": dict(g=None), "exp_avg": dict(m=None), "exp_avg_sq": dict(v=None),
            "n<1": dict(n=0), "n<0": dict(n=-4), "step<1": dict(step=0), "step<0": dict(step=-1),
            "misaligned param": dict(p=ODD), "misaligned grad": dict(g=ODD), "misaligned exp_avg": dict(m=ODD),
            "misaligned exp_avg_sq": dict(v=ODD)}


@pytest.mark.parametrize("case", list(FLAT_BAD))
def test_adam_step_rejects_bad_arguments(case):
    _expect_einval(_flat(**FLAT_BAD[case]), "c2v_adam_step")


def _sharded(p=FAKE, pmc=None, gmc=None, pp=None, gp=None, world=WORLD, m=FAKE, v=FAKE, begin=0, n=64, z=FAKE, zn=64,
             step=1, tables=True):
    if tables:
        pp = _table(pp or {})
        gp = _table(gp or {})
    return _lib.load().c2v_adam_step_sharded(p, pmc, gmc, pp, gp, world, m, v, begin, n, z, zn, 1e-3, 0.9, 0.999, 1e-8,
                                             0.0, step, 0.25, None)


SHARDED_BAD = {
    "param_local": dict(p=None), "exp_avg": dict(m=None), "exp_avg_sq": dict(v=None),
    "no multicast, no peer tables": dict(tables=False),
    "param multicast only": dict(pmc=FAKE, tables=False), "grad multicast only": dict(gmc=FAKE, tables=False),
    "NULL param peer": dict(pp={2: None}), "NULL grad peer": dict(gp={WORLD - 1: None}),
    "NULL param peer 0": dict(pp={0: None}),
    "world 0": dict(world=0), "world 17": dict(world=17), "world<0": dict(world=-1),
    "slice_begin % 4": dict(begin=6), "slice_n % 4": dict(n=66), "zero_n % 4": dict(zn=2),
    "slice_begin<0": dict(begin=-4), "slice_n<0": dict(n=-4), "step<1": dict(step=0),
    "misaligned param_local": dict(p=ODD), "misaligned exp_avg": dict(m=ODD), "misaligned exp_avg_sq": dict(v=ODD),
    "misaligned zero buffer": dict(z=ODD), "misaligned param peer": dict(pp={1: ODD}),
    "misaligned grad peer": dict(gp={WORLD - 1: ODD}),
    "misaligned param multicast": dict(pmc=ODD, gmc=FAKE, tables=False),
    "misaligned grad multicast": dict(pmc=FAKE, gmc=ODD, tables=False),
}


@pytest.mark.parametrize("case", list(SHARDED_BAD))
def test_adam_step_sharded_rejects_bad_arguments(case):
    _expect_einval(_sharded(**SHARDED_BAD[case]), "c2v_adam_step_sharded")


def _bulk(p=FAKE, pp=None, gp=None, world=WORLD, m=FAKE, v=FAKE, begin=0, n=64, step=1, ctas=0, tables=(True, True)):
    pt = _table(pp or {}) if tables[0] else None
    gt = _table(gp or {}) if tables[1] else None
    return _lib.load().c2v_adam_step_sharded_bulk(p, pt, gt, world, m, v, begin, n, 1e-3, 0.9, 0.999, 1e-8, 0.0, step,
                                                  0.25, ctas, None)


BULK_BAD = {
    "param_local": dict(p=None), "exp_avg": dict(m=None), "exp_avg_sq": dict(v=None),
    "param peer table": dict(tables=(False, True)), "grad peer table": dict(tables=(True, False)),
    "NULL param peer": dict(pp={3: None}), "NULL grad peer": dict(gp={0: None}),
    "world 0": dict(world=0), "world 17": dict(world=17),
    "slice_begin % 4": dict(begin=2), "slice_n % 4": dict(n=65), "slice_begin<0": dict(begin=-4),
    "slice_n<0": dict(n=-4), "step<1": dict(step=0),
    "misaligned param_local": dict(p=ODD), "misaligned exp_avg": dict(m=ODD), "misaligned exp_avg_sq": dict(v=ODD),
    "misaligned param peer": dict(pp={WORLD - 1: ODD}), "misaligned grad peer": dict(gp={1: ODD}),
    # an empty slice is checked like any other
    "empty slice, NULL peer": dict(n=0, gp={2: None}), "empty slice, misaligned": dict(n=0, m=ODD),
}


@pytest.mark.parametrize("case", list(BULK_BAD))
def test_adam_step_sharded_bulk_rejects_bad_arguments(case):
    _expect_einval(_bulk(**BULK_BAD[case]), "c2v_adam_step_sharded_bulk")


def test_adam_step_sharded_bulk_empty_slice_is_a_no_op():
    # real (host) buffers rather than made-up addresses; an empty slice launches nothing and makes no CUDA call
    bufs = [torch.full((16,), 7.0) for _ in range(2 + 2 * WORLD + 1)]
    before = [b.clone() for b in bufs]
    ptr = [V(b.data_ptr()) for b in bufs]
    assert all(b.data_ptr() % 16 == 0 for b in bufs)
    pt = (V * WORLD)(*ptr[2:2 + WORLD])
    gt = (V * WORLD)(*ptr[2 + WORLD:2 + 2 * WORLD])
    rc = _lib.load().c2v_adam_step_sharded_bulk(ptr[-1], pt, gt, WORLD, ptr[0], ptr[1], 8, 0, 1e-3, 0.9, 0.999, 1e-8,
                                                0.0, 1, 0.25, 0, None)
    assert rc == _lib.C2V_OK, _lib.load().c2v_last_error()
    assert all(torch.equal(a, b) for a, b in zip(bufs, before))

"""CPU-side checks of the packed variable-name builder, the per-unit context count and the packed host-buffer calls:
argument checks before any CUDA call, and `unit_counts`, the numpy restatement of c2v_count_unit_contexts, pinned to the
reference builder's output."""
import ctypes
import os

import numpy as np
import pytest

from code2vec_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GV = np.load(os.path.join(ROOT, "tests", "golden", "builder_vars.npz"))
X = ctypes.c_void_p(16)                              # a stand-in device pointer: every call below fails its checks first


def unit_counts(offsets, contexts, unit_item, unit_var):
    """int64 [n_units]: the contexts of item unit_item[u] whose start or end is unit_var[u] (0 for an unknown item) --
    the number of contexts unit u's variable-name bag draws from before truncation to max_path_length."""
    offsets, contexts = np.asarray(offsets, np.int64), np.asarray(contexts)
    out = np.zeros(len(unit_item), np.int64)
    for u, (item, v) in enumerate(zip(np.asarray(unit_item, np.int64), np.asarray(unit_var, np.int64))):
        if 0 <= item < len(offsets) - 1:
            c = contexts[offsets[item]:offsets[item + 1]]
            out[u] = int(((c[:, 0] == v) | (c[:, 2] == v)).sum())
    return out


def _err():
    return _lib.load().c2v_last_error().decode()


def test_unit_counts_match_the_reference_builder():
    """min(count, L) is the length of the reference's bag (its paths are never 0) for every unit of the real sample"""
    units, L = GV["real_units"], int(GV["real_L"])
    n = unit_counts(GV["real_offsets"], GV["real_contexts"], units[:, 0], units[:, 1])
    assert np.array_equal(np.minimum(n, L), (GV["real_ref_paths"] != 0).sum(1))
    assert (n > L).any() and (n < L).any()
    assert unit_counts(GV["real_offsets"], GV["real_contexts"], [-1, 48], [5, 5]).tolist() == [0, 0]


def test_count_unit_contexts_rejects_bad_arguments():
    lib = _lib.load()
    args = dict(offsets=X, contexts=X, n_items=5, unit_item=X, unit_var=X, n_units=3, counts=X)
    for bad in ({"offsets": None}, {"contexts": None}, {"unit_item": None}, {"unit_var": None}, {"counts": None},
                {"n_items": 0}, {"n_units": 0}):
        a = {**args, **bad}
        rc = lib.c2v_count_unit_contexts(a["offsets"], a["contexts"], a["n_items"], a["unit_item"], a["unit_var"],
                                         a["n_units"], a["counts"], None)
        assert rc == _lib.C2V_EINVAL, bad
        assert "c2v_count_unit_contexts: bad argument" in _err()


def _vars_packed(**kw):
    a = dict(offsets=X, contexts=X, n_items=5, unit_item=X, unit_var=X, n_units=3, ids=X, B=4, L=7, n_vars=2,
             shuffle=0, bag_off=X, starts=X, paths=X, ends=X)
    a.update(kw)
    return _lib.load().c2v_build_batch_vars_packed(a["offsets"], a["contexts"], a["n_items"], a["unit_item"], a["unit_var"],
                                                   None, a["n_units"], a["ids"], a["B"], a["L"], 0, 1, X, 100, X,
                                                   a["n_vars"], a["shuffle"], a["bag_off"], a["starts"], a["paths"],
                                                   a["ends"], None, None)


@pytest.mark.parametrize("bad", [{"offsets": None}, {"contexts": None}, {"unit_item": None}, {"unit_var": None},
                                 {"ids": None}, {"bag_off": None}, {"starts": None}, {"paths": None}, {"ends": None},
                                 {"n_items": 0}, {"n_units": 0}, {"B": 0}, {"L": 0}])
def test_build_batch_vars_packed_rejects_bad_arguments(bad):
    assert _vars_packed(**bad) == _lib.C2V_EINVAL
    assert "c2v_build_batch_vars_packed: bad argument" in _err()


def test_build_batch_vars_packed_rejects_too_many_variables():
    assert _vars_packed(n_vars=2049) == _lib.C2V_EUNSUPPORTED
    assert "2049 variable indexes (max 2048)" in _err()


def test_forward_host_packed_rejects_a_null_session():
    lib = _lib.load()
    P = _lib.Params(*([ctypes.c_void_p(16)] * 8))
    rc = lib.c2v_forward_host_packed(None, ctypes.byref(P), X, X, X, X, None, 2, 4, None, X, X, None, None, 0)
    assert rc == _lib.C2V_EINVAL and "NULL" in _err()
    t = ctypes.c_int64(0)
    rc = lib.c2v_forward_host_packed_async(None, ctypes.byref(P), X, X, X, X, None, 2, 4, None, X, X, None, None, 0,
                                           ctypes.byref(t))
    assert rc == _lib.C2V_EINVAL and "NULL" in _err()

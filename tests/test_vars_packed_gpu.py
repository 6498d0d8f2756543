"""-m gpu: packed variable-name batches and the packed host-buffer calls against their padded counterparts.

Bag b of a packed batch is row b of the padded batch without its zero suffix, so the builder is checked bit for bit
(PackedBags.padded()), the per-unit counts against the numpy restatement, the model under the eval tolerance and the
training-step criterion of test_packed_gpu.py, and the host-buffer session call by call against c2v_forward_host.
"""
import ctypes

import numpy as np
import pytest
import torch

from code2vec_b200 import _lib
from code2vec_b200 import functional as CF
from code2vec_b200.batch_builder import packed_offsets
from gpu_util import random_params
from philox_ref import dropout_mask
from test_batch_builder_gpu import GV, _var_corpus
from test_packed_gpu import DEV, DROPOUT, EVAL_TOL, _model, _padded_positions, _step
from test_train_step_gpu import _reference, _rho, _scales
from test_vars_packed_abi import unit_counts

pytestmark = pytest.mark.gpu
TAGS = ["synth", "real"]


def _sizes(tag):
    """(T, P, C) that hold every token, path and label of the sample"""
    ctx, units = GV[f"{tag}_contexts"], GV[f"{tag}_units"]
    T = int(max(ctx[:, [0, 2]].max(), GV[f"{tag}_variable_indexes"].max())) + 1
    return T, int(ctx[:, 1].max()) + 1, max(int(units[:, 2].max()) + 1, 64)


def _ids(n_units):
    """every unit, two repeats, and ids outside the units"""
    return np.concatenate([np.arange(n_units), [0, n_units - 1, -1, n_units, 10 ** 6]])


# ---- counts and builder ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", TAGS)
def test_unit_counts_equal_the_oracle(tag):
    c, units = _var_corpus(tag, False)
    ref = unit_counts(GV[f"{tag}_offsets"], GV[f"{tag}_contexts"], units[:, 0], units[:, 1])
    assert c.unit_counts.dtype == np.int64 and np.array_equal(c.unit_counts, ref)
    if tag == "synth":
        assert (ref == 0).any()                                # units without a matching context
    # a unit whose item is not in the corpus counts 0
    ui = np.concatenate([units[:, 0], [-1, c.n_items]])
    uv = np.concatenate([units[:, 1], [units[0, 1]] * 2])
    c.set_variable_units(ui, uv, np.zeros(len(ui), np.int64), GV[f"{tag}_variable_indexes"], c.terminal_count)
    assert np.array_equal(c.unit_counts, np.concatenate([ref, [0, 0]]))


@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("shuffle", [False, True])
@pytest.mark.parametrize("L", [200, 5, 1])
def test_build_vars_packed_equals_build_vars_without_suffix(tag, shuffle, L):
    c, units = _var_corpus(tag, shuffle)
    ids = _ids(len(units))
    for seed in (3, 98765432123456789):
        s, p, e, lab = c.build_vars(torch.from_numpy(ids), L, seed)
        for given in (ids, torch.from_numpy(ids).to(DEV)):        # host ids and device ids
            bags, lab_pk = c.build_vars_packed(given, L, seed)
            assert np.array_equal(bags.offsets_host, packed_offsets(c.unit_counts, ids, L))
            assert torch.equal(bags.offsets.cpu(), torch.from_numpy(bags.offsets_host))
            assert torch.equal(lab_pk, lab)
            assert all(torch.equal(a, b) for a, b in zip(bags.padded(), (s, p, e)))
    n = bags.lengths()
    assert (n[-3:] == 1).all() and (bags.starts[torch.from_numpy(bags.offsets_host[-4:-1]).to(DEV)] == 0).all()
    empty = np.flatnonzero(c.unit_counts[ids[:len(units)]] == 0)
    assert (n[empty] == 1).all() and (s[torch.from_numpy(empty).to(DEV)] == 0).all()


def test_build_vars_packed_writes_only_inside_each_bag():
    """offsets that disagree with the counts (too short, too long, zero, decreasing): every bag writes at most
    min(len, L) rows from its offset, the first ones of its padded row, and nothing else is touched"""
    c, units = _var_corpus("real", True)
    rng = np.random.default_rng(2)
    L, B = 50, len(units)
    ids = np.arange(B)
    s, p, e, _ = c.build_vars(torch.from_numpy(ids), L, 9)
    lens = rng.integers(0, L + 4, B)
    lens[3] = L + 3                                            # bag 3 writes L rows: its last 3 stay untouched
    off = np.zeros(B + 1, np.int64)
    np.cumsum(lens, out=off[1:])
    off[5] = off[4] - 1                                        # bag 4 holds -1; bag 5 starts in bag 3's untouched tail
    N, GUARD = int(off[-1]), 64
    out = [torch.full((N + GUARD,), -7, dtype=torch.int64, device=DEV) for _ in range(3)]
    d_ids, d_off = torch.from_numpy(ids).to(DEV), torch.from_numpy(off).to(DEV)
    P = lambda t: ctypes.c_void_p(t.data_ptr())
    rc = _lib.load().c2v_build_batch_vars_packed(P(c.offsets), P(c.contexts), c.n_items, P(c.unit_item), P(c.unit_var),
                                                 P(c.unit_label), c.n_units, P(d_ids), B, L, 9, c.question_token,
                                                 P(c.var_pos), c.terminal_count, P(c.variable_indexes),
                                                 int(c.variable_indexes.numel()), 1, P(d_off), *(P(t) for t in out), None,
                                                 None)
    _lib.check(rc, "c2v_build_batch_vars_packed")
    want = [np.full(N + GUARD, -7, np.int64) for _ in range(3)]
    pad = [t.cpu().numpy() for t in (s, p, e)]
    for b in range(B):
        k = int(np.clip(off[b + 1] - off[b], 0, L))
        for w, a in zip(want, pad):
            w[off[b]:off[b] + k] = a[b, :k]
    for w, t in zip(want, out):
        assert np.array_equal(t.cpu().numpy(), w)


@pytest.mark.parametrize("rank,world", [(0, 1), (1, 2)])
def test_epoch_vars_packed_visits_the_same_units_in_the_same_order(rank, world):
    c, _ = _var_corpus("real", True)
    pd = list(c.epoch_vars(64, 200, seed=5, rank=rank, world=world))
    pk = list(c.epoch_vars_packed(64, 200, seed=5, rank=rank, world=world))
    assert len(pd) == len(pk) > 1
    for (s, p, e, lab), (bags, lab_pk) in zip(pd, pk):
        assert torch.equal(lab, lab_pk)
        assert torch.equal(bags.offsets.cpu(), torch.from_numpy(bags.offsets_host))
        assert all(torch.equal(a, b) for a, b in zip((s, p, e), bags.padded()))


# ---- model -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", TAGS)
@pytest.mark.parametrize("shape", [(128, 128, 128, _lib.ALGO_TCGEN05), (50, 50, 70, _lib.ALGO_FFMA)])
def test_eval_encode_of_vars_batches_matches_padded(tag, shape):
    Et, Ep, H, algo = shape
    c, units = _var_corpus(tag, True)
    T, P, C = _sizes(tag)
    L = 200
    ids = _ids(len(units))
    s, p, e, _ = c.build_vars(torch.from_numpy(ids), L, 4)
    bags, _ = c.build_vars_packed(ids, L, 4)
    prm = random_params(np.random.default_rng(1), T, P, C, Et, Ep, H)
    t = {k: torch.from_numpy(v).to(DEV) for k, v in prm.items()}
    dims = CF.make_dims(T, P, C, Et, Ep, H)
    params = CF.make_params(t["terminal_embedding.weight"], t["path_embedding.weight"], t["input_linear.weight"],
                            t["input_layer_norm.weight"], t["input_layer_norm.bias"], t["attention_parameter"])
    cv_pad, att_pad = CF.encode_forward(dims, params, s, p, e, algo=algo, check_indices=True)
    cv_pk, att_pk = CF.encode_forward_packed(dims, params, bags, algo=algo, check_indices=True)
    torch.cuda.synchronize()
    # every bag, the ones without a matching context (h(0, 0, 0) in both layouts) included
    assert float((cv_pk - cv_pad).abs().max()) <= EVAL_TOL
    real = torch.from_numpy(np.repeat((s != 0).any(1).cpu().numpy(), bags.lengths())).to(DEV)
    a_pad = att_pad.reshape(-1)[_padded_positions(bags)]
    sel = real & (a_pad > 0)
    assert float(((att_pk - a_pad).abs() / a_pad)[sel].max()) <= EVAL_TOL


def test_training_step_on_vars_batches_matches_padded():
    c, units = _var_corpus("real", True)
    T, P, C = _sizes("real")
    L = 200
    ids = np.flatnonzero(c.unit_counts > 0)                     # units with at least one match: the same mask in both
    B = len(ids)
    s, p, e, label = c.build_vars(torch.from_numpy(ids), L, 6)
    bags, _ = c.build_vars_packed(ids, L, 6)
    m = _model(np.random.default_rng(12), T, P, C, 128, 128, 128).train()
    seed = 0x5EED4321
    l_pd, cv_pd, att_pd, g_pd, _ = _step(m, (s, p, e), label, seed)
    l_pk, cv_pk, att_pk, g_pk, used = _step(m, (bags, None, None), label, seed)
    assert used == [seed] and att_pk.shape == (bags.N,)
    mask = torch.from_numpy(dropout_mask(seed, B * L, 128, DROPOUT).reshape(B, L, 128)).to(DEV)
    params = {k: v.detach() for k, v in m.state_dict().items()}
    r64 = _reference(params, (s, p, e, label), mask, False, torch.float64)
    S = _scales(r64, (s, p, e, label), mask, False)
    att_pk_pad = torch.zeros(B * L, device=DEV).index_put_((_padded_positions(bags),), att_pk).view(B, L)
    checks = [("loss", l_pd, l_pk, r64["loss"], S["loss"]), ("cv", cv_pd, cv_pk, r64["cv"], S["cv"]),
              ("att", att_pd, att_pk_pad, r64["att"], S["att"])]
    checks += [(k, g_pd[k], g_pk[k], r64["grads"][k], S[k]) for k in g_pd]
    failures = []
    for name, a_pd, a_pk, ref, Sx in checks:                    # the criterion of test_packed_gpu.py
        zv = []
        r_pd = _rho(a_pd, ref, Sx, name + " padded", [])
        r_pk = _rho(a_pk, ref, Sx, name, zv)
        if r_pk > max(4.0 * r_pd, 2.0 ** -20) or zv:
            failures.append(f"{name}: rho packed {r_pk:.3g} padded {r_pd:.3g} {zv}")
    assert not failures, failures


# ---- host-buffer session ---------------------------------------------------------------------------------------------
def _pin(t):
    return t.cpu().contiguous().pin_memory()


class _Session:
    """a c2v_session for model m with pinned result buffers for one batch of B bags and at most B * L contexts"""

    def __init__(self, m, B, L):
        self.lib, self.m, self.B, self.L = _lib.load(), m, B, L
        self.dims = m._dims()
        w_out, b_out = m._head()
        self.params = CF.make_params(m.terminal_embedding.weight.data, m.path_embedding.weight.data,
                                     m.input_linear.weight.data, m.input_layer_norm.weight.data,
                                     m.input_layer_norm.bias.data, m.attention_parameter.data, w_out.data, b_out.data)
        self.s = ctypes.c_void_p()
        _lib.check(self.lib.c2v_session_create(0, ctypes.byref(self.dims), B, L, ctypes.byref(self.s)), "session_create")

    def outputs(self, n):
        H = self.dims.encode
        return (torch.empty((self.B, H)).pin_memory(), torch.empty((n,)).pin_memory(),
                torch.empty((self.B,), dtype=torch.int64).pin_memory(), torch.empty((self.B,)).pin_memory())

    def call(self, batch, out, algo=_lib.ALGO_AUTO, ticket=None, B=None, N=None):
        """padded batch = (s, p, e) pinned [B, L]; packed batch = (s, p, e, offsets) pinned, [N] and [B + 1].  With a
        ticket (ctypes int64): the asynchronous call."""
        P = lambda t: ctypes.c_void_p(t.data_ptr())
        cv, att, pred, score = out
        B = self.B if B is None else B
        tail = (None, P(cv), P(att), P(pred), P(score), algo) + ((ctypes.byref(ticket),) if ticket is not None else ())
        if len(batch) == 3:
            fn = self.lib.c2v_forward_host_async if ticket is not None else self.lib.c2v_forward_host
            return fn(self.s, ctypes.byref(self.params), *(P(t) for t in batch), None, B, *tail)
        fn = self.lib.c2v_forward_host_packed_async if ticket is not None else self.lib.c2v_forward_host_packed
        N = batch[0].numel() if N is None else N
        return fn(self.s, ctypes.byref(self.params), *(P(t) for t in batch), None, B, N, *tail)

    def close(self):
        self.lib.c2v_session_destroy(self.s)


def _session_case():
    c, units = _var_corpus("real", True)
    T, P, C = _sizes("real")
    L = 200
    ids = _ids(len(units))
    s, p, e, _ = c.build_vars(torch.from_numpy(ids), L, 8)
    bags, _ = c.build_vars_packed(ids, L, 8)
    m = _model(np.random.default_rng(13), T, P, C, 128, 128, 128).eval()
    padded = tuple(_pin(t) for t in (s, p, e))
    packed = tuple(_pin(t) for t in (bags.starts, bags.paths, bags.ends)) + (_pin(torch.from_numpy(bags.offsets_host)),)
    return m, bags, padded, packed, len(ids), L


def test_forward_host_packed_matches_forward_host():
    m, bags, padded, packed, B, L = _session_case()
    ss = _Session(m, B, L)
    try:
        o_pd, o_pk = ss.outputs(B * L), ss.outputs(bags.N)
        _lib.check(ss.call(padded, o_pd), "c2v_forward_host")
        _lib.check(ss.call(packed, o_pk), "c2v_forward_host_packed")
        assert float((o_pk[0] - o_pd[0]).abs().max()) <= EVAL_TOL
        a_pad = o_pd[1][_padded_positions(bags).cpu()]
        real = torch.from_numpy(np.repeat((padded[0] != 0).any(1).numpy(), bags.lengths()))
        sel = real & (a_pad > 0)
        assert float(((o_pk[1] - a_pad).abs() / a_pad)[sel].max()) <= EVAL_TOL
        assert torch.equal(o_pk[2], o_pd[2])
        # an out-of-range index: C2V_EINDEX, as the padded call
        bad = packed[0].clone().pin_memory()
        bad[3] = m.option.terminal_count + 5
        assert ss.call((bad,) + packed[1:], o_pk) == _lib.C2V_EINDEX
    finally:
        ss.close()


def test_forward_host_packed_rejects_malformed_offsets():
    m, bags, padded, packed, B, L = _session_case()
    ss = _Session(m, B, L)
    try:
        out = ss.outputs(bags.N)
        off = packed[3]

        def with_offsets(fix):
            o = off.clone(); fix(o)
            return packed[:3] + (o.pin_memory(),)
        cases = [("offsets[0] = 1", with_offsets(lambda o: o.add_(1)), {}),
                 ("bag 2 holds 0", with_offsets(lambda o: o.__setitem__(3, o[2])), {}),
                 ("bag 0 holds 201", with_offsets(lambda o: o.__setitem__(1, L + 1)), {}),
                 ("!= N", packed, {"N": bags.N + 1}),
                 (f"B={B + 1} not in", packed, {"B": B + 1})]
        for msg, batch, kw in cases:
            assert ss.call(batch, out, **kw) == _lib.C2V_EINVAL, msg
            assert msg in _lib.load().c2v_last_error().decode(), msg
        _lib.check(ss.call(packed, out), "the session still serves a valid batch")
    finally:
        ss.close()


def test_padded_and_packed_calls_share_a_session():
    """16 asynchronous calls, 4 in flight, alternating the layout on every slot, with C2V_FLAG_REUSE_PREP: each result is
    bit for bit the one of a single call on a fresh session"""
    m, bags, padded, packed, B, L = _session_case()
    ref = {}
    for name, batch, n in (("padded", padded, B * L), ("packed", packed, bags.N)):
        ss = _Session(m, B, L)
        try:
            ref[name] = ss.outputs(n)
            _lib.check(ss.call(batch, ref[name]), name)
        finally:
            ss.close()
    ss = _Session(m, B, L)
    try:
        ticket, pending = ctypes.c_int64(0), []
        for i in range(16):
            name = "packed" if (i // 4 + i) % 2 else "padded"        # call 4k + j on slot j: the layout alternates
            out = ss.outputs(B * L if name == "padded" else bags.N)
            rc = ss.call(padded if name == "padded" else packed, out, algo=_lib.ALGO_AUTO | 0x100, ticket=ticket)
            _lib.check(rc, name)
            pending.append((ticket.value, name, out))
            if len(pending) == 4:
                t, name_done, got = pending.pop(0)
                _lib.check(ss.lib.c2v_session_wait(ss.s, t), "session_wait")
                assert all(torch.equal(a, b) for a, b in zip(got, ref[name_done])), (t, name_done)
        for t, name_done, got in pending:
            _lib.check(ss.lib.c2v_session_wait(ss.s, t), "session_wait")
            assert all(torch.equal(a, b) for a, b in zip(got, ref[name_done])), (t, name_done)
    finally:
        ss.close()

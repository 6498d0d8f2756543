"""Host side of the deterministic mode (no GPU needed): c2v_set_deterministic / c2v_get_deterministic are per thread, the
workspace sizes grow with the mode on and are unchanged with it off, and ShardedFlatAdam's "nvls" rule."""
import ctypes
import threading
import warnings

import pytest
import torch

from code2vec_b200 import _lib
from code2vec_b200 import functional as CF
from code2vec_b200.distributed import ShardedFlatAdam, nvls_allowed


@pytest.fixture
def lib():
    lib = _lib.load()
    yield lib
    lib.c2v_set_deterministic(0)


@pytest.fixture
def torch_switch():
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield
    torch.use_deterministic_algorithms(prev, warn_only=warn)


def test_set_get_is_per_thread(lib):
    assert lib.c2v_get_deterministic() == 0
    assert lib.c2v_set_deterministic(1) == 0
    assert lib.c2v_get_deterministic() == 1
    seen = {}

    def other():
        seen["initial"] = lib.c2v_get_deterministic()
        lib.c2v_set_deterministic(1)
        lib.c2v_set_deterministic(0)
        seen["after"] = lib.c2v_get_deterministic()
    t = threading.Thread(target=other)
    t.start()
    t.join()
    assert seen == {"initial": 0, "after": 0}
    assert lib.c2v_get_deterministic() == 1              # untouched by the other thread
    lib.c2v_set_deterministic(0)
    assert lib.c2v_get_deterministic() == 0


def _sizes(lib, dims, B, L, N):
    d = ctypes.byref(dims)
    return {"backward": lib.c2v_encode_backward_workspace_bytes(d, B, L),
            "backward_packed": lib.c2v_encode_backward_packed_workspace_bytes(d, B, N),
            "label": lib.c2v_label_workspace_bytes(d, B),
            "topk": lib.c2v_label_topk_workspace_bytes(d, B, 5)}


@pytest.mark.parametrize("shape", [(360633, 342846, 8192, 128, 128, 128, 1024, 200), (3000, 4000, 257, 37, 29, 45, 48, 33)])
def test_workspace_sizes(lib, shape):
    T, P, C, Et, Ep, H, B, L = shape
    dims = CF.make_dims(T, P, C, Et, Ep, H)
    N = B * L // 2
    off = _sizes(lib, dims, B, L, N)
    lib.c2v_set_deterministic(1)
    on = _sizes(lib, dims, B, L, N)
    lib.c2v_set_deterministic(0)
    assert _sizes(lib, dims, B, L, N) == off             # back to the default sizes
    for k in ("backward", "backward_packed", "label"):
        assert on[k] > off[k], k
    assert on["topk"] >= on["label"]
    # the dC rows alone: [N, 2E_t + E_p] fp32
    D = 2 * Et + Ep
    assert on["backward"] - off["backward"] >= B * L * D * 4
    assert on["backward_packed"] - off["backward_packed"] >= N * D * 4


def test_sync_follows_torch_switch(lib, torch_switch):
    torch.use_deterministic_algorithms(True)
    assert CF.sync_deterministic() is True and lib.c2v_get_deterministic() == 1
    torch.use_deterministic_algorithms(False)
    assert CF.sync_deterministic() is False and lib.c2v_get_deterministic() == 0


def test_nvls_rule(torch_switch):
    torch.use_deterministic_algorithms(False)
    assert nvls_allowed("auto", 8) and nvls_allowed("nvls", 8)
    torch.use_deterministic_algorithms(True)
    assert nvls_allowed("auto", 1) and nvls_allowed("nvls", 1)      # one rank: no cross-GPU reduction
    assert not nvls_allowed("auto", 8)
    assert not nvls_allowed("p2p", 8) and not nvls_allowed("nccl", 8)
    with pytest.raises(RuntimeError, match="nvls"):
        nvls_allowed("nvls", 8)
    torch.use_deterministic_algorithms(True, warn_only=True)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        assert not nvls_allowed("nvls", 8)
    assert any(issubclass(x.category, UserWarning) and "nvls" in str(x.message) for x in w)


def test_nvls_rule_holds_at_step_time(torch_switch):
    """an optimizer that chose "nvls" before the switch was turned on refuses to step under it (before any device work)"""
    opt = ShardedFlatAdam.__new__(ShardedFlatAdam)
    opt.capturable, opt.transport, opt.world = False, "nvls", 8
    torch.use_deterministic_algorithms(True)
    with pytest.raises(RuntimeError, match="nvls"):
        opt.step()

"""No GPU: the mode-envelope case table (tests/mode_envelope.py) against the library's exported dispatch predicates, the
kernel instantiations the built library holds, and the constants of the deterministic reduction, so that a case whose
expected kernels drift from the code fails on the CPU."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import mode_envelope as ME
import shape_envelope as SE
from code2vec_b200 import _lib
from code2vec_b200 import functional as CF

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "code2vec_b200", "csrc")
CASES = dict(ME.TRAIN, **{"table-past-4GB": ME.TABLE_4GB})


@pytest.mark.parametrize("case", list(CASES))
def test_training_case_path_matches_the_predicates(case):
    """as test_shape_envelope_abi.py: the encode and label paths from the exported predicates, the dW / dC rule restated"""
    c = CASES[case]
    d = CF.make_dims(c["T"], c["P"], c["C"], c["Et"], c["Ep"], c["H"])
    lib = _lib.load()
    assert bool(lib.c2v_encode_supports_tcgen05(ctypes.byref(d))) == (c["paths"]["encode"] == SE.TC)
    assert CF.label_loss_supported(d, c["B"]) == (c["paths"]["label"] == SE.TC)
    E, H = c["Et"], c["H"]
    assert H <= 512, "the encode backward takes H <= 512"
    fits = c["Et"] == c["Ep"] and E <= 256 and H % 4 == 0 and E % 4 == 0
    under_4gb = max(c["T"], c["P"]) * E * 4 < 2 ** 32
    assert (fits and under_4gb) == (c["paths"]["dw"] == SE.TC)
    assert (fits and max(c["T"], c["P"]) * (E // 4) < 2 ** 32 - 1) == (c["paths"]["dc"] == SE.TC)
    assert lib.c2v_encode_backward_workspace_bytes(ctypes.byref(d), c["B"], c["L"]) > 0


def test_every_mode_and_group_is_covered():
    modes = {m for c in CASES.values() for m in c["modes"]}
    assert modes == {ME.DEFAULT, *ME.MODES}
    for shape in ME.GROUP_SHAPES:
        name = "e{}-{}-h{}-b129x33".format(*shape)
        assert CASES[name + "-unstashed"]["modes"] == (ME.DET, ME.DET_SPARSE)
        assert CASES[name + "-angular"]["angular"]
    groups = {tuple(sorted(CASES["e{}-{}-h{}-b129x33".format(*s)]["paths"].items())) for s in ME.GROUP_SHAPES}
    assert len(groups) == len(ME.GROUP_SHAPES), "one shape per group"
    for name, c in SE.TRAIN.items():
        if name != "table-past-4GB":
            assert CASES[name]["modes"] == ME.MODES and CASES[name]["layout"] == c["layout"]


def _library_symbols():
    nm = shutil.which("nm")
    if nm is None:
        pytest.skip("nm (binutils) is not installed")
    out = subprocess.run([nm, "-C", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    return [line for line in out.splitlines() if "c2v::" in line]


def test_every_kernel_prefix_names_an_instantiation():
    """every kernel-name prefix the table expects is a c2v:: symbol of the built library (the host stubs of the kernels
    are listed there under their demangled names), so a typo fails without a GPU"""
    syms = _library_symbols()
    prefixes = set()
    for c in CASES.values():
        for mode in c["modes"]:
            want, never = ME.mode_kernels(c, mode)
            prefixes |= set(want) | {k for k in never if k != "det_"}
    for H in {c["H"] for c in SE.LABEL.values()}:
        prefixes |= set(ME.label_det_kernels(H))
    missing = sorted(k for k in prefixes if not any("c2v::" + k in s for s in syms))
    assert not missing, missing
    assert any("c2v::det_" in s for s in syms)


def test_constants_match_the_deterministic_reduction():
    src = open(os.path.join(CSRC, "c2v_deterministic.cu")).read()
    assert int(re.search(r"constexpr int kChunk = (\d+);", src).group(1)) == ME.K_CHUNK
    assert int(re.search(r"constexpr int kShortRun = (\d+);", src).group(1)) == ME.K_SHORT_RUN
    assert int(re.search(r"constexpr int kCols = (\d+);", src).group(1)) == 256


@pytest.mark.parametrize("case", [k for k, c in ME.TRAIN.items() if c["hot"]])
def test_hot_rows_reach_the_cooperative_merge(case):
    """the hot rows' sorted keys span more than K_SHORT_RUN chunks in both tables, and each hot row's slot in the compact
    gradient is another row inside it: a merge that wrote the row index instead of the slot would write a wrong row"""
    c = ME.TRAIN[case]
    spans = ME.hot_run_chunks(c)
    assert min(spans.values()) > ME.K_SHORT_RUN + 1, spans
    s, p, e, _ = ME.hot_batch(c)
    for hot, idx in ((c["hot"][0], np.concatenate((s.ravel(), e.ravel()))), (c["hot"][1], p.ravel())):
        rows = np.unique(idx)
        slot = int(np.searchsorted(rows, hot))
        assert rows[slot] == hot and slot != hot and hot < len(rows), (hot, slot, len(rows))


def test_wide_embedding_case():
    c = ME.TRAIN["e264-264-h128-b129x33"]
    assert c["Et"] > 256 and c["Ep"] > 256
    assert c["modes"] == (ME.DEFAULT, ME.DET)

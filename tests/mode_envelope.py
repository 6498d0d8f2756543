"""The training modes with kernels of their own, across the shape envelope: one table of cases, each naming the kernels
its shape and mode must reach.

  * deterministic mode (torch.use_deterministic_algorithms(True)): the dC kernels store per-context rows
    (backward_dc_tc_kernel<false, true>, the DET instantiations of backward_rows_kernel / backward_rows_lite_kernel), which
    det_keys / radix sort / det_chunk / det_merge sum per table row; dW, d attention, d gamma, d beta and the label head's
    d code_vector come from slabs (det_slab_sum_kernel); the CUDA-core head sums its loss in loss_sum_kernel /
    angular_sums_kernel;
  * sparse embedding gradients (nn.Embedding.sparse on both tables): dC goes through slot maps
    (backward_dc_tc_kernel<true, false>, the SPARSE instantiations of backward_rows_kernel), and through det_dst(.., slot,
    ..) in det_chunk / det_merge when both modes are on.

test_mode_envelope_abi.py checks the table against the library's exported predicates and symbols (no GPU);
test_mode_envelope_gpu.py runs every case, checks with torch.profiler that the named kernels ran and judges the results
element by element against fp64 (tests/fp64_judge.py), with the bound the same case has in the default mode.
"""
import numpy as np

import shape_envelope as SE
import test_wide_encode_gpu as WE

TC, FFMA = SE.TC, SE.FFMA
DEFAULT, DET, SPARSE, DET_SPARSE = "default", "det", "sparse", "det+sparse"
MODES = (DET, SPARSE, DET_SPARSE)

# c2v_deterministic.cu: sorted keys per chunk, and the longest run (in further chunks) its owner warp sums alone; a longer
# run is summed by the merge CTA's cooperative path (test_mode_envelope_abi.py reads both from the source)
K_CHUNK, K_SHORT_RUN = 32, 64


def _case(Et, Ep, H, B, L, paths, modes=MODES, layout="padded", T=SE.T_SMALL, P=SE.P_SMALL, looser=None, **extra):
    """looser: (table, case) whose default-mode bound applies: test_shape_envelope_gpu.LOOSER ("shape") or
    test_wide_encode_gpu.LOOSER ("wide")"""
    c = dict(Et=Et, Ep=Ep, H=H, B=B, L=L, T=T, P=P, C=SE.C_TRAIN, layout=layout, paths=dict(paths), modes=tuple(modes),
             env={}, hot=None, angular=False, looser=looser)
    c.update(extra)
    return c


def _wide_paths(shape):
    return WE.GROUPS[WE.SHAPES[shape]]


TRAIN = {}
# every training case of the shape envelope.  Its forward-only shape (H = 260) trains since the encode backward takes
# H <= 512: it runs with the paths test_wide_encode_gpu.py gives it.
for _name, _c in SE.TRAIN.items():
    if _name == "table-past-4GB":
        continue
    _shape = (_c["Et"], _c["Ep"], _c["H"])
    _wide = "dw" not in _c["paths"]
    TRAIN[_name] = _case(*_shape, _c["B"], _c["L"], _wide_paths(_shape) if _wide else _c["paths"], layout=_c["layout"],
                         T=_c["T"], P=_c["P"], looser=("wide" if _wide else "shape", _name))
# the encode sizes above 256, at (B, L) = (129, 33)
for _shape in WE.SHAPES:
    _name = "e{}-{}-h{}-b129x33".format(*_shape)
    if _name not in TRAIN:
        TRAIN[_name] = _case(*_shape, 129, 33, _wide_paths(_shape), looser=("wide", _name))

# one shape per group of both tables (the packed shapes are one per group)
GROUP_SHAPES = tuple(SE.PACKED) + (WE.PAPER,)


def _base(shape):
    return TRAIN["e{}-{}-h{}-b129x33".format(*shape)]


# C2V_NO_STASH=1: x is recomputed, so backward_rows_kernel (not the lite kernel) runs next to the tensor-core dC
for _shape in GROUP_SHAPES:
    _b = _base(_shape)
    TRAIN["e{}-{}-h{}-b129x33-unstashed".format(*_shape)] = dict(_b, modes=(DET, DET_SPARSE), env={"C2V_NO_STASH": "1"})

# hot rows: terminal HOT_T as the start and path HOT_P in the first 3/4 of every bag's contexts.  The sorted keys of each
# hot row span a few hundred chunks, past K_SHORT_RUN, so det_merge's cooperative path sums them.  The tables are large
# and the hot rows' indices small, so each hot row's slot in the compact gradient is another row of it.
HOT_T, HOT_P, T_HOT = 1000, 1000, 100_003
for _shape in ((128, 128, 128), (37, 29, 45)):
    _paths = SE.GROUPS["tensor-cores"] if _shape == (128, 128, 128) else SE.GROUPS["cuda-cores"]
    TRAIN["e{}-{}-h{}-b85x200-hot".format(*_shape)] = _case(*_shape, 85, 200, _paths, modes=(DET, DET_SPARSE), T=T_HOT,
                                                            P=T_HOT, hot=(HOT_T, HOT_P), looser=None)

# embeddings wider than 256 (dims_ok takes them): CUDA-core encode, dW and dC, tensor-core label head; det_chunk and
# det_merge make two column passes of 256
TRAIN["e264-264-h128-b129x33"] = _case(264, 264, 128, 129, 33, dict(encode=FFMA, dw=FFMA, dc=FFMA, label=TC),
                                       modes=(DEFAULT, DET))

# the angular-margin head, one shape per group
for _shape in GROUP_SHAPES:
    _b = _base(_shape)
    TRAIN["e{}-{}-h{}-b129x33-angular".format(*_shape)] = dict(_b, modes=(DET,), angular=True)

# a terminal table past 4 GB (shape_envelope's case) with compact gradients: judged on the rows the batch touches
TABLE_4GB = _case(128, 128, 128, 9, 33, SE.TRAIN["table-past-4GB"]["paths"], modes=(SPARSE, DET_SPARSE),
                  T=SE.TRAIN["table-past-4GB"]["T"], P=SE.TRAIN["table-past-4GB"]["P"], looser=("shape", "table-past-4GB"))

# one model stepped with the switch off, on, off
MODE_SWITCH = "e124-124-h128-b129x33"

# the CUDA-core label head where the default mode's sgemm splits K (few output tiles, K = C >= 1024) and the deterministic
# one must not
FFMA_HEAD = dict(B=129, C=4099, H=260)


def hot_batch(c, seed=4):
    """(starts, paths, ends, label) as int64 numpy arrays: bags with a zero-padded suffix (bag 0 full, bag 1 of one
    context), the hot rows in the first 3/4 of every bag's contexts"""
    rng = np.random.default_rng(seed)
    B, L, T, P = c["B"], c["L"], c["T"], c["P"]
    s = rng.integers(1, T, (B, L))
    p = rng.integers(1, P, (B, L))
    e = rng.integers(1, T, (B, L))
    n = rng.integers(L // 2, L + 1, B)
    n[0], n[1] = L, 1
    s[:, : 3 * L // 4], p[:, : 3 * L // 4] = c["hot"]
    valid = np.arange(L)[None, :] < n[:, None]
    return s * valid, p * valid, e * valid, rng.integers(0, c["C"], B)


def hot_run_chunks(c):
    """per table, the number of chunks the hot row's sorted keys span (contexts of attention 0 hold no key)"""
    s, p, e, _ = hot_batch(c)
    return {"terminal": (int((s == c["hot"][0]).sum() + (e == c["hot"][0]).sum()) + K_CHUNK - 1) // K_CHUNK,
            "path": (int((p == c["hot"][1]).sum()) + K_CHUNK - 1) // K_CHUNK}


def _rows_kernel(c, mode, stash):
    """the instantiation of the encode backward's row kernel the case launches in `mode` (c2v_backward.cu)"""
    det, sparse = mode in (DET, DET_SPARSE), mode in (SPARSE, DET_SPARSE)
    packed = "true" if c["layout"] == "packed" else "false"
    b = lambda v: "true" if v else "false"
    if stash and c["paths"]["dc"] == TC and c["H"] % 4 == 0:
        return f"backward_rows_lite_kernel<{(c['H'] + 127) // 128}, {packed}, false, {b(det)}>"
    vec = c["Et"] % 4 == 0 and c["Ep"] % 4 == 0
    sp = sparse and not det and c["paths"]["dc"] == FFMA          # (the SPARSE rows kernel scatters dC itself)
    return f"backward_rows_kernel<{b(vec)}, {packed}, {b(sp)}, false, {b(det)}, {8 if c['H'] <= 256 else 16}>"


def mode_kernels(c, mode):
    """-> (prefixes of kernel names that must run, prefixes of kernel names that must not run) for a training case in
    `mode`, beyond the stage paths of c["paths"]"""
    stash = c["env"].get("C2V_NO_STASH") != "1"
    want, never = [_rows_kernel(c, mode, stash)], []
    if mode in (DET, DET_SPARSE):
        want += ["det_keys_kernel", "det_chunk_kernel", "det_merge_kernel", "det_slab_sum_kernel"]
        never += ["backward_dc_tc_kernel<false, false>", "backward_dc_tc_kernel<true, false>"]
        if c["paths"]["dc"] == TC:
            want.append("backward_dc_tc_kernel<false, true>")
        if c["paths"]["label"] == TC:
            want.append(f"label_dcv_tc_kernel<{(c['H'] + 63) // 64}, true")
        else:
            want.append("angular_sums_kernel" if c["angular"] else "loss_sum_kernel")
    else:
        never += ["det_"]
        if mode == SPARSE and c["paths"]["dc"] == TC:
            want.append("backward_dc_tc_kernel<true, false>")
            never.append("backward_dc_tc_kernel<false, false>")
    return want, never


# the label head in deterministic mode: d code_vector on the tensor cores from kDetLabelSplits slabs
def label_det_kernels(H):
    return [f"label_dcv_tc_kernel<{(H + 63) // 64}, true", "det_slab_sum_kernel"]

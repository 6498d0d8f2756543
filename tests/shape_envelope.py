"""The shape envelope of the kernels: one table of cases, each naming the kernels its shape must reach.

test_shape_envelope_abi.py checks every case's expected path against the library's exported predicates (no GPU), so a
case table that drifts from the dispatch rules fails on the CPU.  test_shape_envelope_gpu.py runs every case, checks with
torch.profiler that the named kernels ran (a silent fallback would make a case test nothing) and judges the results
element by element against fp64 (tests/fp64_judge.py).

Dispatch rules the table encodes (c2v_encode_wgmma.cu tcgen05_shape_ok, c2v_backward_dw_tc.cu / c2v_backward_dc_tc.cu,
c2v_label_tcgen05.cu label_tcgen05_shape_ok):
  * encode on the tensor cores: Et == Ep, Et % 4 == 0, H in {100, 128} with Et <= 128 or H = 256 with Et <= 256, and
    every table under 4 GB (T * Et * 4 < 2^32);
  * dW on the tensor cores: Et == Ep <= 256, H <= 256, both multiples of 4, every table under 4 GB;
  * dC on the tensor cores: the same, but the table bound counts 16-byte units (T * Et / 4 < 2^32 - 1);
  * label head (label GEMM, fused loss / arg-max / top-k, label backward) on the tensor cores: H % 4 == 0, 4 <= H <= 256,
    and for the fused modes B <= 2048.
"""
TC, FFMA = "tc", "ffma"

# the kernels that identify each choice (substrings of the c2v:: kernel names torch.profiler reports)
KERNELS = {
    "encode": {TC: ("encode_wgmma_kernel",), FFMA: ("encode_ffma_kernel",)},
    "dw": {TC: ("backward_dw_tc_kernel",), FFMA: ("backward_dw_kernel",)},
    "dc": {TC: ("backward_dc_tc_kernel",), FFMA: ("backward_rows_kernel",)},
    "label": {TC: ("label_gemm_v2_kernel", "label_dw_tc_kernel", "label_dcv_tc_kernel"), FFMA: ("sgemm_kernel",)},
}

# (Et, Ep, H) -> group, {stage: path}
GROUPS = {
    "tensor-cores": dict(encode=TC, dw=TC, dc=TC, label=TC),
    "ffma-forward": dict(encode=FFMA, dw=TC, dc=TC, label=TC),      # CUDA-core forward, tensor-core dW / dC and label head
    "et-ne-ep": dict(encode=FFMA, dw=FFMA, dc=FFMA, label=TC),
    "cuda-cores": dict(encode=FFMA, dw=FFMA, dc=FFMA, label=FFMA),
    # the encode backward takes H <= 256 (c2v_encode_backward raises NotImplementedError above): forward_loss only
    "forward-only": dict(encode=FFMA, label=FFMA),
}
SHAPES = {
    (4, 4, 100): "tensor-cores", (124, 124, 128): "tensor-cores", (132, 132, 256): "tensor-cores",
    (256, 256, 256): "tensor-cores",
    (200, 200, 192): "ffma-forward", (64, 64, 60): "ffma-forward", (128, 128, 4): "ffma-forward",
    (256, 256, 252): "ffma-forward",
    (128, 96, 128): "et-ne-ep",
    (37, 29, 45): "cuda-cores", (128, 128, 260): "forward-only",
}
BAGS = ((1, 1), (129, 33), (7, 333))           # (B, L): one context; ragged bags over several tiles; bags over many tiles
PACKED = ((124, 124, 128), (200, 200, 192), (128, 96, 128), (37, 29, 45))    # one trainable shape per group, packed too
T_SMALL, P_SMALL, C_TRAIN = 3001, 2999, 1031


def _train_case(Et, Ep, H, B, L, layout="padded", T=T_SMALL, P=P_SMALL, C=C_TRAIN, paths=None):
    return dict(Et=Et, Ep=Ep, H=H, B=B, L=L, T=T, P=P, C=C, layout=layout,
                paths=dict(paths if paths is not None else GROUPS[SHAPES[(Et, Ep, H)]]))


TRAIN = {}
for (_et, _ep, _h) in SHAPES:
    for (_b, _l) in BAGS:
        TRAIN[f"e{_et}-{_ep}-h{_h}-b{_b}x{_l}"] = _train_case(_et, _ep, _h, _b, _l)
for (_et, _ep, _h) in PACKED:
    TRAIN[f"e{_et}-{_ep}-h{_h}-b129x33-packed"] = _train_case(_et, _ep, _h, 129, 33, "packed")
# 17,000 context rows: 133 encode tiles of 128, one more than the 132 SMs of an H100 SXM (persistent grid + one tile)
TRAIN["e128-128-h128-b85x200"] = _train_case(128, 128, 128, 85, 200, T=20011, P=20011, paths=GROUPS["tensor-cores"])
# a terminal table past 4 GB (T * E * 4 = 2^32 + 512): the tensor-core encode and dW turn off, dC stays on; row T - 1
# starts at byte 2^32.  Judged on the compacted rows the batch touches.
TRAIN["table-past-4GB"] = _train_case(128, 128, 128, 9, 33, T=8_388_609, P=4099,
                                      paths=dict(encode=FFMA, dw=FFMA, dc=TC, label=TC))

# label-head cases (functional API, plain and angular head): a covering set over
#   B in {1, 127, 128, 129, 1793, 1920, 2048}, C in {1, 2, 127, 128, 129, 1023, 16896, 16897, 195299},
#   H in {4, 60, 64, 68, 100, 252, 256}
# B = 1793 .. 1920 is mt = 15 m-tiles: at 132 SMs 15 * 8 = 120 CTAs busy in lane order (< 95 %), so with n_tiles >= 132
# the label GEMM takes groups order by default; C = 16897 leaves a last n-tile of one label.  B = 2048 is the largest fused
# batch.
LABEL = {f"b{b}-c{c}-h{h}": dict(B=b, C=c, H=h) for b, c, h in (
    (1, 1, 4), (1, 16897, 256), (127, 2, 60), (127, 1023, 100), (128, 127, 64), (128, 1, 252), (129, 128, 68),
    (129, 195299, 100), (1793, 129, 100), (1793, 16896, 68), (1920, 16897, 252), (1920, 1023, 4), (2048, 16896, 256),
    (2048, 2, 64), (127, 129, 60), (1920, 128, 256))}
LABEL_GROUPS_CASES = ("b1793-c16896-h68", "b1920-c16897-h252")     # groups order by default at 132 SMs


def topk_ks(C):
    return sorted({1, min(16, C)})


def default_label_order(B, C, sms):
    """the label GEMM's default tile order (c2v_label_tcgen05.cu, launch_label_tcgen05_ex): lanes when per_m * mt keeps
    >= 95 % of the CTAs busy, else groups"""
    mt, nt = (B + 127) // 128, (C + 127) // 128
    grid = min(mt * nt, sms)
    per_m = grid // mt if mt <= grid else 0
    if per_m > 0 and per_m * mt * 100 < 95 * grid:
        per_m = 0
    return "lanes" if per_m > 0 else "groups"

// c2v_common.cuh -- shared device helpers and internal launch declarations.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/c2v_b200.h"

#define C2V_NINF (-3.4e38f)   // model.py:12 (finite fp32, NOT -inf)
#define C2V_LN_EPS 1e-5f       // nn.LayerNorm default, model.py:24
#define C2V_MIRROR_MAGIC 0x0C2B200C0FFEE5A5LL   // guards the status-mirror pointer stored in the workspace header

namespace c2v {

// ---------------------------------------------------------------------------------
// error plumbing (host)
// ---------------------------------------------------------------------------------
void set_error(const char *fmt, ...);
extern long long g_launches;
#define C2V_COUNT_LAUNCH() (__atomic_add_fetch(&::c2v::g_launches, 1, __ATOMIC_RELAXED))
#define C2V_CUDA_OK(expr)                                                                     \
    do {                                                                                      \
        cudaError_t _e = (expr);                                                              \
        if (_e != cudaSuccess) {                                                              \
            ::c2v::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, \
                             __LINE__);                                                       \
            return C2V_ECUDA;                                                                 \
        }                                                                                     \
    } while (0)
#define C2V_LAUNCH_OK(name)                                                                   \
    do {                                                                                      \
        C2V_COUNT_LAUNCH();                                                                   \
        cudaError_t _e = cudaGetLastError();                                                  \
        if (_e != cudaSuccess) {                                                              \
            ::c2v::set_error("launch of %s failed: %s", name, cudaGetErrorString(_e));        \
            return C2V_ECUDA;                                                                 \
        }                                                                                     \
    } while (0)

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Timing experiments (skip a role's work to see what the others cost; results become wrong) exist only in builds
// with -DC2V_EXPERIMENTS (C2V_NVCC_EXTRA=-DC2V_EXPERIMENTS python -m code2vec_b200.build); product builds compile them out.
#ifdef C2V_EXPERIMENTS
#define C2V_EXPT(flags, bit) (((flags) & (bit)) != 0)
#else
#define C2V_EXPT(flags, bit) false
#endif

#ifdef __CUDACC__
// Programmatic dependent launch: the kernel may start (prologue, block scheduling) while the previous kernel of the
// stream is still draining; it must execute griddepcontrol.wait (pdl_wait()) before touching anything the previous
// kernel wrote.  C2V_NO_PDL=1 falls back to a plain launch (A/B timing).
bool pdl_enabled();
// per-call switch (thread local, set by the extern "C" entry points): the calls that feed autograd -- the stashing training
// forward, or any call with C2V_FLAG_NO_PDL -- use plain stream-ordered launches
extern thread_local bool g_pdl_this_call;
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args)
{
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = (pdl_enabled() && g_pdl_this_call) ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
#endif

// ---------------------------------------------------------------------------------
// workspace layout of one encode call (all offsets 256-B aligned)
// ---------------------------------------------------------------------------------
struct EncodeWorkspace {
    long long *status;     // [0] out-of-range index count
    float *prep_hdr;       // [0] 1/w_scale (tensor-core path), [1] w_scale
    float *w_t;            // FFMA: W transposed, [D][Hs] fp32 (Hs = H rounded up to 4)
    uint16_t *w_hi;        // tensor cores: per k-block {hi, lo} fp16 tiles of W*scale, K-major SW128
    uint16_t *w_lo;        //          (unused; the lo tile follows its hi tile inside w_hi)
    float *part_m;         // [slots] running max of each (tile, bag) segment
    float *part_s;         // [slots] sum of exp(z - m)
    float *part_v;         // [slots][H] sum of exp(z - m) * h
    int tile_rows;         // rows per softmax partial (64: FFMA CTA tile / 16: tensor-core consumer warp)
    size_t bytes;
};
// Partial slot of (tile t, bag b): t + b.  Walking the context rows in order, each new
// (tile, bag) pair increments t or b (or both), so t + b is unique; needs n_tiles + B slots.  This holds for packed
// batches as well (rows and bags still increase together), with n_tiles counted over their N rows.
EncodeWorkspace carve_encode_workspace(const c2v_dims *d, int B, int L, void *base);
EncodeWorkspace carve_encode_workspace_n(const c2v_dims *d, int B, long long N, void *base, int **row_bag);

struct EncodeArgs {
    const long long *starts, *paths, *ends;
    const float *emb_t, *emb_p, *ln_g, *ln_b, *attn;
    long long T, P;
    int Et, Ep, H, D;
    int L;
    long long N;            // B * L context rows
    int n_tiles;
    float drop_p;           // 0 => no dropout
    float drop_scale;       // 1/(1-p)
    unsigned long long seed;
    float *attention;       // [N] raw masked scores z (finalize turns them into softmax weights)
    float *stash_x;         // optional [N, H]: x = c . W^T (model.py:54) of every row, kept for the backward
    int flags;              // debug switches
    EncodeWorkspace ws;
    // packed (CSR) batches only, NULL for [B, L] ones: bag b owns rows bag_off[b] .. bag_off[b+1]-1 (1 <= length <= L),
    // row_bag [N] maps a row to its bag (built by launch_row_bag).  Kept behind every other field so that the padded
    // kernels see the same parameter layout.
    const long long *bag_off;
    const int *row_bag;
    int n_bags;
    // C2V_DROPOUT_SEED_ON_DEVICE: the dropout key is *seed_dev, loaded at run time by the SEED_DEV instantiations (so that
    // a captured CUDA graph draws a fresh key at every replay); NULL otherwise.  Behind every other field, like bag_off.
    const unsigned long long *seed_dev;
};

#ifdef __CUDACC__
// Row -> bag, first row of a bag, and the Philox row counter of the dropout mask.  A packed context j of bag b draws the
// counter b * L + j: the counter the same context has in the [B, L] layout, so both layouts share one mask.
template <bool PACKED>
__device__ __forceinline__ long long bag_of_row(const EncodeArgs &a, long long row)
{
    if (!PACKED) return row / a.L;
    long long b = a.row_bag[row];
    return b < 0 ? 0 : (b >= a.n_bags ? a.n_bags - 1 : b);
}
template <bool PACKED>
__device__ __forceinline__ long long bag_first_row(const EncodeArgs &a, long long bag)
{
    if (!PACKED) return bag * a.L;
    bag = bag < 0 ? 0 : (bag > a.n_bags ? a.n_bags : bag);      // bag_off has n_bags + 1 entries
    long long r = a.bag_off[bag];
    return r < 0 ? 0 : (r > a.N ? a.N : r);
}
template <bool PACKED>
__device__ __forceinline__ long long dropout_row(const EncodeArgs &a, long long row, long long bag)
{
    return PACKED ? bag * a.L + (row - bag_first_row<true>(a, bag)) : row;
}
// The Philox key of the dropout mask: the launch parameter, or (SEED_DEV) the key the caller keeps in device memory.  Read
// after pdl_wait(): the kernel that wrote the key may be the one this launch overlaps.
template <bool SEED_DEV>
__device__ __forceinline__ unsigned long long dropout_key(const EncodeArgs &a)
{
    return SEED_DEV ? *a.seed_dev : a.seed;
}
#endif
int launch_row_bag(const long long *bag_off, int B, long long N, int *row_bag, cudaStream_t st);

// ---------------------------------------------------------------------------------
// deterministic mode (c2v_set_deterministic, per host thread): every float sum of the training step runs in a fixed
// order instead of through atomics (c2v_deterministic.cu)
// ---------------------------------------------------------------------------------
bool deterministic();
// matmul precision (c2v_set_matmul_precision, per host thread): true under C2V_MATMUL_TF32, where the tensor-core GEMMs of
// the encode, its backward and the label head launch their OnePass instantiations (c2v_tc_ptx.cuh)
bool matmul_tf32();
constexpr int kDetSlabs = 64;          // per-CTA partial slabs of dW (tensor-core CTAs per window / CUDA-core row splits)
constexpr int kDetRowSlabs = 512;      // per-CTA partials of d attention / d gamma / d beta (caps the row kernels' grids)
constexpr int kDetLabelSplits = 32;    // label splits of d code_vector on the tensor cores
// out[i] (+)= sum over s = 0 .. n_slabs-1, in that order, of src[s * slab_stride + i], i < n
int launch_det_slab_sum(const float *src, int n_slabs, size_t slab_stride, size_t n, float *out, bool accumulate,
                        cudaStream_t st);
// the same over n_out * seg columns, column i going to out[i / seg][i % seg] (n_out <= 3), in one launch
int launch_det_slab_sum3(const float *src, int n_slabs, size_t slab_stride, size_t seg, int n_out, float *const *out,
                         bool accumulate, cudaStream_t st);
// workspace of launch_det_embed_grads for N context rows (tables of up to `vocab` rows, rows up to E floats)
size_t det_embed_workspace_bytes(long long N, int E);
// Embedding-table gradient from the per-context rows dc [N, D] (D = 2 Et + Ep: start | path | end sub-vectors):
// terminal (path = false) sums columns [0, Et) of row r into row starts[r] and [Et + Ep, D) into row ends[r], path sums
// [Et, Et + Ep) into row paths[r]; contexts with attention exactly 0 are left out (their rows are 0).  Sorted keys
// row << bits | entry, fixed-size chunks summed in key order, chunk partials of rows that span chunks summed in chunk
// order; one write per row: grad[row] += sum, or grad[slot[row]] += sum with a slot map.
int launch_det_embed_grads(const EncodeArgs &a, const float *att, const float *dc, bool path, float *grad, const int *slot,
                           void *ws, size_t ws_bytes, cudaStream_t st);

int launch_prepare_weights(const c2v_dims *d, const float *W, EncodeWorkspace &ws, bool tcgen05,
                           cudaStream_t st);
int launch_encode_ffma(const EncodeArgs &a, cudaStream_t st);
int launch_encode_tcgen05(const EncodeArgs &a, cudaStream_t st);
bool tcgen05_shape_ok(const c2v_dims *d);
int launch_encode_finalize(const EncodeArgs &a, int B, float *code_vector, cudaStream_t st);

// Generic fp32 GEMM with bias on CUDA cores: C[m,n] = sum_k A(m,k) * B(k,n) (+ bias[n]),
// element strides given explicitly so every transpose combination is one kernel.
int launch_sgemm(int M, int N, int K, const float *A, long long a_sm, long long a_sk,
                 const float *B, long long b_sk, long long b_sn, const float *bias, float *C,
                 long long c_sm, bool accumulate, cudaStream_t st);
// fused loss / dlogits modes of the label GEMM (c2v_label_tcgen05.cu)
struct LabelLossArgs {
    const long long *label;      // [B]
    float *loss;                 // out: mean NLL (or NULL)
    float *lse_out;              // out: [B] logsumexp of every row (or NULL)
    const float *dlogits_lse;    // in: [B] -> `out` receives d loss / d logits instead of the logits (or NULL)
    float dscale;                // dlogits scale: 1 / B (mean) ...
    const float *dscale_ptr;     // ... times *dscale_ptr when not NULL (the upstream gradient of the scalar loss, on the device)
    // angular-margin head (model.py:71-80) when not NULL: [B + C] = 1 / max(|cv_b|, 1e-12) then 1 / max(|W_c|, 1e-12).
    // The logits are s cos (s phi(cos) at the label), the bias is ignored, and dlogits mode writes d loss / d (cv . W^T).
    const float *inv_norms;
    float cos_m, sin_m, inverse_temp;
    // top-k mode when topk_k > 0 (label_topk_workspace_bytes of workspace, no other output, label not read): the topk_k
    // largest logits of every row, value descending then column ascending -> topk_idx / topk_val [B, topk_k], and
    // topk_prob (or NULL) = their softmax probabilities.  With inv_norms the logits are s cos without the margin.
    int topk_k;
    long long *topk_idx;
    float *topk_val, *topk_prob;
    const struct LossOptArgs *opts;   // criterion options (c2v_*_opts), or NULL: weights 1, mean, no ignore_index
};
// criterion options of the loss / dlogits modes, from a checked c2v_loss_options
struct LossOptArgs {
    const float *weight;         // [C] class weights or NULL (all 1)
    long long ignore_index;
    float eps;                   // label smoothing, in [0, 1]
    int reduction;               // C2V_REDUCTION_*
    const float *row_grad;       // dlogits mode, reduction none: [B] upstream gradient of the row losses
    float *coef;                 // [2 B + 1] row coefficients: written by the loss mode, read by the dlogits mode
    void *part;                  // loss mode: label_loss_opts_bytes of workspace for the partials
};
size_t label_loss_opts_bytes(const c2v_dims *d, int B);
size_t label_topk_workspace_bytes(const c2v_dims *d, int B, int k);
float *label_topk_inv_norms(const c2v_dims *d, int B, int k, void *ws);     // where the angular head's inv_norms go
int launch_label_tcgen05_ex(const c2v_dims *d, const float *cv, int B, const float *Wout, const float *bias,
                            float *out, long long *argmax, float *maxval, void *ws, size_t ws_bytes, bool reuse_prep,
                            cudaStream_t st, const LabelLossArgs *la);
// similarity search over a code-vector bank on the label GEMM (c2v_knn_*): top-k mode when k > 0, pairs mode otherwise
struct KnnArgs {
    const float *bank; long long N; int H;
    const float *queries; int Q;
    const long long *exclude; int X;                          // [Q, X] or NULL
    void *prep, *ws; bool reuse_prep;                         // knn_prep_bytes / knn_query_bytes
    int k; long long *indices; float *sims;                   // top-k
    float threshold; long long self_offset, query_base, capacity;    // pairs
    long long *pair_query, *pair_index; float *pair_sim; long long *count;
};
size_t knn_prep_bytes(long long N, int H);
size_t knn_query_bytes(long long N, int H, int Q, int k);
int launch_knn_prepare(const float *bank, long long N, int H, void *prep, cudaStream_t st);
int launch_knn(const KnnArgs &a, cudaStream_t st);

// ---------------------------------------------------------------------------------
// device helpers
// ---------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// tanh with <= ~3e-7 absolute error from two MUFU ops: 1 - 2/(e^{2x}+1).
// (tanh.approx.f32 has 2^-11 relative error and would eat the 1e-4 parity budget.)
__device__ __forceinline__ float tanh_accurate(float x) {
    const float e = __expf(2.0f * x);            // inf for large x -> 1, 0 for very negative -> -1
    return 1.0f - __fdividef(2.0f, e + 1.0f);
}

// Philox4x32-10 (Salmon et al. 2011), counter-based: the dropout mask of element
// (row, col) is output [col & 3] of the block with counter (row_lo, row_hi, col >> 2, 0)
// and key (seed_lo, seed_hi); backward regenerates it from the same triple.
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
    const unsigned M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const unsigned hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
        const unsigned hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
        ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
        key.x += W0; key.y += W1;
    }
    return ctr;
}
__device__ __forceinline__ uint4 dropout_bits(unsigned long long seed, long long row, int col4) {
    return philox4x32_10(make_uint4((unsigned)row, (unsigned)((unsigned long long)row >> 32),
                                    (unsigned)col4, 0u),
                         make_uint2((unsigned)seed, (unsigned)(seed >> 32)));
}
// keep iff uniform24(bits) >= p ; returns the multiplicative mask (0 or 1/(1-p))
__device__ __forceinline__ float dropout_mul(unsigned bits, float p, float scale) {
    const float u = (float)(bits >> 8) * (1.0f / 16777216.0f);
    return u >= p ? scale : 0.0f;
}
__device__ __forceinline__ float dropout_mask_at(unsigned long long seed, long long row, int col,
                                                 float p, float scale) {
    const uint4 b = dropout_bits(seed, row, col >> 2);
    const unsigned w = (col & 3) == 0 ? b.x : (col & 3) == 1 ? b.y : (col & 3) == 2 ? b.z : b.w;
    return dropout_mul(w, p, scale);
}

// 128-bit reduction without a return value (REDG.E.ADD.F32x4): the scatter-add of gradient rows needs no old value, and
// atomicAdd(float4 *) compiles to ATOMG (the returning form) even when the result is dropped.
__device__ __forceinline__ void red_add_v4(float *addr, float4 v) {
    asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};"
                 ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async4(void *smem, const void *gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}
#endif  // __CUDACC__

}  // namespace c2v

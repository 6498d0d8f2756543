// c2v_api.cu -- the extern "C" surface declared in include/c2v_b200.h.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>

#include "c2v_common.cuh"

namespace c2v {

long long g_launches = 0;
bool pdl_enabled()
{
    static int on = -1;
    if (on < 0) { const char *e = getenv("C2V_NO_PDL"); on = (e && e[0] == '1') ? 0 : 1; }
    return on == 1;
}
static thread_local char g_err[512] = "";
thread_local bool g_pdl_this_call = true;
static thread_local int g_matmul = C2V_MATMUL_IEEE;
bool matmul_tf32() { return g_matmul == C2V_MATMUL_TF32; }

void set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

int launch_transpose_w(const float *W, float *Wt, int H, int D, int Hs, cudaStream_t st);
int launch_split_w_tcgen05(const c2v_dims *d, const float *W, EncodeWorkspace &ws, cudaStream_t st);
int launch_angular(const c2v_dims *d, const c2v_params *p, const float *cv, const long long *label,
                   int B, float margin, float inverse_temp, float *out, float *scratch,
                   cudaStream_t st, float *cos_out);
int launch_angular_backward(const c2v_dims *d, const c2v_params *p, const float *cv, const long long *label, int B,
                            float margin, float inverse_temp, const float *cosine, const float *inv_cv, const float *inv_w,
                            float *d_out_inplace, float *d_cv, float *d_w, float *sums, cudaStream_t st);
int launch_loss_argmax(const float *out, const long long *label, int B, long long C, float *loss,
                       long long *argmax, float *maxval, float *d_out, cudaStream_t st);
int launch_loss_argmax_opts(const float *out, const long long *label, int B, long long C, const LossOptArgs &o, float *loss,
                            long long *argmax, float *maxval, float *d_out, cudaStream_t st);
int launch_row_inv_norm(const float *X, long long rows, int H, float *inv, cudaStream_t st);
int launch_angular_project(float *d, const float *x, const float *inv, long long rows, int H, cudaStream_t st);
int launch_colsum(const float *X, int B, long long C, float *out, cudaStream_t st);
int launch_encode_backward(const c2v_dims *d, const c2v_params *p, const EncodeArgs &a, int B,
                           const float *cv, const float *attention, const float *d_cv,
                           const float *d_att, const c2v_grads *g, void *ws, size_t ws_bytes,
                           cudaStream_t st, const float *x_stash, int phase, const c2v_row_slots *slots);
size_t encode_backward_workspace_bytes(const c2v_dims *d, int B, int L);
size_t encode_backward_workspace_bytes_n(const c2v_dims *d, int B, long long N, bool packed);
bool label_tcgen05_shape_ok(const c2v_dims *d);
bool label_backward_tc_ok(const c2v_dims *d);
int label_w_image(const c2v_dims *d, const float *Wout, int B, void *ws, size_t ws_bytes, bool reuse_prep, cudaStream_t st,
                  const uint8_t **img, const float **hdr, unsigned **scratch, const uint8_t **cv_img);
int launch_label_backward_tc(const c2v_dims *d, const float *cv, const float *G, int B, const uint8_t *w_img,
                             const float *w_hdr, float *d_cv, float *d_w, float *d_b, unsigned *scratch, cudaStream_t st,
                             bool absmax_ready, const uint8_t *cv_img, float *dcv_slabs);
size_t label_tcgen05_workspace_bytes(const c2v_dims *d, int B);
void set_deterministic(bool on);
bool label_ws_holds_dlogits_of(const void *ws, const float *cv, int B);

// ---- profiling hook (c2v_profile_enable / c2v_profile_read) ----------------------------
static const int kProfRing = 4096;
static bool g_prof_on = false;
static int g_prof_stride = 1;          // time every n-th encode launch (events between launches defeat
static long long g_prof_calls = 0;     // programmatic dependent launch, so a bench samples instead)
static cudaEvent_t g_prof_ev[kProfRing][2];
static bool g_prof_made = false;
static int g_prof_pending = 0;
static double g_prof_ms = 0.0;
static long long g_prof_count = 0;

static int prof_drain()
{
    for (int i = 0; i < g_prof_pending; ++i) {
        float ms = 0.0f;
        C2V_CUDA_OK(cudaEventSynchronize(g_prof_ev[i][1]));
        C2V_CUDA_OK(cudaEventElapsedTime(&ms, g_prof_ev[i][0], g_prof_ev[i][1]));
        g_prof_ms += ms;
        g_prof_count += 1;
    }
    g_prof_pending = 0;
    return C2V_OK;
}

static bool dims_ok(const c2v_dims *d)
{
    if (!d) { set_error("dims is NULL"); return false; }
    if (d->terminal_count < 1 || d->path_count < 1 || d->terminal_embed < 1 || d->path_embed < 1 ||
        d->encode < 1) {
        set_error("bad dims: T=%lld P=%lld Et=%d Ep=%d H=%d", (long long)d->terminal_count,
                  (long long)d->path_count, d->terminal_embed, d->path_embed, d->encode);
        return false;
    }
    return true;
}

// tile rows used for sizing: the smallest tile any algorithm uses (64) gives the most slots
static const int kMinTileRows = 16;   // tensor-core path: one partial per 16-row consumer warp

// N context rows; a packed batch (row_bag != NULL) gets its row -> bag map (int32 [N]) behind everything else
EncodeWorkspace carve_encode_workspace_n(const c2v_dims *d, int B, long long N, void *base, int **row_bag)
{
    EncodeWorkspace w;
    memset(&w, 0, sizeof(w));
    const int H = d->encode, D = 2 * d->terminal_embed + d->path_embed;
    const int Hs = (H + 3) / 4 * 4;
    const size_t n_tiles = (size_t)((N + kMinTileRows - 1) / kMinTileRows);
    const size_t slots = n_tiles + (size_t)B + 1;
    // tcgen05 split weights: K padded to 64-element blocks, N padded to 128 rows... sized generously
    size_t kblocks = (size_t)(D + 63) / 64 + 3;                // +3: per-sub-vector padding
    const size_t padded = (H > 128 || d->terminal_embed > 128) ? 12 : 6;   // K1e pads each sub-vector to 128 / 256 k
    if (kblocks < padded) kblocks = padded;
    const size_t hp = (size_t)(H + 127) / 128 * 128;
    char *p = static_cast<char *>(base);
    size_t o = 0;
    auto take = [&](size_t bytes) { char *r = p ? p + o : nullptr; o += align_up(bytes, 1024); return r; };
    w.status = reinterpret_cast<long long *>(take(256));
    w.prep_hdr = reinterpret_cast<float *>(take(256));
    w.w_t = reinterpret_cast<float *>(take((size_t)D * Hs * sizeof(float)));
    // per k-block: {hi tile, lo tile}, each [hp x 64] fp16 in the UMMA shared-memory layout
    w.w_hi = reinterpret_cast<uint16_t *>(take(2 * kblocks * hp * 64 * sizeof(uint16_t)));
    w.w_lo = nullptr;
    w.part_m = reinterpret_cast<float *>(take(slots * sizeof(float)));
    w.part_s = reinterpret_cast<float *>(take(slots * sizeof(float)));
    w.part_v = reinterpret_cast<float *>(take(slots * (size_t)H * sizeof(float)));
    if (row_bag) *row_bag = reinterpret_cast<int *>(take((size_t)N * sizeof(int)));
    w.bytes = o;
    return w;
}

EncodeWorkspace carve_encode_workspace(const c2v_dims *d, int B, int L, void *base)
{
    return carve_encode_workspace_n(d, B, (long long)B * L, base, nullptr);
}

// c2v_dropout.training: bit 0 = dropout on, C2V_DROPOUT_SEED_ON_DEVICE = `seed` is the device address of the key.
// Checked before any CUDA call.
static bool dropout_ok(const char *fn, const c2v_dropout *drop)
{
    if (!drop) return true;
    if (drop->training & ~(1 | C2V_DROPOUT_SEED_ON_DEVICE)) {
        set_error("%s: unknown dropout flag bits 0x%x", fn, (unsigned)drop->training);
        return false;
    }
    if ((drop->training & C2V_DROPOUT_SEED_ON_DEVICE) && (drop->seed == 0 || (drop->seed & 7))) {
        set_error("%s: C2V_DROPOUT_SEED_ON_DEVICE needs the 8-byte aligned device address of the key in `seed`", fn);
        return false;
    }
    return true;
}

// the dropout fields of EncodeArgs (model.py:26-29): dropout runs when bit 0 is set and 0 < p < 1
static void set_dropout(EncodeArgs &a, const c2v_dropout *drop)
{
    a.drop_p = 0.0f; a.drop_scale = 1.0f; a.seed = 0; a.seed_dev = nullptr;
    if (drop && (drop->training & 1) && drop->p > 0.0f && drop->p < 1.0f) {
        a.drop_p = drop->p; a.drop_scale = 1.0f / (1.0f - drop->p);
        if (drop->training & C2V_DROPOUT_SEED_ON_DEVICE)
            a.seed_dev = reinterpret_cast<const unsigned long long *>(static_cast<uintptr_t>(drop->seed));
        else
            a.seed = drop->seed;
    }
}

// splitmix64 (Steele, Lea and Flood 2014): the output for the generator state x
__device__ __forceinline__ unsigned long long splitmix64(unsigned long long x)
{
    unsigned long long z = x + 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

__global__ void next_dropout_key_kernel(long long *state, unsigned long long *key)
{
    const long long counter = state[1];
    *key = splitmix64((unsigned long long)state[0] + (unsigned long long)counter);
    state[1] = counter + 1;
}

}  // namespace c2v

using namespace c2v;

extern "C" {

int c2v_abi_version(void) { return C2V_ABI_VERSION; }

int c2v_set_deterministic(int32_t on)
{
    set_deterministic(on != 0);
    return C2V_OK;
}

int c2v_get_deterministic(void) { return deterministic() ? 1 : 0; }

int c2v_set_matmul_precision(int32_t mode)
{
    if (mode != C2V_MATMUL_IEEE && mode != C2V_MATMUL_TF32) {
        set_error("c2v_set_matmul_precision: mode %d is neither C2V_MATMUL_IEEE (0) nor C2V_MATMUL_TF32 (1)", (int)mode);
        return C2V_EINVAL;
    }
    g_matmul = mode;
    return C2V_OK;
}

int c2v_get_matmul_precision(void) { return g_matmul; }
const char *c2v_last_error(void) { return g_err; }
int64_t c2v_launch_count(void) { return __atomic_load_n(&g_launches, __ATOMIC_RELAXED); }

int c2v_get_device_info(int device, c2v_device_info *out)
{
    if (!out) { set_error("out is NULL"); return C2V_EINVAL; }
    cudaDeviceProp pr;
    C2V_CUDA_OK(cudaGetDeviceProperties(&pr, device));
    out->cc_major = pr.major; out->cc_minor = pr.minor; out->sm_count = pr.multiProcessorCount;
    out->reserved = 0;
    out->global_mem_bytes = (int64_t)pr.totalGlobalMem;
    out->smem_per_block_optin = (int64_t)pr.sharedMemPerBlockOptin;
    return C2V_OK;
}

int c2v_encode_supports_tcgen05(const c2v_dims *d)
{
    if (!dims_ok(d)) return 0;
    return tcgen05_shape_ok(d) ? 1 : 0;
}

size_t c2v_encode_workspace_bytes(const c2v_dims *d, int32_t B, int32_t L)
{
    if (!dims_ok(d) || B < 1 || L < 1) return 0;
    return carve_encode_workspace(d, B, L, nullptr).bytes;
}

int c2v_encode_forward(const c2v_dims *d, const c2v_params *p, const int64_t *starts,
                       const int64_t *paths, const int64_t *ends, int32_t B, int32_t L,
                       const c2v_dropout *drop, float *code_vector, float *attention,
                       void *workspace, size_t workspace_bytes, int32_t algo, void *stream)
{
    return c2v_encode_forward_stash(d, p, starts, paths, ends, B, L, drop, code_vector, attention, nullptr, workspace,
                                    workspace_bytes, algo, stream);
}

// The encode of both layouts once the caller's argument checks have passed: [B, L] (offsets == NULL, N = B * L) or
// packed (bag b = rows offsets[b] .. offsets[b+1]-1, N rows in all).
static int encode_forward_impl(const char *fn, const c2v_dims *d, const c2v_params *p, const int64_t *starts,
                               const int64_t *paths, const int64_t *ends, const int64_t *offsets, int32_t B, long long N,
                               int32_t L, const c2v_dropout *drop, float *code_vector, float *attention, float *x_stash,
                               void *workspace, size_t workspace_bytes, int32_t algo, void *stream)
{
    if (!p->terminal_embedding || !p->path_embedding || !p->input_linear || !p->ln_weight ||
        !p->ln_bias || !p->attention) {
        set_error("%s: NULL parameter pointer", fn);
        return C2V_EINVAL;
    }
    if (!dropout_ok(fn, drop)) return C2V_EINVAL;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    int *row_bag = nullptr;
    EncodeWorkspace ws = carve_encode_workspace_n(d, B, N, workspace, offsets ? &row_bag : nullptr);
    if (ws.bytes > workspace_bytes) {
        set_error("workspace too small: %zu < %zu", workspace_bytes, ws.bytes);
        return C2V_EWORKSPACE;
    }
    const bool reuse_prep = (algo & C2V_FLAG_REUSE_PREP) != 0;
    g_pdl_this_call = (algo & C2V_FLAG_NO_PDL) == 0 && x_stash == nullptr;
    algo &= 0xff;
    bool use_tc;
    if (algo == C2V_ALGO_TCGEN05) {
        if (!tcgen05_shape_ok(d)) {
            set_error("tcgen05 encode does not support Et=%d Ep=%d H=%d", d->terminal_embed,
                      d->path_embed, d->encode);
            return C2V_EUNSUPPORTED;
        }
        use_tc = true;
    } else if (algo == C2V_ALGO_FFMA) {
        use_tc = false;
    } else if (algo == C2V_ALGO_AUTO) {
        use_tc = tcgen05_shape_ok(d);
    } else {
        set_error("%s: unknown algo %d", fn, algo);
        return C2V_EINVAL;
    }

    EncodeArgs a;
    memset(&a, 0, sizeof(a));
    a.starts = reinterpret_cast<const long long *>(starts);
    a.paths = reinterpret_cast<const long long *>(paths);
    a.ends = reinterpret_cast<const long long *>(ends);
    a.emb_t = p->terminal_embedding; a.emb_p = p->path_embedding;
    a.ln_g = p->ln_weight; a.ln_b = p->ln_bias; a.attn = p->attention;
    a.T = d->terminal_count; a.P = d->path_count;
    a.Et = d->terminal_embed; a.Ep = d->path_embed; a.H = d->encode;
    a.D = 2 * a.Et + a.Ep;
    a.L = L; a.N = N;
    set_dropout(a, drop);
    a.attention = attention;
    a.stash_x = x_stash;
    a.flags = 0;
    a.bag_off = reinterpret_cast<const long long *>(offsets);
    a.row_bag = row_bag;
    a.n_bags = B;
    // rows per softmax partial: 64-row CTA tiles (FFMA) or 16-row consumer warps (tensor cores)
    ws.tile_rows = use_tc ? 16 : 64;
    const int cta_rows = use_tc ? 128 : 64;
    a.n_tiles = (int)((a.N + cta_rows - 1) / cta_rows);
    a.ws = ws;

    // status[0] accumulates out-of-range indices during the encode kernel; the finalize kernel publishes it to
    // status[3] and clears it for the next call, so a steady-state call (REUSE_PREP) needs no memset and the encode
    // kernel can be launched as a programmatic dependent of whatever ran before it on the stream.
    if (!reuse_prep) C2V_CUDA_OK(cudaMemsetAsync(ws.status, 0, 256, st));
#ifdef TM_INSTRUMENT
    C2V_CUDA_OK(cudaMemsetAsync(ws.status + 16, 0x7f, 8, st));   // min-reduced slots of the instrumented build
    C2V_CUDA_OK(cudaMemsetAsync(ws.status + 20, 0x7f, 8, st));
#endif
    int rc = C2V_OK;
    if (!reuse_prep)
        rc = use_tc ? launch_split_w_tcgen05(d, p->input_linear, a.ws, st)
                    : launch_transpose_w(p->input_linear, ws.w_t, a.H, a.D, (a.H + 3) / 4 * 4, st);
    if (rc != C2V_OK) return rc;
    if (row_bag) {
        rc = launch_row_bag(a.bag_off, B, N, row_bag, st);
        if (rc != C2V_OK) return rc;
    }
    int slot = -1;
    if (g_prof_on && (g_prof_calls++ % g_prof_stride) == 0) {
        if (g_prof_pending == kProfRing) { rc = prof_drain(); if (rc != C2V_OK) return rc; }
        slot = g_prof_pending;
        C2V_CUDA_OK(cudaEventRecord(g_prof_ev[slot][0], st));
    }
    rc = use_tc ? launch_encode_tcgen05(a, st) : launch_encode_ffma(a, st);
    if (rc != C2V_OK) return rc;
    if (slot >= 0) {
        C2V_CUDA_OK(cudaEventRecord(g_prof_ev[slot][1], st));
        g_prof_pending = slot + 1;
    }
    return launch_encode_finalize(a, B, code_vector, st);
}

int c2v_encode_forward_stash(const c2v_dims *d, const c2v_params *p, const int64_t *starts,
                             const int64_t *paths, const int64_t *ends, int32_t B, int32_t L,
                             const c2v_dropout *drop, float *code_vector, float *attention, float *x_stash,
                             void *workspace, size_t workspace_bytes, int32_t algo, void *stream)
{
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !starts || !paths || !ends || !code_vector || !attention || !workspace) {
        set_error("c2v_encode_forward: NULL pointer argument");
        return C2V_EINVAL;
    }
    if (B < 1 || L < 1) { set_error("c2v_encode_forward: B=%d L=%d", B, L); return C2V_EINVAL; }
    return encode_forward_impl("c2v_encode_forward", d, p, starts, paths, ends, nullptr, B, (long long)B * L, L, drop,
                               code_vector, attention, x_stash, workspace, workspace_bytes, algo, stream);
}

// shape checks of the packed entry points
static bool packed_shape_ok(const char *fn, int32_t B, int64_t N, int32_t L)
{
    if (B < 1 || L < 1 || N < B || N > (int64_t)B * L) {
        set_error("%s: B=%d N=%lld L=%d: needs B >= 1, L >= 1 and B <= N <= B * L (every bag holds 1 .. L contexts)", fn, B,
                  (long long)N, L);
        return false;
    }
    return true;
}

size_t c2v_encode_packed_workspace_bytes(const c2v_dims *d, int32_t B, int64_t N)
{
    if (!dims_ok(d) || B < 1 || N < B) return 0;
    int *row_bag = nullptr;
    return carve_encode_workspace_n(d, B, N, nullptr, &row_bag).bytes;
}

int c2v_encode_forward_packed(const c2v_dims *d, const c2v_params *p, const int64_t *starts, const int64_t *paths,
                              const int64_t *ends, const int64_t *offsets, int32_t B, int64_t N, int32_t L,
                              const c2v_dropout *drop, float *code_vector, float *attention, float *x_stash,
                              void *workspace, size_t workspace_bytes, int32_t algo, void *stream)
{
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !starts || !paths || !ends || !offsets || !code_vector || !attention || !workspace) {
        set_error("c2v_encode_forward_packed: NULL pointer argument");
        return C2V_EINVAL;
    }
    if (!packed_shape_ok("c2v_encode_forward_packed", B, N, L)) return C2V_EINVAL;
    return encode_forward_impl("c2v_encode_forward_packed", d, p, starts, paths, ends, offsets, B, N, L, drop, code_vector,
                               attention, x_stash, workspace, workspace_bytes, algo, stream);
}

int c2v_profile_enable(int32_t on)
{
    if (on && !g_prof_made) {
        for (int i = 0; i < kProfRing; ++i)
            for (int j = 0; j < 2; ++j) C2V_CUDA_OK(cudaEventCreate(&g_prof_ev[i][j]));
        g_prof_made = true;
    }
    g_prof_on = on != 0;
    g_prof_stride = on > 1 ? on : 1;
    g_prof_calls = 0;
    g_prof_pending = 0; g_prof_ms = 0.0; g_prof_count = 0;
    return C2V_OK;
}

int c2v_profile_read(double *kernel_ms, int64_t *launches)
{
    int rc = prof_drain();
    if (rc != C2V_OK) return rc;
    if (kernel_ms) *kernel_ms = g_prof_ms;
    if (launches) *launches = g_prof_count;
    return C2V_OK;
}

int64_t c2v_workspace_status(void *workspace, void *stream)
{
    if (!workspace) { set_error("workspace is NULL"); return C2V_EINVAL; }
    long long v = 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    C2V_CUDA_OK(cudaMemcpyAsync(&v, static_cast<const char *>(workspace) + 24, sizeof(v), cudaMemcpyDeviceToHost, st));
    C2V_CUDA_OK(cudaStreamSynchronize(st));
    return v;
}

int c2v_workspace_set_status_mirror(void *workspace, int64_t *pinned_host_word, void *stream)
{
    if (!workspace) { set_error("workspace is NULL"); return C2V_EINVAL; }
    long long hdr[2] = {0, 0};
    if (pinned_host_word) {
        cudaPointerAttributes at;
        C2V_CUDA_OK(cudaPointerGetAttributes(&at, pinned_host_word));
        if (at.type != cudaMemoryTypeHost || !at.devicePointer) {
            set_error("c2v_workspace_set_status_mirror: the mirror must be pinned (page-locked, device-mapped) host memory");
            return C2V_EINVAL;
        }
        hdr[0] = (long long)reinterpret_cast<uintptr_t>(at.devicePointer);
        hdr[1] = hdr[0] ^ C2V_MIRROR_MAGIC;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    // pageable source: the copy is staged before the call returns, so the stack buffer may go away
    C2V_CUDA_OK(cudaMemcpyAsync(static_cast<char *>(workspace) + 512, hdr, sizeof(hdr), cudaMemcpyHostToDevice, st));
    return C2V_OK;
}

size_t c2v_label_workspace_bytes(const c2v_dims *d, int32_t B)
{
    if (!dims_ok(d) || B < 1) return 0;
    // split fp16 images of cv and W_out for the tcgen05 label GEMM (unused by the FFMA path); deterministic mode: then
    // the label splits' d code_vector slabs of c2v_label_backward_ws
    return align_up(label_tcgen05_workspace_bytes(d, B), 1024) +
           (deterministic() ? align_up((size_t)kDetLabelSplits * B * d->encode * 4, 1024) : 0);
}

// What every tensor-core label entry point does once its own argument checks have passed: apply the flags of `algo`
// (C2V_FLAG_REUSE_PREP, C2V_FLAG_NO_PDL) and launch the label GEMM in the mode `la` selects (NULL: the logits, with the
// fused arg-max when argmax / maxval are given).  The angular head ignores output_bias.
static int label_gemm(const c2v_dims *d, const c2v_params *p, const float *code_vector, int32_t B, float *out,
                      int64_t *argmax, float *maxval, void *workspace, size_t workspace_bytes, int32_t algo, void *stream,
                      const LabelLossArgs *la)
{
    g_pdl_this_call = (algo & C2V_FLAG_NO_PDL) == 0;
    return launch_label_tcgen05_ex(d, code_vector, B, p->output_weight, p->output_bias, out,
                                   reinterpret_cast<long long *>(argmax), maxval, workspace, workspace_bytes,
                                   (algo & C2V_FLAG_REUSE_PREP) != 0, static_cast<cudaStream_t>(stream), la);
}

// the angular head's inverse row norms: inv[0, B) of the code vectors, then inv[B, B + C) of the W_out rows
static int angular_inv_norms(const c2v_dims *d, const c2v_params *p, const float *code_vector, int32_t B, float *inv,
                             void *stream)
{
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = launch_row_inv_norm(code_vector, B, d->encode, inv, st);
    return rc != C2V_OK ? rc : launch_row_inv_norm(p->output_weight, d->label_count, d->encode, inv + B, st);
}

int c2v_label_logits(const c2v_dims *d, const c2v_params *p, const float *code_vector, int32_t B,
                     float *outputs, void *workspace, size_t workspace_bytes, int32_t algo,
                     void *stream)
{
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !outputs || B < 1 || d->label_count < 1) {
        set_error("c2v_label_logits: bad argument");
        return C2V_EINVAL;
    }
    return c2v_label_logits_argmax(d, p, code_vector, B, outputs, nullptr, nullptr, workspace, workspace_bytes, algo, stream);
}

int c2v_label_logits_argmax(const c2v_dims *d, const c2v_params *p, const float *code_vector, int32_t B,
                            float *outputs, int64_t *argmax, float *maxval, void *workspace,
                            size_t workspace_bytes, int32_t algo, void *stream)
{
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || B < 1 || d->label_count < 1 || (!outputs && !argmax && !maxval)) {
        set_error("c2v_label_logits_argmax: bad argument");
        return C2V_EINVAL;
    }
    if (!outputs && !c2v_label_loss_supported(d, B)) {       // arg-max without the logits needs the fused tensor-core epilogue
        set_error("c2v_label_logits_argmax: outputs == NULL needs encode_size %% 4 == 0, <= 256 and B <= 2048");
        return C2V_EUNSUPPORTED;
    }
    const int base_algo = algo & 0xff;
    if (base_algo == C2V_ALGO_TCGEN05 || (base_algo == C2V_ALGO_AUTO && label_tcgen05_shape_ok(d)))
        return label_gemm(d, p, code_vector, B, outputs, argmax, maxval, workspace, workspace_bytes, algo, stream, nullptr);
    if (!outputs) {
        set_error("c2v_label_logits_argmax: outputs == NULL needs the tensor-core label GEMM (got algo %d)", base_algo);
        return C2V_EINVAL;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int H = d->encode;
    const long long C = d->label_count;
    // outputs[b,c] = sum_h cv[b,h] * W_out[c,h] + bias[c]   (model.py:83)
    int rc = launch_sgemm(B, (int)C, H, code_vector, H, 1, p->output_weight, 1, H, p->output_bias, outputs, C, false, st);
    if (rc != C2V_OK || (!argmax && !maxval)) return rc;
    return launch_loss_argmax(outputs, nullptr, B, C, nullptr, reinterpret_cast<long long *>(argmax), maxval, nullptr, st);
}

int c2v_label_loss_supported(const c2v_dims *d, int32_t B)
{
    if (!dims_ok(d) || B < 1) return 0;
    return (label_tcgen05_shape_ok(d) && B <= 2048) ? 1 : 0;
}

int c2v_label_loss_argmax(const c2v_dims *d, const c2v_params *p, const float *code_vector, const int64_t *label,
                          int32_t B, float *outputs, float *loss, float *lse, int64_t *argmax, float *maxval,
                          void *workspace, size_t workspace_bytes, int32_t algo, void *stream)
{
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !label || B < 1 || d->label_count < 1 || (!loss && !lse)) {
        set_error("c2v_label_loss_argmax: bad argument");
        return C2V_EINVAL;
    }
    if (!c2v_label_loss_supported(d, B)) {
        set_error("c2v_label_loss_argmax: the fused loss needs encode_size %% 4 == 0, <= 256 and B <= 2048 (got %d, %d); use "
                  "c2v_label_logits + c2v_loss_argmax", d->encode, B);
        return C2V_EUNSUPPORTED;
    }
    LabelLossArgs la = {};
    la.label = reinterpret_cast<const long long *>(label); la.loss = loss; la.lse_out = lse;
    return label_gemm(d, p, code_vector, B, outputs, argmax, maxval, workspace, workspace_bytes, algo, stream, &la);
}

int c2v_label_dlogits(const c2v_dims *d, const c2v_params *p, const float *code_vector, const int64_t *label,
                      const float *lse, int32_t B, float scale, const float *scale_device, float *d_outputs,
                      void *workspace, size_t workspace_bytes, int32_t algo, void *stream)
{
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !label || !lse || !d_outputs || B < 1 || d->label_count < 1) {
        set_error("c2v_label_dlogits: bad argument");
        return C2V_EINVAL;
    }
    if (!label_tcgen05_shape_ok(d)) {
        set_error("c2v_label_dlogits: needs encode_size %% 4 == 0 and <= 256 (got %d)", d->encode);
        return C2V_EUNSUPPORTED;
    }
    LabelLossArgs la = {};
    la.label = reinterpret_cast<const long long *>(label); la.dlogits_lse = lse; la.dscale = scale; la.dscale_ptr = scale_device;
    return label_gemm(d, p, code_vector, B, d_outputs, nullptr, nullptr, workspace, workspace_bytes, algo | C2V_FLAG_NO_PDL,
                      stream, &la);
}

int c2v_angular_loss_argmax(const c2v_dims *d, const c2v_params *p, const float *code_vector, const int64_t *label,
                            int32_t B, float margin, float inverse_temp, float *outputs, float *loss, float *lse,
                            int64_t *argmax, float *maxval, float *inv_norms, void *workspace, size_t workspace_bytes,
                            int32_t algo, void *stream)
{
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !label || !inv_norms || B < 1 || d->label_count < 1 || (!loss && !lse)) {
        set_error("c2v_angular_loss_argmax: bad argument (NULL pointer, B < 1 or neither loss nor lse)");
        return C2V_EINVAL;
    }
    if (!c2v_label_loss_supported(d, B)) {
        set_error("c2v_angular_loss_argmax: the fused loss needs encode_size %% 4 == 0, <= 256 and B <= 2048 (got %d, %d); use "
                  "c2v_angular_forward_train + c2v_loss_argmax", d->encode, B);
        return C2V_EUNSUPPORTED;
    }
    const int rc = angular_inv_norms(d, p, code_vector, B, inv_norms, stream);
    if (rc != C2V_OK) return rc;
    LabelLossArgs la = {};
    la.label = reinterpret_cast<const long long *>(label); la.loss = loss; la.lse_out = lse;
    la.inv_norms = inv_norms; la.cos_m = cosf(margin); la.sin_m = sinf(margin); la.inverse_temp = inverse_temp;
    return label_gemm(d, p, code_vector, B, outputs, argmax, maxval, workspace, workspace_bytes, algo, stream, &la);
}

int c2v_angular_dlogits(const c2v_dims *d, const c2v_params *p, const float *code_vector, const int64_t *label,
                        const float *lse, const float *inv_norms, int32_t B, float margin, float inverse_temp, float scale,
                        const float *scale_device, float *d_dot, void *workspace, size_t workspace_bytes, int32_t algo,
                        void *stream)
{
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !label || !lse || !inv_norms || !d_dot || B < 1 || d->label_count < 1) {
        set_error("c2v_angular_dlogits: bad argument (NULL pointer or B < 1)");
        return C2V_EINVAL;
    }
    if (!label_tcgen05_shape_ok(d)) {
        set_error("c2v_angular_dlogits: needs encode_size %% 4 == 0 and <= 256 (got %d)", d->encode);
        return C2V_EUNSUPPORTED;
    }
    LabelLossArgs la = {};
    la.label = reinterpret_cast<const long long *>(label); la.dlogits_lse = lse; la.dscale = scale; la.dscale_ptr = scale_device;
    la.inv_norms = inv_norms; la.cos_m = cosf(margin); la.sin_m = sinf(margin); la.inverse_temp = inverse_temp;
    return label_gemm(d, p, code_vector, B, d_dot, nullptr, nullptr, workspace, workspace_bytes, algo | C2V_FLAG_NO_PDL, stream,
                      &la);
}

// ---- criterion options (c2v_loss_options) ------------------------------------------------------------------------------
// o != NULL -> *out; every check before any CUDA call.  dlogits: the call that needs row_grad for reduction none.
static int loss_opts_ok(const char *fn, const c2v_loss_options *o, bool dlogits, LossOptArgs *out)
{
    if (!(o->label_smoothing >= 0.0f && o->label_smoothing <= 1.0f)) {          // (false for NaN)
        set_error("%s: label_smoothing %g is not in [0, 1]", fn, (double)o->label_smoothing);
        return C2V_EINVAL;
    }
    if (o->reduction != C2V_REDUCTION_MEAN && o->reduction != C2V_REDUCTION_SUM && o->reduction != C2V_REDUCTION_NONE) {
        set_error("%s: unknown reduction %d", fn, o->reduction);
        return C2V_EINVAL;
    }
    if ((uintptr_t)o->class_weight % alignof(float) != 0) {
        set_error("%s: class_weight is not 4-byte aligned", fn);
        return C2V_EINVAL;
    }
    if (dlogits && o->reduction == C2V_REDUCTION_NONE && !o->row_grad) {
        set_error("%s: reduction none needs row_grad", fn);
        return C2V_EINVAL;
    }
    *out = LossOptArgs{};
    out->weight = o->class_weight; out->ignore_index = o->ignore_index; out->eps = o->label_smoothing;
    out->reduction = o->reduction; out->row_grad = dlogits ? o->row_grad : nullptr;
    return C2V_OK;
}

size_t c2v_label_loss_opts_workspace_bytes(const c2v_dims *d, int32_t B)
{
    if (!dims_ok(d) || B < 1) return 0;
    return align_up(c2v_label_workspace_bytes(d, B), 1024) + label_loss_opts_bytes(d, B);
}

// the checks every fused loss call with options adds to those of the call it extends
static int loss_opts_call_ok(const char *fn, const c2v_dims *d, int32_t B, const c2v_loss_options *options, float *coef,
                             void *workspace, size_t workspace_bytes, LossOptArgs *oa)
{
    int rc = loss_opts_ok(fn, options, false, oa);
    if (rc != C2V_OK) return rc;
    if (!coef) { set_error("%s: coef is NULL", fn); return C2V_EINVAL; }
    const size_t need = c2v_label_loss_opts_workspace_bytes(d, B);
    if (!workspace || workspace_bytes < need) {
        set_error("%s: workspace too small: %zu < %zu", fn, workspace ? workspace_bytes : (size_t)0, need);
        return C2V_EWORKSPACE;
    }
    oa->coef = coef;
    oa->part = static_cast<uint8_t *>(workspace) + align_up(c2v_label_workspace_bytes(d, B), 1024);
    return C2V_OK;
}

int c2v_label_loss_argmax_opts(const c2v_dims *d, const c2v_params *p, const float *code_vector, const int64_t *label,
                               int32_t B, const c2v_loss_options *options, float *outputs, float *loss, float *lse,
                               float *coef, int64_t *argmax, float *maxval, void *workspace, size_t workspace_bytes,
                               int32_t algo, void *stream)
{
    if (!options)
        return c2v_label_loss_argmax(d, p, code_vector, label, B, outputs, loss, lse, argmax, maxval, workspace,
                                     workspace_bytes, algo, stream);
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !label || B < 1 || d->label_count < 1 || (!loss && !lse)) {
        set_error("c2v_label_loss_argmax_opts: bad argument");
        return C2V_EINVAL;
    }
    LossOptArgs oa;
    int rc = loss_opts_call_ok("c2v_label_loss_argmax_opts", d, B, options, coef, workspace, workspace_bytes, &oa);
    if (rc != C2V_OK) return rc;
    if (!c2v_label_loss_supported(d, B)) {
        set_error("c2v_label_loss_argmax_opts: the fused loss needs encode_size %% 4 == 0, <= 256 and B <= 2048 (got %d, %d); "
                  "use c2v_label_logits + c2v_loss_argmax_opts", d->encode, B);
        return C2V_EUNSUPPORTED;
    }
    LabelLossArgs la = {};
    la.label = reinterpret_cast<const long long *>(label); la.loss = loss; la.lse_out = lse; la.opts = &oa;
    return label_gemm(d, p, code_vector, B, outputs, argmax, maxval, workspace, workspace_bytes, algo, stream, &la);
}

int c2v_label_dlogits_opts(const c2v_dims *d, const c2v_params *p, const float *code_vector, const int64_t *label,
                           const float *lse, const float *coef, int32_t B, const c2v_loss_options *options, float scale,
                           const float *scale_device, float *d_outputs, void *workspace, size_t workspace_bytes,
                           int32_t algo, void *stream)
{
    if (!options)
        return c2v_label_dlogits(d, p, code_vector, label, lse, B, scale, scale_device, d_outputs, workspace, workspace_bytes,
                                 algo, stream);
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !label || !lse || !coef || !d_outputs || B < 1 || d->label_count < 1) {
        set_error("c2v_label_dlogits_opts: bad argument");
        return C2V_EINVAL;
    }
    LossOptArgs oa;
    const int rc = loss_opts_ok("c2v_label_dlogits_opts", options, true, &oa);
    if (rc != C2V_OK) return rc;
    if (!label_tcgen05_shape_ok(d)) {
        set_error("c2v_label_dlogits_opts: needs encode_size %% 4 == 0 and <= 256 (got %d)", d->encode);
        return C2V_EUNSUPPORTED;
    }
    oa.coef = const_cast<float *>(coef);                     // (read only in the dlogits mode)
    LabelLossArgs la = {};
    la.label = reinterpret_cast<const long long *>(label); la.dlogits_lse = lse; la.dscale = scale; la.dscale_ptr = scale_device;
    la.opts = &oa;
    return label_gemm(d, p, code_vector, B, d_outputs, nullptr, nullptr, workspace, workspace_bytes, algo | C2V_FLAG_NO_PDL,
                      stream, &la);
}

int c2v_angular_loss_argmax_opts(const c2v_dims *d, const c2v_params *p, const float *code_vector, const int64_t *label,
                                 int32_t B, float margin, float inverse_temp, const c2v_loss_options *options,
                                 float *outputs, float *loss, float *lse, float *coef, int64_t *argmax, float *maxval,
                                 float *inv_norms, void *workspace, size_t workspace_bytes, int32_t algo, void *stream)
{
    if (!options)
        return c2v_angular_loss_argmax(d, p, code_vector, label, B, margin, inverse_temp, outputs, loss, lse, argmax, maxval,
                                       inv_norms, workspace, workspace_bytes, algo, stream);
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !label || !inv_norms || B < 1 || d->label_count < 1 || (!loss && !lse)) {
        set_error("c2v_angular_loss_argmax_opts: bad argument (NULL pointer, B < 1 or neither loss nor lse)");
        return C2V_EINVAL;
    }
    LossOptArgs oa;
    int rc = loss_opts_call_ok("c2v_angular_loss_argmax_opts", d, B, options, coef, workspace, workspace_bytes, &oa);
    if (rc != C2V_OK) return rc;
    if (!c2v_label_loss_supported(d, B)) {
        set_error("c2v_angular_loss_argmax_opts: the fused loss needs encode_size %% 4 == 0, <= 256 and B <= 2048 (got %d, "
                  "%d); use c2v_angular_forward_train + c2v_loss_argmax_opts", d->encode, B);
        return C2V_EUNSUPPORTED;
    }
    rc = angular_inv_norms(d, p, code_vector, B, inv_norms, stream);
    if (rc != C2V_OK) return rc;
    LabelLossArgs la = {};
    la.label = reinterpret_cast<const long long *>(label); la.loss = loss; la.lse_out = lse; la.opts = &oa;
    la.inv_norms = inv_norms; la.cos_m = cosf(margin); la.sin_m = sinf(margin); la.inverse_temp = inverse_temp;
    return label_gemm(d, p, code_vector, B, outputs, argmax, maxval, workspace, workspace_bytes, algo, stream, &la);
}

int c2v_angular_dlogits_opts(const c2v_dims *d, const c2v_params *p, const float *code_vector, const int64_t *label,
                             const float *lse, const float *coef, const float *inv_norms, int32_t B, float margin,
                             float inverse_temp, const c2v_loss_options *options, float scale, const float *scale_device,
                             float *d_dot, void *workspace, size_t workspace_bytes, int32_t algo, void *stream)
{
    if (!options)
        return c2v_angular_dlogits(d, p, code_vector, label, lse, inv_norms, B, margin, inverse_temp, scale, scale_device,
                                   d_dot, workspace, workspace_bytes, algo, stream);
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !label || !lse || !coef || !inv_norms || !d_dot || B < 1 ||
        d->label_count < 1) {
        set_error("c2v_angular_dlogits_opts: bad argument (NULL pointer or B < 1)");
        return C2V_EINVAL;
    }
    LossOptArgs oa;
    const int rc = loss_opts_ok("c2v_angular_dlogits_opts", options, true, &oa);
    if (rc != C2V_OK) return rc;
    if (!label_tcgen05_shape_ok(d)) {
        set_error("c2v_angular_dlogits_opts: needs encode_size %% 4 == 0 and <= 256 (got %d)", d->encode);
        return C2V_EUNSUPPORTED;
    }
    oa.coef = const_cast<float *>(coef);
    LabelLossArgs la = {};
    la.label = reinterpret_cast<const long long *>(label); la.dlogits_lse = lse; la.dscale = scale; la.dscale_ptr = scale_device;
    la.inv_norms = inv_norms; la.cos_m = cosf(margin); la.sin_m = sinf(margin); la.inverse_temp = inverse_temp;
    la.opts = &oa;
    return label_gemm(d, p, code_vector, B, d_dot, nullptr, nullptr, workspace, workspace_bytes, algo | C2V_FLAG_NO_PDL, stream,
                      &la);
}

int c2v_angular_backward_ws(const c2v_dims *d, const c2v_params *p, const float *code_vector, const float *d_dot,
                            const float *inv_norms, int32_t B, float *d_code_vector, float *d_output_weight, void *workspace,
                            size_t workspace_bytes, int32_t algo, void *stream)
{
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !d_dot || !inv_norms || B < 1 || d->label_count < 1) {
        set_error("c2v_angular_backward_ws: bad argument (NULL pointer or B < 1)");
        return C2V_EINVAL;
    }
    // d_cv_raw = G . W, dW_raw = G^T . cv (the plain label backward, no bias), then the radial projection of F.normalize
    int rc = c2v_label_backward_ws(d, p, code_vector, d_dot, B, d_code_vector, d_output_weight, nullptr, workspace,
                                   workspace_bytes, algo, stream);
    if (rc != C2V_OK) return rc;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (d_code_vector) rc = launch_angular_project(d_code_vector, code_vector, inv_norms, B, d->encode, st);
    if (rc == C2V_OK && d_output_weight)
        rc = launch_angular_project(d_output_weight, p->output_weight, inv_norms + B, d->label_count, d->encode, st);
    return rc;
}

int c2v_angular_logits(const c2v_dims *d, const c2v_params *p, const float *code_vector,
                       const int64_t *label, int32_t B, float margin, float inverse_temp,
                       float *outputs, void *stream)
{
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !outputs || !label || B < 1) {
        set_error("c2v_angular_logits: bad argument");
        return C2V_EINVAL;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    float *scratch = nullptr;
    C2V_CUDA_OK(cudaMallocAsync(&scratch, (size_t)(B + d->label_count) * sizeof(float), st));
    int rc = launch_angular(d, p, code_vector, reinterpret_cast<const long long *>(label), B, margin,
                            inverse_temp, outputs, scratch, st, nullptr);
    cudaFreeAsync(scratch, st);
    return rc;
}

int c2v_label_topk_supported(const c2v_dims *d, int32_t B, int32_t k)
{
    if (!dims_ok(d) || k < 1 || k > C2V_TOPK_MAX || k > d->label_count) return 0;
    return c2v_label_loss_supported(d, B);
}

size_t c2v_label_topk_workspace_bytes(const c2v_dims *d, int32_t B, int32_t k)
{
    if (!dims_ok(d) || B < 1 || k < 1 || k > C2V_TOPK_MAX || k > d->label_count) return 0;
    const size_t topk = align_up(label_topk_workspace_bytes(d, B, k), 1024), label = c2v_label_workspace_bytes(d, B);
    return topk > label ? topk : label;       // (larger in deterministic mode only)
}

// argument checks shared by c2v_label_topk / c2v_angular_topk, all before any CUDA call
static int topk_args_ok(const char *fn, const c2v_dims *d, const c2v_params *p, const float *code_vector, int32_t B,
                        int32_t k, const int64_t *indices, const float *values, const void *workspace, size_t workspace_bytes,
                        int32_t algo)
{
    if (!d) { set_error("%s: dims is NULL", fn); return C2V_EINVAL; }
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !indices || !values) {
        set_error("%s: NULL pointer argument", fn);
        return C2V_EINVAL;
    }
    if (B < 1 || k < 1 || k > d->label_count) {
        set_error("%s: B=%d, k=%d: needs B >= 1 and 1 <= k <= label_count (%lld)", fn, B, k, (long long)d->label_count);
        return C2V_EINVAL;
    }
    const int base_algo = algo & 0xff;
    if (base_algo != C2V_ALGO_AUTO && base_algo != C2V_ALGO_FFMA && base_algo != C2V_ALGO_TCGEN05) {
        set_error("%s: unknown algo %d", fn, base_algo);
        return C2V_EINVAL;
    }
    if (!c2v_label_topk_supported(d, B, k) || base_algo == C2V_ALGO_FFMA) {
        set_error("%s: the fused top-k runs on the tensor cores and needs encode_size %% 4 == 0 and <= 256, B <= 2048 and "
                  "k <= %d (got encode_size %d, B %d, k %d, algo %d); take the top k of c2v_label_logits' output instead",
                  fn, C2V_TOPK_MAX, d->encode, B, k, base_algo);
        return C2V_EUNSUPPORTED;
    }
    const size_t need = label_topk_workspace_bytes(d, B, k);
    if (!workspace || workspace_bytes < need) {
        set_error("%s: workspace too small: %zu < %zu", fn, workspace ? workspace_bytes : (size_t)0, need);
        return C2V_EWORKSPACE;
    }
    return C2V_OK;
}

int c2v_label_topk(const c2v_dims *d, const c2v_params *p, const float *code_vector, int32_t B, int32_t k,
                   int64_t *indices, float *values, float *probs, void *workspace, size_t workspace_bytes, int32_t algo,
                   void *stream)
{
    const int rc = topk_args_ok("c2v_label_topk", d, p, code_vector, B, k, indices, values, workspace, workspace_bytes, algo);
    if (rc != C2V_OK) return rc;
    LabelLossArgs la = {};
    la.topk_k = k; la.topk_idx = reinterpret_cast<long long *>(indices); la.topk_val = values; la.topk_prob = probs;
    return label_gemm(d, p, code_vector, B, nullptr, nullptr, nullptr, workspace, workspace_bytes, algo, stream, &la);
}

int c2v_angular_topk(const c2v_dims *d, const c2v_params *p, const float *code_vector, int32_t B, int32_t k,
                     float inverse_temp, int64_t *indices, float *values, float *probs, void *workspace,
                     size_t workspace_bytes, int32_t algo, void *stream)
{
    int rc = topk_args_ok("c2v_angular_topk", d, p, code_vector, B, k, indices, values, workspace, workspace_bytes, algo);
    if (rc != C2V_OK) return rc;
    float *inv = label_topk_inv_norms(d, B, k, workspace);
    rc = angular_inv_norms(d, p, code_vector, B, inv, stream);
    if (rc != C2V_OK) return rc;
    LabelLossArgs la = {};
    la.inv_norms = inv; la.inverse_temp = inverse_temp;
    la.topk_k = k; la.topk_idx = reinterpret_cast<long long *>(indices); la.topk_val = values; la.topk_prob = probs;
    return label_gemm(d, p, code_vector, B, nullptr, nullptr, nullptr, workspace, workspace_bytes, algo, stream, &la);
}

// ---- similarity search (c2v_knn_*) ------------------------------------------------------------------------------------
static const long long kKnnMaxN = 0xFFFFFFFEll;      // the top-k keys hold ~column in 32 bits: N < 2^32 - 1
static const int kKnnMaxQ = 2048;

static bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

// the bank's shape: C2V_EINVAL / C2V_EUNSUPPORTED with the message, or C2V_OK
static int knn_shape_ok(const char *fn, long long N, int H)
{
    if (N < 1 || N > kKnnMaxN || H < 1) {
        set_error("%s: N=%lld, H=%d: needs 1 <= N < 2^32 - 1 and H >= 1", fn, N, H);
        return C2V_EINVAL;
    }
    if (H % 4 != 0 || H > 256) {
        set_error("%s: the tensor-core similarity needs encode_size %% 4 == 0 and <= 256 (got %d)", fn, H);
        return C2V_EUNSUPPORTED;
    }
    return C2V_OK;
}

size_t c2v_knn_prep_workspace_bytes(int64_t N, int32_t H)
{
    if (N < 1 || N > kKnnMaxN || H < 4 || H > 256 || H % 4) return 0;
    return align_up(knn_prep_bytes(N, H), 1024);
}

size_t c2v_knn_topk_workspace_bytes(int64_t N, int32_t H, int32_t Q, int32_t k)
{
    if (!c2v_knn_prep_workspace_bytes(N, H) || Q < 1 || Q > kKnnMaxQ || k < 1 || k > C2V_TOPK_MAX) return 0;
    return align_up(knn_query_bytes(N, H, Q, k), 1024);
}

size_t c2v_knn_pairs_workspace_bytes(int64_t N, int32_t H, int32_t Q)
{
    if (!c2v_knn_prep_workspace_bytes(N, H) || Q < 1 || Q > kKnnMaxQ) return 0;
    return align_up(knn_query_bytes(N, H, Q, 0), 1024);
}

int c2v_knn_prepare(const float *bank, int64_t N, int32_t H, void *prep, size_t prep_bytes, void *stream)
{
    if (!bank || !aligned16(bank)) { set_error("c2v_knn_prepare: bank is NULL or not 16-byte aligned"); return C2V_EINVAL; }
    const int rc = knn_shape_ok("c2v_knn_prepare", N, H);
    if (rc != C2V_OK) return rc;
    const size_t need = knn_prep_bytes(N, H);
    if (!prep || prep_bytes < need || !aligned16(prep)) {
        set_error("c2v_knn_prepare: prep workspace missing, misaligned or too small: %zu < %zu", prep ? prep_bytes : (size_t)0,
                  need);
        return C2V_EWORKSPACE;
    }
    return launch_knn_prepare(bank, N, H, prep, static_cast<cudaStream_t>(stream));
}

// argument checks shared by c2v_knn_topk / c2v_knn_pairs (k == 0: pairs), all before any CUDA call
static int knn_args_ok(const char *fn, const float *bank, long long N, int H, const float *queries, int Q, int k,
                       const int64_t *exclude, int X, void *prep, size_t prep_bytes, const void *ws, size_t ws_bytes,
                       int flags)
{
    if (!bank || !queries) { set_error("%s: NULL bank / queries", fn); return C2V_EINVAL; }
    if (!aligned16(bank) || !aligned16(queries)) { set_error("%s: bank / queries must be 16-byte aligned", fn); return C2V_EINVAL; }
    int rc = knn_shape_ok(fn, N, H);
    if (rc != C2V_OK) return rc;
    if (Q < 1 || Q > kKnnMaxQ) { set_error("%s: Q=%d: needs 1 <= Q <= %d (cut larger query sets into chunks)", fn, Q, kKnnMaxQ); return C2V_EINVAL; }
    if (X < 0 || X > C2V_KNN_EXCLUDE_MAX || (X > 0 && !exclude)) {
        set_error("%s: X=%d exclusions per query: needs 0 <= X <= %d and exclude != NULL when X > 0", fn, X, C2V_KNN_EXCLUDE_MAX);
        return C2V_EINVAL;
    }
    if (flags & ~(C2V_FLAG_REUSE_PREP | C2V_FLAG_NO_PDL)) { set_error("%s: unknown flags 0x%x", fn, flags); return C2V_EINVAL; }
    if (k > 0 && (k > C2V_TOPK_MAX || (long long)k > N - X)) {
        set_error("%s: k=%d: needs 1 <= k <= %d and k <= N - X (N=%lld, X=%d)", fn, k, C2V_TOPK_MAX, N, X);
        return C2V_EINVAL;
    }
    const size_t need_prep = knn_prep_bytes(N, H), need = knn_query_bytes(N, H, Q, k);
    if (!prep || prep_bytes < need_prep || !aligned16(prep)) {
        set_error("%s: prep workspace missing, misaligned or too small: %zu < %zu", fn, prep ? prep_bytes : (size_t)0, need_prep);
        return C2V_EWORKSPACE;
    }
    if (!ws || ws_bytes < need || !aligned16(ws)) {
        set_error("%s: workspace missing, misaligned or too small: %zu < %zu", fn, ws ? ws_bytes : (size_t)0, need);
        return C2V_EWORKSPACE;
    }
    return C2V_OK;
}

static int knn_run(KnnArgs &a, int flags, void *stream)
{
    g_pdl_this_call = (flags & C2V_FLAG_NO_PDL) == 0;
    a.reuse_prep = (flags & C2V_FLAG_REUSE_PREP) != 0;
    return launch_knn(a, static_cast<cudaStream_t>(stream));
}

int c2v_knn_topk(const float *bank, int64_t N, int32_t H, const float *queries, int32_t Q, int32_t k,
                 const int64_t *exclude, int32_t X, int64_t *indices, float *sims, void *prep, size_t prep_bytes,
                 void *workspace, size_t workspace_bytes, int32_t flags, void *stream)
{
    if (!indices || !sims) { set_error("c2v_knn_topk: NULL indices / sims"); return C2V_EINVAL; }
    if (k < 1) { set_error("c2v_knn_topk: k=%d < 1", k); return C2V_EINVAL; }
    const int rc = knn_args_ok("c2v_knn_topk", bank, N, H, queries, Q, k, exclude, X, prep, prep_bytes, workspace,
                               workspace_bytes, flags);
    if (rc != C2V_OK) return rc;
    KnnArgs a = {};
    a.bank = bank; a.N = N; a.H = H; a.queries = queries; a.Q = Q;
    a.exclude = X > 0 ? reinterpret_cast<const long long *>(exclude) : nullptr; a.X = X;
    a.prep = prep; a.ws = workspace;
    a.k = k; a.indices = reinterpret_cast<long long *>(indices); a.sims = sims;
    return knn_run(a, flags, stream);
}

int c2v_knn_pairs(const float *bank, int64_t N, int32_t H, const float *queries, int32_t Q, float threshold,
                  const int64_t *exclude, int32_t X, int64_t self_offset, int64_t query_base, int64_t capacity, int64_t *pair_query,
                  int64_t *pair_index, float *pair_sim, int64_t *count, void *prep, size_t prep_bytes, void *workspace,
                  size_t workspace_bytes, int32_t flags, void *stream)
{
    if (!count) { set_error("c2v_knn_pairs: NULL count"); return C2V_EINVAL; }
    if (capacity < 0 || (capacity > 0 && (!pair_query || !pair_index || !pair_sim))) {
        set_error("c2v_knn_pairs: capacity=%lld: needs capacity >= 0 and the three outputs when it is > 0", (long long)capacity);
        return C2V_EINVAL;
    }
    if (threshold != threshold) { set_error("c2v_knn_pairs: threshold is NaN"); return C2V_EINVAL; }
    const int rc = knn_args_ok("c2v_knn_pairs", bank, N, H, queries, Q, 0, exclude, X, prep, prep_bytes, workspace,
                               workspace_bytes, flags);
    if (rc != C2V_OK) return rc;
    KnnArgs a = {};
    a.bank = bank; a.N = N; a.H = H; a.queries = queries; a.Q = Q;
    a.exclude = X > 0 ? reinterpret_cast<const long long *>(exclude) : nullptr; a.X = X;
    a.prep = prep; a.ws = workspace;
    a.threshold = threshold; a.self_offset = self_offset < 0 ? -1 : self_offset; a.query_base = query_base;
    a.capacity = capacity;
    a.pair_query = reinterpret_cast<long long *>(pair_query); a.pair_index = reinterpret_cast<long long *>(pair_index);
    a.pair_sim = pair_sim; a.count = reinterpret_cast<long long *>(count);
    return knn_run(a, flags, stream);
}

int c2v_angular_forward_train(const c2v_dims *d, const c2v_params *p, const float *code_vector, const int64_t *label,
                              int32_t B, float margin, float inverse_temp, float *outputs, float *cosine,
                              float *inv_norms, void *stream)
{
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !outputs || !label || !cosine || !inv_norms || B < 1) {
        set_error("c2v_angular_forward_train: bad argument");
        return C2V_EINVAL;
    }
    return launch_angular(d, p, code_vector, reinterpret_cast<const long long *>(label), B, margin, inverse_temp, outputs,
                          inv_norms, static_cast<cudaStream_t>(stream), cosine);
}

int c2v_angular_backward(const c2v_dims *d, const c2v_params *p, const float *code_vector, const int64_t *label,
                         int32_t B, float margin, float inverse_temp, const float *cosine, const float *inv_norms,
                         float *d_outputs, float *d_code_vector, float *d_output_weight, float *scratch, void *stream)
{
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !label || !cosine || !inv_norms || !d_outputs || !scratch || B < 1) {
        set_error("c2v_angular_backward: bad argument");
        return C2V_EINVAL;
    }
    return launch_angular_backward(d, p, code_vector, reinterpret_cast<const long long *>(label), B, margin, inverse_temp,
                                   cosine, inv_norms, inv_norms + B, d_outputs, d_code_vector, d_output_weight, scratch,
                                   static_cast<cudaStream_t>(stream));
}

int c2v_loss_argmax(const float *outputs, const int64_t *label, int32_t B, int64_t C, float *loss,
                    int64_t *argmax, float *maxval, float *d_outputs, void *stream)
{
    if (!outputs || B < 1 || C < 1) { set_error("c2v_loss_argmax: bad argument"); return C2V_EINVAL; }
    if ((loss || d_outputs) && !label) {
        set_error("c2v_loss_argmax: loss / d_outputs need label");
        return C2V_EINVAL;
    }
    if (deterministic() && loss && (!argmax || !maxval)) {
        set_error("c2v_loss_argmax: the deterministic loss needs argmax and maxval (its per-bag terms pass through maxval)");
        return C2V_EINVAL;
    }
    return launch_loss_argmax(outputs, reinterpret_cast<const long long *>(label), B, C, loss,
                              reinterpret_cast<long long *>(argmax), maxval, d_outputs,
                              static_cast<cudaStream_t>(stream));
}

int c2v_loss_argmax_opts(const float *outputs, const int64_t *label, int32_t B, int64_t C,
                         const c2v_loss_options *options, float *loss, int64_t *argmax, float *maxval, float *d_outputs,
                         void *stream)
{
    if (!options) return c2v_loss_argmax(outputs, label, B, C, loss, argmax, maxval, d_outputs, stream);
    if (!outputs || !label || B < 1 || C < 1 || (!loss && !d_outputs)) {
        set_error("c2v_loss_argmax_opts: bad argument (NULL outputs / label, B < 1, C < 1 or neither loss nor d_outputs)");
        return C2V_EINVAL;
    }
    LossOptArgs oa;
    const int rc = loss_opts_ok("c2v_loss_argmax_opts", options, false, &oa);
    if (rc != C2V_OK) return rc;
    return launch_loss_argmax_opts(outputs, reinterpret_cast<const long long *>(label), B, C, oa, loss,
                                   reinterpret_cast<long long *>(argmax), maxval, d_outputs, static_cast<cudaStream_t>(stream));
}

int c2v_label_backward(const c2v_dims *d, const c2v_params *p, const float *code_vector,
                       const float *d_outputs, int32_t B, float *d_code_vector,
                       float *d_output_weight, float *d_output_bias, void *stream)
{
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !d_outputs || B < 1) {
        set_error("c2v_label_backward: bad argument");
        return C2V_EINVAL;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int H = d->encode;
    const long long C = d->label_count;
    int rc = C2V_OK;
    if (d_code_vector)   // d_cv[b,h] = sum_c d_out[b,c] W_out[c,h]
        rc = launch_sgemm(B, H, (int)C, d_outputs, C, 1, p->output_weight, H, 1, nullptr,
                          d_code_vector, H, false, st);
    if (rc != C2V_OK) return rc;
    if (d_output_weight) // dW_out[c,h] = sum_b d_out[b,c] cv[b,h]
        rc = launch_sgemm((int)C, H, B, d_outputs, 1, C, code_vector, H, 1, nullptr, d_output_weight,
                          H, false, st);
    if (rc != C2V_OK) return rc;
    if (d_output_bias) rc = launch_colsum(d_outputs, B, C, d_output_bias, st);
    return rc;
}

int c2v_label_backward_ws(const c2v_dims *d, const c2v_params *p, const float *code_vector, const float *d_outputs,
                          int32_t B, float *d_code_vector, float *d_output_weight, float *d_output_bias, void *workspace,
                          size_t workspace_bytes, int32_t algo, void *stream)
{
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !p->output_weight || !code_vector || !d_outputs || B < 1) {
        set_error("c2v_label_backward_ws: bad argument");
        return C2V_EINVAL;
    }
    const int base_algo = algo & 0xff;
    const bool tc = base_algo != C2V_ALGO_FFMA && workspace != nullptr && label_backward_tc_ok(d) &&
                    (d_output_weight != nullptr || d_output_bias == nullptr);
    if (!tc) {
        if (base_algo == C2V_ALGO_TCGEN05) {
            set_error("tensor-core label backward needs a label workspace, encode_size %% 4 == 0 and <= 256");
            return C2V_EUNSUPPORTED;
        }
        return c2v_label_backward(d, p, code_vector, d_outputs, B, d_code_vector, d_output_weight, d_output_bias, stream);
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const uint8_t *img = nullptr, *cv_img = nullptr; const float *hdr = nullptr; unsigned *scratch = nullptr;
    int rc = label_w_image(d, p->output_weight, B, workspace, workspace_bytes, (algo & C2V_FLAG_REUSE_PREP) != 0, st, &img, &hdr,
                           &scratch, &cv_img);
    if (rc != C2V_OK) return rc;
    // after c2v_label_dlogits on this workspace (the flag's contract: same code_vector, nothing in between) the workspace also
    // holds max |d_outputs| and the fp16 image of code_vector: the backward reads both instead of recomputing them
    const bool from_dlogits = (algo & C2V_FLAG_GRAD_ABSMAX_READY) != 0 && label_ws_holds_dlogits_of(workspace, code_vector, B);
    float *dcv_slabs = nullptr;
    if (deterministic() && d_code_vector) {
        const size_t need = c2v_label_workspace_bytes(d, B);
        if (workspace_bytes < need) {
            set_error("c2v_label_backward_ws: workspace too small for the deterministic mode: %zu < %zu", workspace_bytes, need);
            return C2V_EWORKSPACE;
        }
        dcv_slabs = reinterpret_cast<float *>(static_cast<char *>(workspace) + align_up(label_tcgen05_workspace_bytes(d, B), 1024));
    }
    return launch_label_backward_tc(d, code_vector, d_outputs, B, img, hdr, d_code_vector, d_output_weight, d_output_bias,
                                    scratch, st, from_dlogits, from_dlogits ? cv_img : nullptr, dcv_slabs);
}

size_t c2v_encode_backward_workspace_bytes(const c2v_dims *d, int32_t B, int32_t L)
{
    if (!dims_ok(d) || B < 1 || L < 1) return 0;
    return encode_backward_workspace_bytes(d, B, L);
}

int c2v_encode_backward(const c2v_dims *d, const c2v_params *p, const int64_t *starts,
                        const int64_t *paths, const int64_t *ends, int32_t B, int32_t L,
                        const c2v_dropout *drop, const float *code_vector, const float *attention,
                        const float *d_code_vector, const float *d_attention, const c2v_grads *grads,
                        void *workspace, size_t workspace_bytes, void *stream)
{
    return c2v_encode_backward_stashed(d, p, starts, paths, ends, B, L, drop, code_vector, attention, nullptr,
                                       d_code_vector, d_attention, grads, workspace, workspace_bytes, stream);
}

int c2v_encode_backward_stashed(const c2v_dims *d, const c2v_params *p, const int64_t *starts,
                                const int64_t *paths, const int64_t *ends, int32_t B, int32_t L,
                                const c2v_dropout *drop, const float *code_vector, const float *attention,
                                const float *x_stash, const float *d_code_vector, const float *d_attention,
                                const c2v_grads *grads, void *workspace, size_t workspace_bytes, void *stream)
{
    return c2v_encode_backward_phased(d, p, starts, paths, ends, B, L, drop, code_vector, attention, x_stash, d_code_vector,
                                      d_attention, grads, workspace, workspace_bytes, 0, stream);
}

// the backward of both layouts (offsets == NULL: [B, L], N = B * L) once the caller's argument checks have passed
static int encode_backward_impl(const c2v_dims *d, const c2v_params *p, const int64_t *starts, const int64_t *paths,
                                const int64_t *ends, const int64_t *offsets, int32_t B, long long N, int32_t L,
                                const c2v_dropout *drop, const float *code_vector, const float *attention,
                                const float *x_stash, const float *d_code_vector, const float *d_attention,
                                const c2v_grads *grads, void *workspace, size_t workspace_bytes, int32_t phase, void *stream,
                                const c2v_row_slots *slots = nullptr)
{
    if (!grads->terminal_embedding || !grads->path_embedding || !grads->input_linear ||
        !grads->ln_weight || !grads->ln_bias || !grads->attention) {
        set_error("c2v_encode_backward: NULL gradient pointer");
        return C2V_EINVAL;
    }
    if (!dropout_ok("c2v_encode_backward", drop)) return C2V_EINVAL;
    EncodeArgs a;
    memset(&a, 0, sizeof(a));
    a.starts = reinterpret_cast<const long long *>(starts);
    a.paths = reinterpret_cast<const long long *>(paths);
    a.ends = reinterpret_cast<const long long *>(ends);
    a.emb_t = p->terminal_embedding; a.emb_p = p->path_embedding;
    a.ln_g = p->ln_weight; a.ln_b = p->ln_bias; a.attn = p->attention;
    a.T = d->terminal_count; a.P = d->path_count;
    a.Et = d->terminal_embed; a.Ep = d->path_embed; a.H = d->encode;
    a.D = 2 * a.Et + a.Ep;
    a.L = L; a.N = N;
    set_dropout(a, drop);
    a.bag_off = reinterpret_cast<const long long *>(offsets);
    a.n_bags = B;
    return launch_encode_backward(d, p, a, B, code_vector, attention, d_code_vector, d_attention,
                                  grads, workspace, workspace_bytes,
                                  static_cast<cudaStream_t>(stream), x_stash, phase, slots);
}

int c2v_encode_backward_phased(const c2v_dims *d, const c2v_params *p, const int64_t *starts,
                               const int64_t *paths, const int64_t *ends, int32_t B, int32_t L,
                               const c2v_dropout *drop, const float *code_vector, const float *attention,
                               const float *x_stash, const float *d_code_vector, const float *d_attention,
                               const c2v_grads *grads, void *workspace, size_t workspace_bytes, int32_t phase, void *stream)
{
    if (phase < 0 || phase > 2) { set_error("c2v_encode_backward_phased: phase %d", phase); return C2V_EINVAL; }
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !starts || !paths || !ends || !code_vector || !attention || !d_code_vector || !grads ||
        !workspace || B < 1 || L < 1) {
        set_error("c2v_encode_backward: bad argument");
        return C2V_EINVAL;
    }
    return encode_backward_impl(d, p, starts, paths, ends, nullptr, B, (long long)B * L, L, drop, code_vector, attention,
                                x_stash, d_code_vector, d_attention, grads, workspace, workspace_bytes, phase, stream);
}

size_t c2v_encode_backward_packed_workspace_bytes(const c2v_dims *d, int32_t B, int64_t N)
{
    if (!dims_ok(d) || B < 1 || N < B) return 0;
    return encode_backward_workspace_bytes_n(d, B, N, true);
}

int c2v_encode_backward_packed(const c2v_dims *d, const c2v_params *p, const int64_t *starts, const int64_t *paths,
                               const int64_t *ends, const int64_t *offsets, int32_t B, int64_t N, int32_t L,
                               const c2v_dropout *drop, const float *code_vector, const float *attention,
                               const float *x_stash, const float *d_code_vector, const float *d_attention,
                               const c2v_grads *grads, void *workspace, size_t workspace_bytes, int32_t phase, void *stream)
{
    if (phase < 0 || phase > 2) { set_error("c2v_encode_backward_packed: phase %d", phase); return C2V_EINVAL; }
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !starts || !paths || !ends || !offsets || !code_vector || !attention || !d_code_vector || !grads ||
        !workspace) {
        set_error("c2v_encode_backward_packed: NULL pointer argument");
        return C2V_EINVAL;
    }
    if (!packed_shape_ok("c2v_encode_backward_packed", B, N, L)) return C2V_EINVAL;
    return encode_backward_impl(d, p, starts, paths, ends, offsets, B, N, L, drop, code_vector, attention, x_stash,
                                d_code_vector, d_attention, grads, workspace, workspace_bytes, phase, stream);
}

// the checks the sparse backwards add to those of their dense counterparts
static bool row_slots_ok(const char *fn, const c2v_row_slots *slots, const c2v_grads *grads)
{
    if (!slots || !grads) {
        set_error("%s: NULL pointer argument", fn);
        return false;
    }
    const uintptr_t sa = reinterpret_cast<uintptr_t>(slots->terminal) | reinterpret_cast<uintptr_t>(slots->path);
    uintptr_t va = 0;
    if (slots->terminal) va |= reinterpret_cast<uintptr_t>(grads->terminal_embedding);
    if (slots->path) va |= reinterpret_cast<uintptr_t>(grads->path_embedding);
    if ((sa & 3) || (va & 15)) {
        set_error("%s: misaligned pointer (slot maps: 4 bytes, compact gradient buffers: 16)", fn);
        return false;
    }
    return true;
}

int c2v_encode_backward_sparse(const c2v_dims *d, const c2v_params *p, const int64_t *starts, const int64_t *paths,
                               const int64_t *ends, int32_t B, int32_t L, const c2v_dropout *drop,
                               const float *code_vector, const float *attention, const float *x_stash,
                               const float *d_code_vector, const float *d_attention, const c2v_grads *grads,
                               const c2v_row_slots *slots, void *workspace, size_t workspace_bytes, int32_t phase,
                               void *stream)
{
    if (phase < 0 || phase > 2) { set_error("c2v_encode_backward_sparse: phase %d", phase); return C2V_EINVAL; }
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !starts || !paths || !ends || !code_vector || !attention || !d_code_vector || !grads ||
        !workspace || B < 1 || L < 1) {
        set_error("c2v_encode_backward_sparse: bad argument");
        return C2V_EINVAL;
    }
    if (!row_slots_ok("c2v_encode_backward_sparse", slots, grads)) return C2V_EINVAL;
    return encode_backward_impl(d, p, starts, paths, ends, nullptr, B, (long long)B * L, L, drop, code_vector, attention,
                                x_stash, d_code_vector, d_attention, grads, workspace, workspace_bytes, phase, stream, slots);
}

int c2v_encode_backward_packed_sparse(const c2v_dims *d, const c2v_params *p, const int64_t *starts,
                                      const int64_t *paths, const int64_t *ends, const int64_t *offsets, int32_t B,
                                      int64_t N, int32_t L, const c2v_dropout *drop, const float *code_vector,
                                      const float *attention, const float *x_stash, const float *d_code_vector,
                                      const float *d_attention, const c2v_grads *grads, const c2v_row_slots *slots,
                                      void *workspace, size_t workspace_bytes, int32_t phase, void *stream)
{
    if (phase < 0 || phase > 2) { set_error("c2v_encode_backward_packed_sparse: phase %d", phase); return C2V_EINVAL; }
    if (!dims_ok(d)) return C2V_EINVAL;
    if (!p || !starts || !paths || !ends || !offsets || !code_vector || !attention || !d_code_vector || !grads ||
        !workspace) {
        set_error("c2v_encode_backward_packed_sparse: NULL pointer argument");
        return C2V_EINVAL;
    }
    if (!packed_shape_ok("c2v_encode_backward_packed_sparse", B, N, L)) return C2V_EINVAL;
    if (!row_slots_ok("c2v_encode_backward_packed_sparse", slots, grads)) return C2V_EINVAL;
    return encode_backward_impl(d, p, starts, paths, ends, offsets, B, N, L, drop, code_vector, attention, x_stash,
                                d_code_vector, d_attention, grads, workspace, workspace_bytes, phase, stream, slots);
}

int c2v_next_dropout_key(int64_t *rng_state, uint64_t *key_out, void *stream)
{
    if (!rng_state || !key_out || (reinterpret_cast<uintptr_t>(rng_state) & 7) || (reinterpret_cast<uintptr_t>(key_out) & 7)) {
        set_error("c2v_next_dropout_key: rng_state and key_out must be 8-byte aligned device pointers");
        return C2V_EINVAL;
    }
    next_dropout_key_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<long long *>(rng_state),
                                                                            reinterpret_cast<unsigned long long *>(key_out));
    C2V_LAUNCH_OK("next_dropout_key_kernel");
    return C2V_OK;
}

}  // extern "C"

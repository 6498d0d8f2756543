// c2v_sampled.cu -- sampled softmax over the plain label head (Jean et al. 2015; TensorFlow's sampled_softmax_loss with
// num_true = 1, remove_accidental_hits and subtract_log_q).
//
// One training step scores every row against S shared candidates and its own true label instead of all C labels:
//   sample   S candidate ids drawn i.i.d. from q (an fp64 CDF on the device), Philox4x32-10 + binary search
//   gather   W_hat = W_out[ids], b_hat = b_out[ids] - log(S q(ids)) for ids = (s_1 .. s_S, y_1 .. y_B) [S + B]
//   logits   the label head's own GEMM (c2v_label_logits) on W_hat, b_hat: [B, S + B]; column S + i is row i's true logit
//   loss     per row, over the candidates that are not an accidental hit and the row's own true column: lse and the mean
//            of lse_i - z_i+ in a fixed order
//   dlogits  written over the [B, S + B] logits; the label head's backward then gives d cv, d W_hat and d b_hat
//   scatter  d W_hat / d b_hat added into the dense [C, H] / [C] gradients: the S + B ids are sorted and every distinct id
//            sums its rows in sorted order, so the result does not depend on scheduling.
#include <cub/device/device_radix_sort.cuh>

#include "c2v_common.cuh"

namespace c2v {

// Counter word 3 of every sampler block; the dropout mask's blocks all have word 3 = 0, so the two never share a counter.
constexpr unsigned kSampledCounterTag = 1u;

// Draw j: Philox block with counter (j >> 1, 0, 0, 1) and key (key_lo, key_hi); words (x, y) for even j, (z, w) for odd j,
// as u = ((hi << 32 | lo) >> 11) * 2^-53 in [0, 1).  The id is the first c with u < cdf[c] (cdf[C - 1] == 1).
__global__ void __launch_bounds__(256)
sampled_candidates_kernel(const double *__restrict__ cdf, long long C, int S, unsigned long long key,
                          const unsigned long long *__restrict__ key_dev, long long *__restrict__ out)
{
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= S) return;
    const unsigned long long k = key_dev ? *key_dev : key;
    const uint4 w = philox4x32_10(make_uint4((unsigned)j >> 1, 0u, 0u, kSampledCounterTag),
                                  make_uint2((unsigned)k, (unsigned)(k >> 32)));
    const unsigned hi = (j & 1) ? w.z : w.x, lo = (j & 1) ? w.w : w.y;
    const double u = (double)((((unsigned long long)hi << 32) | lo) >> 11) * 0x1p-53;
    long long a = 0, b = C - 1;
    while (a < b) {
        const long long m = (a + b) >> 1;
        if (u < cdf[m]) b = m; else a = m + 1;
    }
    out[j] = a;
}

// One warp per row r of W_hat: r < S is candidate r, r >= S the label of batch row r - S.  An id outside [0, C) (a bad
// label) gets a zero row and a NaN bias, so its batch row's loss is NaN, as the full head's fused loss makes it.
__global__ void __launch_bounds__(256)
sampled_gather_kernel(const float *__restrict__ W, const float *__restrict__ bias, const double *__restrict__ log_q,
                      long long C, int H, const long long *__restrict__ cand, int S, const long long *__restrict__ label,
                      int B, float *__restrict__ w_hat, float *__restrict__ b_hat, long long *__restrict__ ids)
{
    const long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (r >= (long long)S + B) return;
    const long long id = r < S ? cand[r] : label[r - S];
    const bool ok = id >= 0 && id < C;
    const float *src = W + (ok ? id : 0) * (long long)H;
    float *dst = w_hat + r * H;
    for (int c = lane; c < H; c += 32) dst[c] = ok ? src[c] : 0.0f;
    if (lane == 0) {
        b_hat[r] = ok ? (float)((double)bias[id] - (log((double)S) + log_q[id])) : __int_as_float(0x7fc00000);
        ids[r] = id;
    }
}

// fixed-order block sum / max over 256 threads (the result is in every thread)
__device__ __forceinline__ float sampled_block_reduce(float v, bool is_max, float *red)
{
    v = is_max ? warp_max(v) : warp_sum(v);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();                                   // red may still be read by an earlier call
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = red[0];
#pragma unroll
    for (int i = 1; i < 8; ++i) t = is_max ? fmaxf(t, red[i]) : t + red[i];
    return t;
}

// One CTA per batch row: lse over the row's included columns -- candidate j unless ids[j] == its label, and its own
// true column S + i.  The other rows' true columns are never read.
__global__ void __launch_bounds__(256)
sampled_row_lse_kernel(const float *__restrict__ logits, const long long *__restrict__ ids, int S, int B,
                       float *__restrict__ lse)
{
    __shared__ float red[8];
    const int i = blockIdx.x;
    const long long n = (long long)S + B;
    const float *z = logits + (long long)i * n;
    const long long y = ids[S + i];
    const float zt = z[S + i];
    float m = zt;
    for (int j = threadIdx.x; j < S; j += blockDim.x)
        if (ids[j] != y) m = fmaxf(m, z[j]);
    m = sampled_block_reduce(m, true, red);
    float s = threadIdx.x == 0 ? expf(zt - m) : 0.0f;
    for (int j = threadIdx.x; j < S; j += blockDim.x)
        if (ids[j] != y) s += expf(z[j] - m);
    s = sampled_block_reduce(s, false, red);
    if (threadIdx.x == 0) lse[i] = m + logf(s);
}

// One CTA: loss = sum_i (lse_i - z_i+) / B, each thread over a fixed stride of rows, then the fixed-order block sum.
__global__ void __launch_bounds__(256)
sampled_mean_kernel(const float *__restrict__ logits, const float *__restrict__ lse, int S, int B, float *__restrict__ loss)
{
    __shared__ float red[8];
    const long long n = (long long)S + B;
    float s = 0.0f;
    for (int i = threadIdx.x; i < B; i += blockDim.x) s += lse[i] - logits[(long long)i * n + S + i];
    s = sampled_block_reduce(s, false, red);
    if (threadIdx.x == 0) *loss = s / (float)B;
}

// In place over the [B, S + B] logits: d loss / d z = g (p - [true]) on included columns, exactly 0 elsewhere;
// g = scale (* *scale_dev).
__global__ void __launch_bounds__(256)
sampled_dlogits_kernel(float *__restrict__ logits, const long long *__restrict__ ids, const float *__restrict__ lse, int S,
                       int B, float scale, const float *__restrict__ scale_dev)
{
    const int i = blockIdx.y;
    const long long n = (long long)S + B;
    const long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const float g = scale_dev ? scale * *scale_dev : scale;
    float *z = logits + (long long)i * n;
    float d = 0.0f;
    if (j < S) {
        if (ids[j] != ids[S + i]) d = expf(z[j] - lse[i]) * g;
    } else if (j == S + i) {
        d = (expf(z[j] - lse[i]) - 1.0f) * g;
    }
    z[j] = d;
}

// key of entry e: id << pbits | e, ids outside [0, C) as the sentinel C (sorted behind every real row, never written)
__global__ void __launch_bounds__(256)
scatter_keys_kernel(const long long *__restrict__ ids, long long n, long long C, int pbits,
                    unsigned long long *__restrict__ keys)
{
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    long long id = ids[e];
    if (id < 0 || id >= C) id = C;
    keys[e] = (unsigned long long)id << pbits | (unsigned long long)e;
}

// One warp per sorted position; the warp at the first position of a run of equal ids sums the run's rows in sorted
// (= entry) order and adds the sum to the id's row, its only writer.
__global__ void __launch_bounds__(256)
scatter_rows_kernel(const unsigned long long *__restrict__ keys, long long n, int pbits, long long C,
                    const float *__restrict__ rows, const float *__restrict__ bias, int H, float *__restrict__ dst,
                    float *__restrict__ dst_bias)
{
    const long long p = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (p >= n) return;
    const unsigned long long id = keys[p] >> pbits;
    if (id >= (unsigned long long)C || (p > 0 && (keys[p - 1] >> pbits) == id)) return;
    long long end = p + 1;
    while (end < n && (keys[end] >> pbits) == id) ++end;
    const unsigned long long emask = (1ull << pbits) - 1;
    if (rows) {
        for (int c = lane; c < H; c += 32) {
            float s = 0.0f;
#pragma unroll 4
            for (long long q = p; q < end; ++q) s += rows[(long long)(keys[q] & emask) * H + c];
            dst[(long long)id * H + c] += s;
        }
    }
    if (bias && lane == 0) {
        float s = 0.0f;
        for (long long q = p; q < end; ++q) s += bias[keys[q] & emask];
        dst_bias[id] += s;
    }
}

static int sampled_bit_length(unsigned long long x)
{
    int b = 0;
    while (x) { ++b; x >>= 1; }
    return b;
}

// keys double buffer [2 n] u64 | CUB scratch: one byte per key plus 1 MB (checked against CUB's own figure at every call)
static size_t scatter_sort_bound(long long n) { return (size_t)n + (1u << 20); }
static size_t scatter_ws(long long n) { return align_up((size_t)n * 16, 1024) + scatter_sort_bound(n); }

}  // namespace c2v

using namespace c2v;

static bool sm_misaligned(const void *ptr, uintptr_t a) { return (reinterpret_cast<uintptr_t>(ptr) & (a - 1)) != 0; }

extern "C" int c2v_sampled_candidates(const double *cdf, int64_t C, int32_t S, uint64_t key, const uint64_t *key_device,
                                      int64_t *candidates, void *stream)
{
    if (C < 1 || S < 1 || S > C2V_SAMPLED_MAX) {
        set_error("c2v_sampled_candidates: C = %lld < 1 or S = %d outside [1, %d]", (long long)C, S, C2V_SAMPLED_MAX);
        return C2V_EINVAL;
    }
    if (!cdf || !candidates) {
        set_error("c2v_sampled_candidates: NULL pointer argument");
        return C2V_EINVAL;
    }
    if (sm_misaligned(cdf, 8) || sm_misaligned(candidates, 8) || sm_misaligned(key_device, 8)) {
        set_error("c2v_sampled_candidates: misaligned pointer (cdf, key_device, candidates: 8 bytes)");
        return C2V_EINVAL;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    sampled_candidates_kernel<<<(unsigned)((S + 255) / 256), 256, 0, st>>>(
        cdf, C, S, key, reinterpret_cast<const unsigned long long *>(key_device), reinterpret_cast<long long *>(candidates));
    C2V_LAUNCH_OK("sampled_candidates_kernel");
    return C2V_OK;
}

extern "C" int c2v_sampled_gather(const float *output_weight, const float *output_bias, const double *log_q, int64_t C,
                                  int32_t H, const int64_t *candidates, int32_t S, const int64_t *label, int32_t B,
                                  float *w_hat, float *b_hat, int64_t *ids, void *stream)
{
    if (C < 1 || H < 1 || S < 1 || S > C2V_SAMPLED_MAX || B < 1 || (long long)S + B >= (1ll << 31)) {
        set_error("c2v_sampled_gather: C = %lld, H = %d, S = %d or B = %d out of range (C, H, B >= 1, S in [1, %d])",
                  (long long)C, H, S, B, C2V_SAMPLED_MAX);
        return C2V_EINVAL;
    }
    if (!output_weight || !output_bias || !log_q || !candidates || !label || !w_hat || !b_hat || !ids) {
        set_error("c2v_sampled_gather: NULL pointer argument");
        return C2V_EINVAL;
    }
    if (sm_misaligned(output_weight, 4) || sm_misaligned(output_bias, 4) || sm_misaligned(log_q, 8) ||
        sm_misaligned(candidates, 8) || sm_misaligned(label, 8) || sm_misaligned(w_hat, 4) || sm_misaligned(b_hat, 4) ||
        sm_misaligned(ids, 8)) {
        set_error("c2v_sampled_gather: misaligned pointer (log_q, candidates, label, ids: 8 bytes, floats: 4)");
        return C2V_EINVAL;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long rows = (long long)S + B;
    sampled_gather_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(
        output_weight, output_bias, log_q, C, H, reinterpret_cast<const long long *>(candidates), S,
        reinterpret_cast<const long long *>(label), B, w_hat, b_hat, reinterpret_cast<long long *>(ids));
    C2V_LAUNCH_OK("sampled_gather_kernel");
    return C2V_OK;
}

static int sampled_rows_check(const char *name, int32_t S, int32_t B)
{
    if (S < 1 || S > C2V_SAMPLED_MAX || B < 1 || (long long)S + B >= (1ll << 31)) {
        set_error("%s: S = %d outside [1, %d] or B = %d < 1", name, S, C2V_SAMPLED_MAX, B);
        return C2V_EINVAL;
    }
    return C2V_OK;
}

extern "C" int c2v_sampled_loss(const float *logits, const int64_t *ids, int32_t S, int32_t B, float *lse, float *loss,
                                void *stream)
{
    if (sampled_rows_check("c2v_sampled_loss", S, B) != C2V_OK) return C2V_EINVAL;
    if (!logits || !ids || !lse || !loss) {
        set_error("c2v_sampled_loss: NULL pointer argument");
        return C2V_EINVAL;
    }
    if (sm_misaligned(logits, 4) || sm_misaligned(ids, 8) || sm_misaligned(lse, 4) || sm_misaligned(loss, 4)) {
        set_error("c2v_sampled_loss: misaligned pointer (ids: 8 bytes, floats: 4)");
        return C2V_EINVAL;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long *id = reinterpret_cast<const long long *>(ids);
    sampled_row_lse_kernel<<<(unsigned)B, 256, 0, st>>>(logits, id, S, B, lse);
    C2V_LAUNCH_OK("sampled_row_lse_kernel");
    sampled_mean_kernel<<<1, 256, 0, st>>>(logits, lse, S, B, loss);
    C2V_LAUNCH_OK("sampled_mean_kernel");
    return C2V_OK;
}

extern "C" int c2v_sampled_dlogits(float *logits, const int64_t *ids, const float *lse, int32_t S, int32_t B, float scale,
                                   const float *scale_device, void *stream)
{
    if (sampled_rows_check("c2v_sampled_dlogits", S, B) != C2V_OK) return C2V_EINVAL;
    if (B > 65535) {
        set_error("c2v_sampled_dlogits: B = %d > 65535", B);
        return C2V_EINVAL;
    }
    if (!logits || !ids || !lse) {
        set_error("c2v_sampled_dlogits: NULL pointer argument");
        return C2V_EINVAL;
    }
    if (sm_misaligned(logits, 4) || sm_misaligned(ids, 8) || sm_misaligned(lse, 4) || sm_misaligned(scale_device, 4)) {
        set_error("c2v_sampled_dlogits: misaligned pointer (ids: 8 bytes, floats: 4)");
        return C2V_EINVAL;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long n = (long long)S + B;
    sampled_dlogits_kernel<<<dim3((unsigned)((n + 255) / 256), (unsigned)B), 256, 0, st>>>(
        logits, reinterpret_cast<const long long *>(ids), lse, S, B, scale, scale_device);
    C2V_LAUNCH_OK("sampled_dlogits_kernel");
    return C2V_OK;
}

extern "C" size_t c2v_scatter_rows_add_workspace_bytes(int64_t n)
{
    if (n < 1 || n >= (1ll << 31)) return 0;
    return scatter_ws(n);
}

extern "C" int c2v_scatter_rows_add(const int64_t *ids, int64_t n, const float *rows, const float *bias, int32_t H,
                                    int64_t C, float *dst, float *dst_bias, void *workspace, size_t workspace_bytes,
                                    void *stream)
{
    if (n < 1 || n >= (1ll << 31) || C < 1 || C >= (1ll << 31) || H < 1) {
        set_error("c2v_scatter_rows_add: n = %lld or C = %lld outside [1, 2^31), or H = %d < 1",
                  (long long)n, (long long)C, H);
        return C2V_EINVAL;
    }
    if (!ids || !workspace || (!rows != !dst) || (!bias != !dst_bias) || (!rows && !bias)) {
        set_error("c2v_scatter_rows_add: NULL pointer argument (rows / dst and bias / dst_bias go in pairs, one pair at "
                  "least)");
        return C2V_EINVAL;
    }
    if (sm_misaligned(ids, 8) || sm_misaligned(rows, 4) || sm_misaligned(bias, 4) || sm_misaligned(dst, 4) ||
        sm_misaligned(dst_bias, 4) || sm_misaligned(workspace, 16)) {
        set_error("c2v_scatter_rows_add: misaligned pointer (ids: 8 bytes, floats: 4, workspace: 16)");
        return C2V_EINVAL;
    }
    const size_t need = scatter_ws(n);
    if (workspace_bytes < need) {
        set_error("c2v_scatter_rows_add: workspace too small: %zu < %zu", workspace_bytes, need);
        return C2V_EWORKSPACE;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    char *base = static_cast<char *>(workspace);
    unsigned long long *k0 = reinterpret_cast<unsigned long long *>(base), *k1 = k0 + n;
    void *scratch = base + align_up((size_t)n * 16, 1024);
    const int pbits = sampled_bit_length((unsigned long long)(n - 1)) > 0 ? sampled_bit_length((unsigned long long)(n - 1)) : 1;
    const int rbits = sampled_bit_length((unsigned long long)C);           // C - 1 < sentinel C < 2^rbits
    scatter_keys_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(reinterpret_cast<const long long *>(ids), n, C, pbits,
                                                                      k0);
    C2V_LAUNCH_OK("scatter_keys_kernel");
    cub::DoubleBuffer<unsigned long long> keys(k0, k1);
    size_t sort_bytes = 0;
    C2V_CUDA_OK(cub::DeviceRadixSort::SortKeys(nullptr, sort_bytes, keys, (int)n, 0, pbits + rbits, st));
    if (sort_bytes > scatter_sort_bound(n)) {
        set_error("c2v_scatter_rows_add: the radix sort needs %zu B of scratch, %zu reserved", sort_bytes,
                  scatter_sort_bound(n));
        return C2V_EWORKSPACE;
    }
    C2V_CUDA_OK(cub::DeviceRadixSort::SortKeys(scratch, sort_bytes, keys, (int)n, 0, pbits + rbits, st));
    C2V_COUNT_LAUNCH();
    scatter_rows_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(keys.Current(), n, pbits, C, rows, bias, H, dst, dst_bias);
    C2V_LAUNCH_OK("scatter_rows_kernel");
    return C2V_OK;
}

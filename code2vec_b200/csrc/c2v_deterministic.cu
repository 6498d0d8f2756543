// c2v_deterministic.cu -- fixed-order reductions of the deterministic training mode (c2v_set_deterministic).
//
// The default backward adds its large sums with float atomics, whose order changes from launch to launch.  In this mode
// every such sum has a fixed order instead:
//   - partial slabs (one per CTA / split, plain stores) added in slab order: launch_det_slab_sum;
//   - embedding-table gradients: the dC kernels store every context's dC row to a [N, D] buffer, and
//     launch_det_embed_grads sums those rows per table row in the order of their sorted keys.
//
// Embedding rows.  Key of entry e (one per context and sub-vector of the table): row << ebits | e, with e = 2r (start) and
// 2r + 1 (end) of context r for the terminal table and e = r for the path table; out-of-range indices count as row 0, as
// the encode reads them.  Contexts whose attention weight is exactly 0 (padding) have dC == 0 and get the sentinel row
// 2^rbits - 1, which sorts behind every real row and is never written.  The keys are unique, so the sorted order is a
// function of the batch alone.  The sorted array is cut into chunks of kChunk positions; one warp walks a chunk in key
// order and sums each run of equal rows.  A run inside one chunk is written straight away (grad[row] += sum: it is the
// row's only writer).  A run that touches a chunk boundary and continues in the neighbour leaves its partial in a chunk
// slot, and det_merge_kernel -- one warp for the chunk where such a run starts -- adds the partials of its chunks in chunk
// order and writes the row once.  A row that occurs in every bag of a batch spans many chunks and is still summed by
// many warps in parallel.
#include <cub/device/device_radix_sort.cuh>

#include "c2v_common.cuh"

namespace c2v {

static thread_local bool g_det = false;
bool deterministic() { return g_det; }
void set_deterministic(bool on) { g_det = on; }

namespace det {
constexpr int kChunk = 32;                  // sorted positions per warp (one key per lane)
constexpr int kCols = 256;                  // columns per pass of a warp over a chunk (8 per lane)
constexpr unsigned kSingle = 2, kLastOpenRight = 4, kFirstOpenLeft = 8;
constexpr int kMergeWarps = 16;             // warps of a merge CTA: one chunk each, all of them on a long run
constexpr int kShortRun = 64;               // a run over at most this many further chunks is summed by its owner warp alone
}  // namespace det

// One CTA per 32 columns: warp w sums slabs w, w + 8, w + 16, ... of its column (loads eight at a time), then warp 0 adds
// the eight warp sums in warp order.  The assignment depends on n_slabs only, so the order is fixed.  Column i goes to
// out[i / seg][i % seg] (up to three output segments of seg columns each).
__global__ void __launch_bounds__(256)
det_slab_sum_kernel(const float *__restrict__ src, int n_slabs, size_t stride, size_t n, float *out0, float *out1,
                    float *out2, size_t seg, int accumulate)
{
    __shared__ float red[8][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t i = (size_t)blockIdx.x * 32 + lane;
    float s = 0.0f;
    if (i < n) {
        int k = warp;
        for (; k + 7 * 8 < n_slabs; k += 8 * 8) {
            float v[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) v[q] = src[(size_t)(k + 8 * q) * stride + i];
#pragma unroll
            for (int q = 0; q < 8; ++q) s += v[q];
        }
        for (; k < n_slabs; k += 8) s += src[(size_t)k * stride + i];
    }
    red[warp][lane] = s;
    __syncthreads();
    if (warp != 0 || i >= n) return;
    s = red[0][lane];
#pragma unroll
    for (int w = 1; w < 8; ++w) s += red[w][lane];
    const size_t o = i / seg;
    float *out = (o == 0 ? out0 : o == 1 ? out1 : out2) + (i - o * seg);
    *out = accumulate ? *out + s : s;
}

int launch_det_slab_sum3(const float *src, int n_slabs, size_t slab_stride, size_t seg, int n_out, float *const *out,
                         bool accumulate, cudaStream_t st)
{
    const size_t n = seg * n_out;
    if (n == 0) return C2V_OK;
    det_slab_sum_kernel<<<(unsigned)((n + 31) / 32), 256, 0, st>>>(src, n_slabs, slab_stride, n, out[0],
                                                                 n_out > 1 ? out[1] : nullptr, n_out > 2 ? out[2] : nullptr,
                                                                 seg, accumulate ? 1 : 0);
    C2V_LAUNCH_OK("det_slab_sum_kernel");
    return C2V_OK;
}

int launch_det_slab_sum(const float *src, int n_slabs, size_t slab_stride, size_t n, float *out, bool accumulate,
                        cudaStream_t st)
{
    return launch_det_slab_sum3(src, n_slabs, slab_stride, n, 1, &out, accumulate, st);
}

static int bit_length(unsigned long long x)
{
    int b = 0;
    while (x) { ++b; x >>= 1; }
    return b;
}

// n_per = 2 (terminal: starts, ends) or 1 (path)
__global__ void __launch_bounds__(256)
det_keys_kernel(const long long *__restrict__ idx_a, const long long *__restrict__ idx_b, long long N, long long vocab,
                const float *__restrict__ att, int ebits, unsigned long long sentinel_row, unsigned long long *__restrict__ keys)
{
    const int n_per = idx_b ? 2 : 1;
    const long long n = N * n_per;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
        const long long r = e / n_per;
        long long v = ((e - r * n_per) ? idx_b : idx_a)[r];
        if (v < 0 || v >= vocab) v = 0;
        const unsigned long long row = att[r] == 0.0f ? sentinel_row : (unsigned long long)v;
        keys[e] = row << ebits | (unsigned long long)e;
    }
}

// the columns of entry e in the [N, D] dC buffer
__device__ __forceinline__ const float *det_src(const float *dc, long long e, int n_per, int D, int col_a, int col_b)
{
    const long long r = e / n_per;
    return dc + r * D + ((e - r * n_per) ? col_b : col_a);
}

__device__ __forceinline__ float *det_dst(float *grad, const int *slot, unsigned long long row, int E)
{
    return grad + (size_t)(slot ? (long long)slot[row] : (long long)row) * E;
}

// one warp per chunk of det::kChunk sorted positions
__global__ void __launch_bounds__(256)
det_chunk_kernel(const unsigned long long *__restrict__ keys, long long n, int ebits, unsigned long long sentinel_row,
                 const float *__restrict__ dc, int D, int n_per, int col_a, int col_b, int E, float *__restrict__ grad,
                 const int *__restrict__ slot, float *__restrict__ part, unsigned *__restrict__ cflags,
                 unsigned long long *__restrict__ crow, long long n_chunks)
{
    const int lane = threadIdx.x & 31;
    const long long c = (long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
    if (c >= n_chunks) return;
    const long long p0 = c * det::kChunk;
    const int cnt = (int)(n - p0 < det::kChunk ? n - p0 : det::kChunk);
    const unsigned long long emask = (1ull << ebits) - 1;
    const unsigned long long my_key = lane < cnt ? keys[p0 + lane] : ~0ull;
    const unsigned long long my_row = my_key >> ebits;
    const unsigned long long left_row = p0 > 0 ? keys[p0 - 1] >> ebits : ~0ull;
    const unsigned long long right_row = p0 + cnt < n ? keys[p0 + cnt] >> ebits : ~0ull;
    const unsigned long long row0 = __shfl_sync(0xffffffffu, my_row, 0);
    const unsigned long long row_last = __shfl_sync(0xffffffffu, my_row, cnt - 1);
    if (lane == 0) {
        unsigned f = 0;
        if (row0 == row_last) f |= det::kSingle;
        if (row0 == left_row && row0 != sentinel_row) f |= det::kFirstOpenLeft;
        if (row_last == right_row && row_last != sentinel_row) f |= det::kLastOpenRight;
        cflags[c] = f;
        crow[c] = row_last;
    }
    for (int cb = 0; cb < E; cb += det::kCols) {
        float acc[det::kCols / 32];
        unsigned long long cur = __shfl_sync(0xffffffffu, my_row, 0);
        int run_start = 0;
        auto flush = [&](int run_end) {                       // run [run_start, run_end] of row `cur`
            if (cur == sentinel_row) return;
            const bool open_left = run_start == 0 && cur == left_row;
            const bool open_right = run_end == cnt - 1 && cur == right_row;
            float *dst;
            if (open_left || open_right) {
                dst = part + ((size_t)c * 2 + (run_start == 0 ? 0 : 1)) * E;
#pragma unroll
                for (int k = 0; k < det::kCols / 32; ++k) {
                    const int col = cb + lane + 32 * k;
                    if (col < E) dst[col] = acc[k];
                }
            } else {
                dst = det_dst(grad, slot, cur, E);
#pragma unroll
                for (int k = 0; k < det::kCols / 32; ++k) {
                    const int col = cb + lane + 32 * k;
                    if (col < E) dst[col] += acc[k];
                }
            }
        };
#pragma unroll
        for (int k = 0; k < det::kCols / 32; ++k) acc[k] = 0.0f;
        for (int t = 0; t < cnt; ++t) {
            const unsigned long long key = __shfl_sync(0xffffffffu, my_key, t);
            const unsigned long long row = key >> ebits;
            if (row != cur) {
                flush(t - 1);
                cur = row; run_start = t;
#pragma unroll
                for (int k = 0; k < det::kCols / 32; ++k) acc[k] = 0.0f;
            }
            if (row == sentinel_row) break;                  // the sentinel sorts last: nothing real follows
            const float *src = det_src(dc, (long long)(key & emask), n_per, D, col_a, col_b);
#pragma unroll
            for (int k = 0; k < det::kCols / 32; ++k) {
                const int col = cb + lane + 32 * k;
                if (col < E) acc[k] += src[col];
            }
        }
        flush(cnt - 1);
    }
}

// One warp per chunk; the warp of the chunk where a multi-chunk run starts (its owner) adds the partials of the run's
// chunks in chunk order and writes the row once.  A run over at most kShortRun further chunks is summed by its owner warp
// alone.  A longer one (a row in a large share of the batch: thousands of chunks) is summed by all warps of the CTA: warp
// w takes the w-th of kMergeWarps equal contiguous pieces of the run, and the owner's partial and the piece sums are
// added in piece order.  Both splits depend on the run's length only, so the order is fixed.
__global__ void __launch_bounds__(det::kMergeWarps * 32)
det_merge_kernel(const unsigned *__restrict__ cflags, const unsigned long long *__restrict__ crow,
                 const float *__restrict__ part, long long n_chunks, int E, float *__restrict__ grad, const int *__restrict__ slot)
{
    __shared__ long long s_c[det::kMergeWarps], s_last[det::kMergeWarps];
    __shared__ int s_n;
    __shared__ float s_piece[det::kMergeWarps][det::kCols];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long c = (long long)blockIdx.x * det::kMergeWarps + warp;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    const unsigned f = c < n_chunks ? cflags[c] : 0u;
    const bool owner = (f & det::kLastOpenRight) && !((f & det::kSingle) && (f & det::kFirstOpenLeft));
    const int s0 = (f & det::kSingle) ? 0 : 1;
    long long last = c + 1;
    if (owner) {
        // the run's last chunk: the first chunk after c that does not continue it to the right, 32 chunks per step (it
        // exists: the run is open to the right of c, and the last chunk of the array never is)
        for (;;) {
            const long long j = last + lane;
            const unsigned fj = j < n_chunks ? cflags[j] : 0u;
            const unsigned stop = __ballot_sync(0xffffffffu, !((fj & det::kSingle) && (fj & det::kLastOpenRight)));
            if (stop) { last += __ffs(stop) - 1; break; }
            last += 32;
        }
        if (last - c <= det::kShortRun) {
            float *dst = det_dst(grad, slot, crow[c], E);
            for (int col = lane; col < E; col += 32) {
                float s = part[((size_t)c * 2 + s0) * E + col];
                for (long long j = c + 1; j <= last; ++j) s += part[(size_t)j * 2 * E + col];
                dst[col] += s;
            }
        } else if (lane == 0) {
            const int q = atomicAdd(&s_n, 1);         // (the order of the long runs in this list does not matter)
            s_c[q] = c;
            s_last[q] = last;
        }
    }
    __syncthreads();
    const int n_long = s_n;
    for (int q = 0; q < n_long; ++q) {
        const long long oc = s_c[q], first = oc + 1, len = s_last[q] - oc;
        const long long lo = first + len * warp / det::kMergeWarps, hi = first + len * (warp + 1) / det::kMergeWarps;
        for (int cb = 0; cb < E; cb += det::kCols) {
            for (int k = 0; k < det::kCols / 32; ++k) {
                const int col = cb + lane + 32 * k;
                if (col >= E) break;
                float s = 0.0f;
                long long j = lo;
                for (; j + 8 <= hi; j += 8) {
                    float v[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u) v[u] = part[(size_t)(j + u) * 2 * E + col];
#pragma unroll
                    for (int u = 0; u < 8; ++u) s += v[u];
                }
                for (; j < hi; ++j) s += part[(size_t)j * 2 * E + col];
                s_piece[warp][col - cb] = s;
            }
            __syncthreads();
            if (warp == 0) {
                const unsigned of = cflags[oc];
                float *dst = det_dst(grad, slot, crow[oc], E);
                for (int col = cb + lane; col < E && col < cb + det::kCols; col += 32) {
                    float s = part[((size_t)oc * 2 + ((of & det::kSingle) ? 0 : 1)) * E + col];
#pragma unroll
                    for (int w = 0; w < det::kMergeWarps; ++w) s += s_piece[w][col - cb];
                    dst[col] += s;
                }
            }
            __syncthreads();
        }
    }
}

// workspace: keys [2][n] | flags [n_chunks] | rows [n_chunks] | partials [n_chunks][2][E] | sort scratch
struct DetEmbedLayout {
    size_t keys, flags, rows, part, sort, total;
};
static size_t det_sort_bound(long long n)
{
    // CUB's one-sweep radix sort over a double buffer needs its digit histograms and a look-back array of a few bytes per
    // tile of keys; one byte per key plus 1 MB is well above that (checked against CUB's own figure at every call)
    return (size_t)n + (1u << 20);
}
static DetEmbedLayout det_layout(long long N, int E)
{
    const long long n = 2 * N, n_chunks = (n + det::kChunk - 1) / det::kChunk;
    DetEmbedLayout l;
    size_t o = 0;
    auto take = [&](size_t b) { const size_t r = o; o += align_up(b, 1024); return r; };
    l.keys = take((size_t)2 * n * 8);
    l.flags = take((size_t)n_chunks * 4);
    l.rows = take((size_t)n_chunks * 8);
    l.part = take((size_t)n_chunks * 2 * E * 4);
    l.sort = take(det_sort_bound(n));
    l.total = o;
    return l;
}

size_t det_embed_workspace_bytes(long long N, int E)
{
    return det_layout(N, E).total;
}

int launch_det_embed_grads(const EncodeArgs &a, const float *att, const float *dc, bool path, float *grad, const int *slot,
                           void *ws, size_t ws_bytes, cudaStream_t st)
{
    const int E = path ? a.Ep : a.Et;
    const long long vocab = path ? a.P : a.T;
    const DetEmbedLayout l = det_layout(a.N, a.Et > a.Ep ? a.Et : a.Ep);
    if (ws_bytes < l.total) {
        set_error("deterministic embedding gradients: workspace too small: %zu < %zu", ws_bytes, l.total);
        return C2V_EWORKSPACE;
    }
    if (a.N >= (1ll << 31) || vocab >= (1ll << 31)) {
        set_error("deterministic embedding gradients: N = %lld or %lld table rows >= 2^31", (long long)a.N, (long long)vocab);
        return C2V_EUNSUPPORTED;
    }
    char *base = static_cast<char *>(ws);
    unsigned long long *k0 = reinterpret_cast<unsigned long long *>(base + l.keys);
    const int n_per = path ? 1 : 2;
    const long long n = a.N * n_per;
    unsigned long long *k1 = k0 + n;
    unsigned *cflags = reinterpret_cast<unsigned *>(base + l.flags);
    unsigned long long *crow = reinterpret_cast<unsigned long long *>(base + l.rows);
    float *part = reinterpret_cast<float *>(base + l.part);
    const int ebits = bit_length((unsigned long long)(n - 1)) > 0 ? bit_length((unsigned long long)(n - 1)) : 1;
    const int rbits = bit_length((unsigned long long)vocab);            // vocab - 1 < sentinel = 2^rbits - 1
    const unsigned long long sentinel = (1ull << rbits) - 1;
    long long blocks = (n + 255) / 256;
    if (blocks > 8192) blocks = 8192;
    det_keys_kernel<<<(unsigned)blocks, 256, 0, st>>>(path ? a.paths : a.starts, path ? nullptr : a.ends, a.N, vocab, att, ebits,
                                                      sentinel, k0);
    C2V_LAUNCH_OK("det_keys_kernel");
    cub::DoubleBuffer<unsigned long long> keys(k0, k1);
    size_t need = 0;
    C2V_CUDA_OK(cub::DeviceRadixSort::SortKeys(nullptr, need, keys, (int)n, 0, ebits + rbits, st));
    if (need > det_sort_bound(n)) {
        set_error("deterministic embedding gradients: the radix sort needs %zu B of scratch, %zu reserved", need,
                  det_sort_bound(n));
        return C2V_EWORKSPACE;
    }
    C2V_CUDA_OK(cub::DeviceRadixSort::SortKeys(base + l.sort, need, keys, (int)n, 0, ebits + rbits, st));
    C2V_COUNT_LAUNCH();
    const long long n_chunks = (n + det::kChunk - 1) / det::kChunk;
    const unsigned grid = (unsigned)((n_chunks + 7) / 8);
    const int col_a = path ? a.Et : 0, col_b = a.Et + a.Ep;
    det_chunk_kernel<<<grid, 256, 0, st>>>(keys.Current(), n, ebits, sentinel, dc, a.D, n_per, col_a, col_b, E, grad, slot,
                                           part, cflags, crow, n_chunks);
    C2V_LAUNCH_OK("det_chunk_kernel");
    det_merge_kernel<<<(unsigned)((n_chunks + det::kMergeWarps - 1) / det::kMergeWarps), det::kMergeWarps * 32, 0, st>>>(
        cflags, crow, part, n_chunks, E, grad, slot);
    C2V_LAUNCH_OK("det_merge_kernel");
    return C2V_OK;
}

}  // namespace c2v

// c2v_sparse.cu -- row maps of the sparse embedding gradients (nn.Embedding(sparse=True)).
//
// For one table and one batch: which rows the batch indexes (rows, ascending), how many (U) and where each one's gradient
// goes in the compact [U, E] values buffer (slot[row]).  Three passes over the vocabulary, no sort:
//   mark     flag[clamp(idx)] = 1 for every index of the batch                          (n scattered byte stores)
//   count    per chunk of CHUNK rows: number of flags                                     (reads the flags)
//   scan     exclusive prefix of the chunk counts (one CTA), U = the total
//   compact  per chunk: block-wide exclusive scan of its flags + the chunk's prefix = the slot of every marked row;
//            writes slot[row] (-1 for unmarked rows) and rows[slot] = row
// Out-of-range indices count as row 0: the encode reads them as row 0 (and reports them), so row 0 receives their
// gradient.
// c2v_sparse_union_rows runs the same count / scan / compact passes behind a mark pass of its own over the W row lists
// that the ranks of a data-parallel step all-gathered: their union, ascending, and its size on the device.
#include "c2v_common.cuh"

namespace c2v {

namespace srows {
constexpr int THREADS = 1024, PER_THREAD = 8, CHUNK = THREADS * PER_THREAD;     // 8192 rows per chunk
}

__global__ void __launch_bounds__(256)
sparse_mark_kernel(const long long *__restrict__ ia, long long na, const long long *__restrict__ ib, long long nb,
                   long long vocab, uint8_t *__restrict__ flag)
{
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < na + nb; i += (long long)gridDim.x * blockDim.x) {
        long long v = i < na ? ia[i] : ib[i - na];
        if (v < 0 || v >= vocab) v = 0;
        flag[v] = 1;
    }
}

// The mark pass of c2v_sparse_union_rows: the W padded row lists [W, u_max] of a data-parallel exchange, list r valid up
// to counts[r] (clamped to [0, u_max]); padding is never read.  Rows outside [0, vocab) are not marked: no rank's step
// can apply them (c2v_sparse_adam_step skips them too).
__global__ void __launch_bounds__(256)
sparse_union_mark_kernel(const long long *__restrict__ rows, const long long *__restrict__ counts, int world,
                         long long u_max, long long vocab, uint8_t *__restrict__ flag)
{
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < world * u_max; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / u_max, j = i - r * u_max;
        if (j >= counts[r]) continue;                        // (a negative count marks nothing)
        const long long v = rows[i];
        if (v >= 0 && v < vocab) flag[v] = 1;
    }
}

// the 8 flags of this thread in chunk blockIdx.x (the flag array is padded to whole chunks with zeros)
__device__ __forceinline__ uint2 sr_load(const uint8_t *flag) {
    return *reinterpret_cast<const uint2 *>(flag + (size_t)blockIdx.x * srows::CHUNK + threadIdx.x * srows::PER_THREAD);
}
__device__ __forceinline__ int sr_popc(uint2 f) { return __popc(f.x) + __popc(f.y); }    // flags are 0 / 1 bytes

// block-wide scan of x over the 1024 threads: returns the exclusive prefix, *total (shared) gets the block's sum
__device__ __forceinline__ int sr_block_exclusive(int x, int *total) {
    __shared__ int wsum[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        int w = wsum[lane], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += y;
        }
        wsum[lane] = wi - w;                       // exclusive prefix of the warp sums
        if (lane == 31) *total = wi;
    }
    __syncthreads();
    return wsum[warp] + inc - x;
}

__global__ void __launch_bounds__(srows::THREADS)
sparse_count_kernel(const uint8_t *__restrict__ flag, long long *__restrict__ chunk_count)
{
    __shared__ int total;
    sr_block_exclusive(sr_popc(sr_load(flag)), &total);
    if (threadIdx.x == 0) chunk_count[blockIdx.x] = total;
}

// one CTA: chunk_count -> exclusive prefix in place, *count = U
__global__ void __launch_bounds__(srows::THREADS)
sparse_scan_kernel(long long *__restrict__ chunk_count, int n_chunks, long long *__restrict__ count)
{
    __shared__ long long part[srows::THREADS];
    const int per = (n_chunks + srows::THREADS - 1) / srows::THREADS;
    const int lo = threadIdx.x * per, hi = min(lo + per, n_chunks);
    long long s = 0;
    for (int i = lo; i < hi; ++i) s += chunk_count[i];
    part[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {                          // 1024 partial sums: a serial pass is cheap next to the chunk passes
        long long run = 0;
        for (int t = 0; t < srows::THREADS; ++t) { const long long v = part[t]; part[t] = run; run += v; }
        *count = run;
    }
    __syncthreads();
    long long run = part[threadIdx.x];
    for (int i = lo; i < hi; ++i) { const long long v = chunk_count[i]; chunk_count[i] = run; run += v; }
}

__global__ void __launch_bounds__(srows::THREADS)
sparse_compact_kernel(const uint8_t *__restrict__ flag, const long long *__restrict__ chunk_off, long long vocab,
                      int *__restrict__ slot, long long *__restrict__ rows)
{
    __shared__ int total;
    const uint2 f = sr_load(flag);
    int pos = sr_block_exclusive(sr_popc(f), &total);
    const long long base = chunk_off[blockIdx.x];
    const long long r0 = (long long)blockIdx.x * srows::CHUNK + threadIdx.x * srows::PER_THREAD;
    const unsigned w[2] = {f.x, f.y};
#pragma unroll
    for (int k = 0; k < srows::PER_THREAD; ++k) {
        const long long r = r0 + k;
        if (r >= vocab) break;
        if ((w[k >> 2] >> (8 * (k & 3))) & 0xffu) {
            const long long s = base + pos++;
            slot[r] = (int)s;
            rows[s] = r;
        } else {
            slot[r] = -1;
        }
    }
}

static long long sr_chunks(long long vocab) { return (vocab + srows::CHUNK - 1) / srows::CHUNK; }

// [0, flag bytes) flags, padded to whole chunks | chunk counts / offsets (int64)
static size_t sparse_rows_ws(long long vocab) {
    return align_up((size_t)sr_chunks(vocab) * srows::CHUNK, 256) + align_up((size_t)sr_chunks(vocab) * 8, 256);
}

}  // namespace c2v

using namespace c2v;

static bool sr_misaligned(const void *ptr, uintptr_t a) { return (reinterpret_cast<uintptr_t>(ptr) & (a - 1)) != 0; }

// the passes behind the mark: count, scan and compact of the marked flags into rows / *count (and slot)
static int sr_count_scan_compact(const uint8_t *flag, long long *chunk, long long n_chunks, long long vocab, int *slot,
                                 long long *rows, long long *count, cudaStream_t st)
{
    sparse_count_kernel<<<(unsigned)n_chunks, srows::THREADS, 0, st>>>(flag, chunk);
    C2V_LAUNCH_OK("sparse_count_kernel");
    sparse_scan_kernel<<<1, srows::THREADS, 0, st>>>(chunk, (int)n_chunks, count);
    C2V_LAUNCH_OK("sparse_scan_kernel");
    sparse_compact_kernel<<<(unsigned)n_chunks, srows::THREADS, 0, st>>>(flag, chunk, vocab, slot, rows);
    C2V_LAUNCH_OK("sparse_compact_kernel");
    return C2V_OK;
}

extern "C" size_t c2v_sparse_rows_workspace_bytes(int64_t vocab)
{
    if (vocab < 1 || vocab >= (1LL << 31)) return 0;
    return sparse_rows_ws(vocab);
}

extern "C" int c2v_sparse_rows(const int64_t *idx_a, int64_t n_a, const int64_t *idx_b, int64_t n_b, int64_t vocab,
                               int32_t *slot, int64_t *rows, int64_t *count, void *workspace, size_t workspace_bytes,
                               void *stream)
{
    if (vocab < 1 || vocab >= (1LL << 31)) {
        set_error("c2v_sparse_rows: vocab = %lld outside [1, 2^31): slot is int32", (long long)vocab);
        return C2V_EINVAL;
    }
    if (n_a < 0 || n_b < 0) {
        set_error("c2v_sparse_rows: negative index count (n_a = %lld, n_b = %lld)", (long long)n_a, (long long)n_b);
        return C2V_EINVAL;
    }
    if ((n_a > 0 && !idx_a) || (n_b > 0 && !idx_b) || !slot || !count || !workspace || (n_a + n_b > 0 && !rows)) {
        set_error("c2v_sparse_rows: NULL pointer argument");
        return C2V_EINVAL;
    }
    if (sr_misaligned(idx_a, 8) || sr_misaligned(idx_b, 8) || sr_misaligned(slot, 4) || sr_misaligned(rows, 8) ||
        sr_misaligned(count, 8) || sr_misaligned(workspace, 16)) {
        set_error("c2v_sparse_rows: misaligned pointer (indices, rows, count: 8 bytes, slot: 4, workspace: 16)");
        return C2V_EINVAL;
    }
    const size_t need = sparse_rows_ws(vocab);
    if (workspace_bytes < need) {
        set_error("c2v_sparse_rows: workspace too small: %zu < %zu", workspace_bytes, need);
        return C2V_EWORKSPACE;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long n_chunks = sr_chunks(vocab);
    uint8_t *flag = static_cast<uint8_t *>(workspace);
    long long *chunk = reinterpret_cast<long long *>(flag + align_up((size_t)n_chunks * srows::CHUNK, 256));
    C2V_CUDA_OK(cudaMemsetAsync(flag, 0, (size_t)n_chunks * srows::CHUNK, st));
    if (n_a + n_b > 0) {
        long long blocks = (n_a + n_b + 255) / 256;
        if (blocks > 4096) blocks = 4096;
        sparse_mark_kernel<<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const long long *>(idx_a), n_a,
                                                            reinterpret_cast<const long long *>(idx_b), n_b, vocab, flag);
        C2V_LAUNCH_OK("sparse_mark_kernel");
    }
    return sr_count_scan_compact(flag, chunk, n_chunks, vocab, slot, reinterpret_cast<long long *>(rows),
                                 reinterpret_cast<long long *>(count), st);
}

static const int64_t UNION_WORLD_MAX = 1024;

// [0, sparse_rows_ws) the workspace of c2v_sparse_rows | slot map int32 [vocab] (written by the compact pass, not used)
static size_t union_rows_ws(long long vocab) { return sparse_rows_ws(vocab) + align_up((size_t)vocab * 4, 256); }

extern "C" size_t c2v_sparse_union_rows_workspace_bytes(int64_t vocab)
{
    if (vocab < 1 || vocab >= (1LL << 31)) return 0;
    return union_rows_ws(vocab);
}

extern "C" int c2v_sparse_union_rows(const int64_t *rows, const int64_t *counts, int32_t world, int64_t u_max,
                                     int64_t vocab, int64_t *union_rows, int64_t *union_count, void *workspace,
                                     size_t workspace_bytes, void *stream)
{
    if (vocab < 1 || vocab >= (1LL << 31)) {
        set_error("c2v_sparse_union_rows: vocab = %lld outside [1, 2^31)", (long long)vocab);
        return C2V_EINVAL;
    }
    if (world < 1 || world > UNION_WORLD_MAX || u_max < 0 || u_max > vocab) {
        set_error("c2v_sparse_union_rows: world = %d outside [1, %lld] or u_max = %lld outside [0, vocab = %lld]", world,
                  (long long)UNION_WORLD_MAX, (long long)u_max, (long long)vocab);
        return C2V_EINVAL;
    }
    if ((u_max > 0 && (!rows || !union_rows)) || !counts || !union_count || !workspace) {
        set_error("c2v_sparse_union_rows: NULL pointer argument");
        return C2V_EINVAL;
    }
    if (sr_misaligned(rows, 8) || sr_misaligned(counts, 8) || sr_misaligned(union_rows, 8) ||
        sr_misaligned(union_count, 8) || sr_misaligned(workspace, 16)) {
        set_error("c2v_sparse_union_rows: misaligned pointer (rows, counts, union_rows, union_count: 8 bytes, "
                  "workspace: 16)");
        return C2V_EINVAL;
    }
    const size_t need = union_rows_ws(vocab);
    if (workspace_bytes < need) {
        set_error("c2v_sparse_union_rows: workspace too small: %zu < %zu", workspace_bytes, need);
        return C2V_EWORKSPACE;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long n_chunks = sr_chunks(vocab);
    uint8_t *flag = static_cast<uint8_t *>(workspace);
    long long *chunk = reinterpret_cast<long long *>(flag + align_up((size_t)n_chunks * srows::CHUNK, 256));
    int *slot = reinterpret_cast<int *>(static_cast<uint8_t *>(workspace) + sparse_rows_ws(vocab));
    C2V_CUDA_OK(cudaMemsetAsync(flag, 0, (size_t)n_chunks * srows::CHUNK, st));
    if (u_max > 0) {
        long long blocks = (world * u_max + 255) / 256;
        if (blocks > 4096) blocks = 4096;
        sparse_union_mark_kernel<<<(unsigned)blocks, 256, 0, st>>>(reinterpret_cast<const long long *>(rows),
                                                                   reinterpret_cast<const long long *>(counts), world,
                                                                   u_max, vocab, flag);
        C2V_LAUNCH_OK("sparse_union_mark_kernel");
    }
    return sr_count_scan_compact(flag, chunk, n_chunks, vocab, slot, reinterpret_cast<long long *>(union_rows),
                                 reinterpret_cast<long long *>(union_count), st);
}

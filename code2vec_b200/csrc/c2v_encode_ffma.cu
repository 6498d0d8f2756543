// c2v_encode_ffma.cu -- any-shape fp32 CUDA-core encode path + the per-bag finalize.
//
// Replaces model.py:48-69 and get_attention (model.py:90-96) of the reference with
//   K1a encode_ffma_kernel : gathers + concat + input_linear + LayerNorm + tanh (+dropout)
//                            + masked score + per-(tile,bag) online-softmax partials
//   K1f encode_finalize    : merges the partials of each bag -> code_vector, attention
// The [N, D] concat, the [N, H] activations and both expanded products of the eager
// pipeline are never written to HBM.
//
// This is the path for shapes the tensor-core kernel does not take (and for C2V_ALGO_FFMA); it is FFMA-bound.
#include "c2v_ffma_tile.cuh"

namespace c2v {

// ------------------------------------------------------------------------------------
// W [H, D] -> W^T [D][Hs] so the k-chunks of the B operand are coalesced 16-B copies.
// ------------------------------------------------------------------------------------
__global__ void transpose_w_kernel(const float *__restrict__ W, float *__restrict__ Wt, int H,
                                   int D, int Hs)
{
    __shared__ float tile[32][33];
    const int k0 = blockIdx.x * 32, h0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int h = h0 + i, k = k0 + threadIdx.x;
        tile[i][threadIdx.x] = (h < H && k < D) ? W[(size_t)h * D + k] : 0.0f;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int k = k0 + i, h = h0 + threadIdx.x;
        if (k < D && h < Hs) Wt[(size_t)k * Hs + h] = tile[threadIdx.x][i];
    }
}

int launch_transpose_w(const float *W, float *Wt, int H, int D, int Hs, cudaStream_t st)
{
    dim3 grid((D + 31) / 32, (Hs + 31) / 32), block(32, 8);
    transpose_w_kernel<<<grid, block, 0, st>>>(W, Wt, H, D, Hs);
    C2V_LAUNCH_OK("transpose_w_kernel");
    return C2V_OK;
}

// ------------------------------------------------------------------------------------
// K1a
// ------------------------------------------------------------------------------------
template <bool VEC, bool PACKED = false>
__global__ void __launch_bounds__(THREADS)
encode_ffma_kernel(const EncodeArgs a, const int Hs)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const FfmaSmem lay = ffma_smem_layout(Hs);
    long long *sidx = reinterpret_cast<long long *>(smem + lay.idx);
    float *Ac = reinterpret_cast<float *>(smem + lay.ac);
    float *Wc = reinterpret_cast<float *>(smem + lay.wc);
    float *X = reinterpret_cast<float *>(smem + lay.x);
    float *zbuf = reinterpret_cast<float *>(smem + lay.z);
    float *ebuf = reinterpret_cast<float *>(smem + lay.e);
    float *mbuf = reinterpret_cast<float *>(smem + lay.m);

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int H = a.H;

    for (int tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
        const long long row0 = (long long)tile * TM;
        tile_load_indices(a, row0, sidx);                    // model.py:48-50
        __syncthreads();
        tile_gemm_xw<VEC>(a, sidx, Ac, Wc, X, Hs);           // x = c . W^T (model.py:51-54)
        if (a.stash_x) {                                     // training forward: keep x for the backward
            for (int i = threadIdx.x; i < TM * a.H; i += THREADS) {
                const int r = i / a.H, c = i % a.H;
                if (row0 + r < a.N) a.stash_x[(size_t)(row0 + r) * a.H + c] = X[r * Hs + c];
            }
            __syncthreads();                                 // the per-row loop below overwrites X in place (tanh output)
        }

        // ---- LayerNorm + tanh (+dropout) + score, one warp per row (model.py:55-61, 92-93)
        for (int r = warp; r < TM; r += THREADS / 32) {
            const long long row = row0 + r;
            float *xr = X + r * Hs;
            float s = 0.0f;
            for (int c = lane; c < H; c += 32) s += xr[c];
            const float mean = warp_sum(s) / (float)H;
            float v = 0.0f;
            for (int c = lane; c < H; c += 32) { const float d = xr[c] - mean; v = fmaf(d, d, v); }
            const float rstd = 1.0f / sqrtf(warp_sum(v) / (float)H + C2V_LN_EPS);
            const long long drow = (PACKED && row < a.N) ? dropout_row<true>(a, row, bag_of_row<true>(a, row)) : row;
            float u = 0.0f;
            for (int c = lane; c < H; c += 32) {
                float y = tanh_accurate((xr[c] - mean) * rstd * a.ln_g[c] + a.ln_b[c]);
                if (a.drop_p > 0.0f) y *= dropout_mask_at(a.seed, drow, c, a.drop_p, a.drop_scale);
                xr[c] = y;
                u = fmaf(y, a.attn[c], u);
            }
            u = warp_sum(u);
            if (lane == 0) {
                // model.py:64 mask = starts > 0 ; model.py:93 score*mask + (1-mask)*NINF
                const float z = (row < a.N && sidx[r] > 0) ? u : C2V_NINF;
                zbuf[r] = z;
                if (row < a.N) a.attention[row] = z;
            }
        }
        __syncthreads();

        // ---- per-(tile,bag) segment max and exp weights
        const int rows_here = (int)((a.N - row0) < TM ? (a.N - row0) : TM);
        if (tid < rows_here) {
            const long long row = row0 + tid;
            const long long bag = bag_of_row<PACKED>(a, row);
            long long lo = bag_first_row<PACKED>(a, bag) - row0; if (lo < 0) lo = 0;
            long long hi = bag_first_row<PACKED>(a, bag + 1) - row0; if (hi > rows_here) hi = rows_here;
            float m = C2V_NINF;
            for (int q = (int)lo; q < (int)hi; ++q) m = fmaxf(m, zbuf[q]);
            mbuf[tid] = m;
            ebuf[tid] = __expf(zbuf[tid] - m);
        }
        __syncthreads();
        const long long bag_first = bag_of_row<PACKED>(a, row0), bag_last = bag_of_row<PACKED>(a, row0 + rows_here - 1);
        for (long long bag = bag_first; bag <= bag_last; ++bag) {
            long long lo = bag_first_row<PACKED>(a, bag) - row0; if (lo < 0) lo = 0;
            long long hi = bag_first_row<PACKED>(a, bag + 1) - row0; if (hi > rows_here) hi = rows_here;
            const size_t slot = (size_t)tile + (size_t)bag;
            for (int h = tid; h < H; h += THREADS) {
                float v = 0.0f;
                for (int q = (int)lo; q < (int)hi; ++q) v = fmaf(ebuf[q], X[q * Hs + h], v);
                a.ws.part_v[slot * H + h] = v;
            }
            if (tid == 0) {
                float s = 0.0f;
                for (int q = (int)lo; q < (int)hi; ++q) s += ebuf[q];
                a.ws.part_m[slot] = mbuf[lo];
                a.ws.part_s[slot] = s;
            }
        }
        __syncthreads();
    }
}

int launch_encode_ffma(const EncodeArgs &a, cudaStream_t st)
{
    const int Hs = (a.H + 3) / 4 * 4;
    const FfmaSmem lay = ffma_smem_layout(Hs);
    const bool vec = (a.Et % 4 == 0) && (a.Ep % 4 == 0);
    int dev = 0, sms = 0;
    C2V_CUDA_OK(cudaGetDevice(&dev));
    C2V_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    if (lay.total > 227 * 1024) {
        set_error("encode_ffma: encode_size %d needs %d B of shared memory (> 227 KB)", a.H, lay.total);
        return C2V_EUNSUPPORTED;
    }
    auto kern = a.bag_off ? (vec ? encode_ffma_kernel<true, true> : encode_ffma_kernel<false, true>)
                          : (vec ? encode_ffma_kernel<true> : encode_ffma_kernel<false>);
    C2V_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, lay.total));
    int occ = 1;
    C2V_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, THREADS, lay.total));
    if (occ < 1) occ = 1;
    int grid = a.n_tiles < sms * occ ? a.n_tiles : sms * occ;
    if (grid < 1) grid = 1;
    kern<<<grid, THREADS, lay.total, st>>>(a, Hs);
    C2V_LAUNCH_OK("encode_ffma_kernel");
    return C2V_OK;
}

// ------------------------------------------------------------------------------------
// K1f: merge the (tile, bag) partials of every bag (model.py:96 softmax, :68-69 sum)
// ------------------------------------------------------------------------------------
template <bool PACKED = false>
__global__ void __launch_bounds__(128)
encode_finalize_kernel(const EncodeArgs a, const int tile_rows, float *__restrict__ code_vector)
{
    pdl_wait();                                   // launched as a programmatic dependent of the encode kernel
    const long long bag = blockIdx.x;
    if (bag == 0 && threadIdx.x == 0) {           // publish + clear the out-of-range counter (c2v_api.cu)
        const long long bad = a.ws.status[0];
        a.ws.status[3] = bad;
        a.ws.status[0] = 0;
        // host mirror (c2v_workspace_set_status_mirror): a pinned host word the caller polls at its next call, so that
        // an out-of-range index raises IndexError without a synchronisation (the reference's CUDA device-assert is just
        // as deferred).  Words 64 / 65 of the workspace: pointer and pointer ^ magic (never touched by the memsets).
        long long *mirror = reinterpret_cast<long long *>(a.ws.status[64]);
        if (bad != 0 && mirror != nullptr && a.ws.status[65] == (a.ws.status[64] ^ C2V_MIRROR_MAGIC)) {
            atomicAdd_system(reinterpret_cast<unsigned long long *>(mirror), (unsigned long long)bad);
            __threadfence_system();
        }
    }
    // L: the rows of this bag (every row of it in a [B, L] batch)
    const int L = PACKED ? (int)(bag_first_row<true>(a, bag + 1) - bag_first_row<true>(a, bag)) : a.L, H = a.H;
    const long long r0 = bag_first_row<PACKED>(a, bag);
    const int t0 = (int)(r0 / tile_rows), t1 = (int)((r0 + L - 1) / tile_rows);
    const int np = t1 - t0 + 1;
    const size_t slot0 = (size_t)t0 + bag;
    constexpr int NP = 14;                        // partials per bag on the fast path (L = 200, 16-row slices: 13 or 14)
    if (np <= NP && H <= 128) {
        // every load is issued before anything is consumed: one L2 round trip instead of a chain of three
        float pm[NP], ps[NP], pv[NP], z[2];
        const int h = threadIdx.x;
#pragma unroll
        for (int t = 0; t < NP; ++t) {
            const bool on = t < np;
            pm[t] = on ? a.ws.part_m[slot0 + t] : C2V_NINF;
            ps[t] = on ? a.ws.part_s[slot0 + t] : 0.0f;
            pv[t] = (on && h < H) ? a.ws.part_v[(slot0 + t) * H + h] : 0.0f;
        }
        const bool two = L <= 2 * 128;
        if (two) {
#pragma unroll
            for (int k = 0; k < 2; ++k) z[k] = (h + k * 128 < L) ? a.attention[r0 + h + k * 128] : 0.0f;
        }
        float M = C2V_NINF;
#pragma unroll
        for (int t = 0; t < NP; ++t) M = fmaxf(M, pm[t]);
        float S = 0.0f, v = 0.0f;
#pragma unroll
        for (int t = 0; t < NP; ++t) {
            const float w = t < np ? __expf(pm[t] - M) : 0.0f;
            S = fmaf(ps[t], w, S);
            v = fmaf(pv[t], w, v);
        }
        const float inv = 1.0f / S;
        if (h < H) code_vector[bag * H + h] = v * inv;
        if (two) {
#pragma unroll
            for (int k = 0; k < 2; ++k)
                if (h + k * 128 < L) a.attention[r0 + h + k * 128] = __expf(z[k] - M) * inv;
        } else {
            for (int j = h; j < L; j += 128) a.attention[r0 + j] = __expf(a.attention[r0 + j] - M) * inv;
        }
        return;
    }
    float M = C2V_NINF;
    for (int t = t0; t <= t1; ++t) M = fmaxf(M, a.ws.part_m[(size_t)t + bag]);
    float S = 0.0f;
    for (int t = t0; t <= t1; ++t) {
        const size_t slot = (size_t)t + bag;
        S += a.ws.part_s[slot] * __expf(a.ws.part_m[slot] - M);
    }
    const float inv = 1.0f / S;
    for (int h = threadIdx.x; h < H; h += blockDim.x) {
        float v = 0.0f;
        for (int t = t0; t <= t1; ++t) {
            const size_t slot = (size_t)t + bag;
            v = fmaf(a.ws.part_v[slot * H + h], __expf(a.ws.part_m[slot] - M), v);
        }
        code_vector[bag * H + h] = v * inv;
    }
    for (int j = threadIdx.x; j < L; j += blockDim.x) {
        const float z = a.attention[r0 + j];
        a.attention[r0 + j] = __expf(z - M) * inv;
    }
}

// ------------------------------------------------------------------------------------
// packed batches: row_bag[r] = the bag of context row r (one warp per bag; offsets clamped into [0, N])
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
row_bag_kernel(const long long *__restrict__ off, int B, long long N, int *__restrict__ row_bag)
{
    const int bag = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (bag >= B) return;
    long long lo = off[bag], hi = off[bag + 1];
    lo = lo < 0 ? 0 : (lo > N ? N : lo);
    hi = hi < lo ? lo : (hi > N ? N : hi);
    for (long long r = lo + lane; r < hi; r += 32) row_bag[r] = bag;
}

int launch_row_bag(const long long *bag_off, int B, long long N, int *row_bag, cudaStream_t st)
{
    row_bag_kernel<<<(unsigned)((B + 7) / 8), 256, 0, st>>>(bag_off, B, N, row_bag);
    C2V_LAUNCH_OK("row_bag_kernel");
    return C2V_OK;
}

int launch_encode_finalize(const EncodeArgs &a, int B, float *code_vector, cudaStream_t st)
{
    C2V_CUDA_OK(launch_pdl(a.bag_off ? encode_finalize_kernel<true> : encode_finalize_kernel<false>, dim3((unsigned)B), dim3(128), 0,
                           st, a, a.ws.tile_rows, code_vector));
    C2V_LAUNCH_OK("encode_finalize_kernel");
    return C2V_OK;
}

}  // namespace c2v

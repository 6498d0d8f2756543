// c2v_backward_dc_tc.cu -- K3c: dC = dX . W on the tensor cores (wgmma) + scatter into the embedding gradients
// (terminal_embed = path_embed = E <= 256, encode = H <= 256, multiples of 4; zero-padded to 128 inside the panels).
//
// The gradient of the gathered context vectors (autograd of model.py:48-54 under loss.backward(), main.py:174):
//   dC[r, d] = sum_h dX[r, h] * W[h, d],  then  dE_t[starts_r] += dC[r, 0:128], dE_p[paths_r] += dC[r, 128:256],
//   dE_t[ends_r] += dC[r, 256:384]   (nn.Embedding's dense backward; PAD row 0 is a learned row and gets its share).
// M = 128 context rows per tile, N = 128 columns of one sub-vector at a time, K = 128 h.
// A = dX, K-major: the same [128 rows x 64 h] fp16 128-byte-swizzled hi/lo panels the dW kernel builds
// (c2v_backward_dw_tc.cu), read here with K-major descriptors.  B = W^T as a K-major image [128 d x 64 h] per
// (sub-vector, k-block), built once per call by split_wt_kernel and streamed from L2 with 32 KB cp.async.bulk copies.
// 3-pass fp16 hi/lo split, fp32 accumulation in registers; dX is pre-scaled by the power of two from max |dx|, W by the
// one from max |W|.
//
// Warps: 0-7 two consumer warpgroups (warpgroup g: rows 64g .. 64g+63 of the tile; m64n128 wgmma into registers, then
// the scatter straight from the accumulator fragments with vector atomics into the embedding rows) | 8-15 dX producers |
// 16 W^T producer | 17-19 idle.  Work items run (row tile, sub-vector, h block); the dX panels of a row tile are
// re-staged for every sub-vector (L2 hits after the first).
// Sizes above 128: blockIdx.y = db selects the 128-wide window of d inside every sub-vector (its own grid of CTAs over the
// row tiles); the contraction over h runs as n_hb blocks of 128 through the same operand stages, accumulating in
// registers, and the accumulator is scattered after the last block -- so every dC element is still added to the
// embedding gradient exactly once.
#include <cuda_fp16.h>

#include "c2v_tc_ptx.cuh"

namespace c2v {

namespace dct {
constexpr int ROWS = 128, H = 128, E = 128, D = 3 * E;
constexpr int PANEL = ROWS * 64 * 2;                  // 16 KB
constexpr int A_STAGE = 4 * PANEL;                    // hi k0 | hi k1 | lo k0 | lo k1   (k-block = 64 h)
constexpr int B_SLOT = 2 * PANEL;                     // hi | lo of one (sub-vector, k-block) tile of W^T
constexpr int N_PROD_WARPS = 8, PROD_WARP0 = 8, W_WARP = 16;   // warps 0-7: two consumer warpgroups
constexpr int THREADS = 20 * 32;
constexpr int ROWS_PER_PW = ROWS / N_PROD_WARPS;      // 16
constexpr int NB = 6;                                 // W^T tiles per window: (sv, kb), kb minor
constexpr int SMEM_A_OFF = 0, SMEM_B_OFF = 2 * A_STAGE, SMEM_BAR_OFF = SMEM_B_OFF + 2 * B_SLOT;
constexpr int SMEM_BYTES = SMEM_BAR_OFF + 128 + 1024;
constexpr int IMG_BYTES = NB * B_SLOT;                // 192 KB
}  // namespace dct

// W [H][D = 3E] fp32 -> per (db, hb) window pair 6 tiles (sv * 2 + kb) of {hi, lo} [128 d x 64 h] fp16, K-major
// SWIZZLE_128B (d = 128 db + row, h = 128 hb + 64 kb + column; zeros beyond E / H), scaled by the power of two that lifts
// max |W| (bits in *absmax_bits, found by wt_absmax_kernel) just below 2^14.  Image order: [db][hb][sv][kb].
__global__ void wt_absmax_kernel(const float *__restrict__ W, int n, unsigned *__restrict__ absmax_bits)
{
    float m = 0.0f;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) m = fmaxf(m, fabsf(W[i]));
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0) atomicMax(absmax_bits, __float_as_uint(m));
}
__global__ void __launch_bounds__(256)
split_wt_kernel(const float *__restrict__ W, int H, int E, int n_hb, int n_db, const unsigned *__restrict__ absmax_bits,
                uint8_t *__restrict__ img, float *__restrict__ hdr)
{
    const float mx = __uint_as_float(*absmax_bits);
    float scale = 1.0f;
    if (mx > 0.0f && mx < 3.0e38f) {
        int e;
        frexpf(mx, &e);
        int k = 14 - e;
        k = k > 60 ? 60 : (k < -60 ? -60 : k);
        scale = ldexpf(1.0f, k);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) { hdr[0] = 1.0f / scale; hdr[1] = scale; }
    // one thread = 4 consecutive d of one h of one window pair's PADDED [128 h][3 x 128 d] matrix (zeros beyond H / E);
    // coalesced 16-B reads of W's rows ([H][3E] row-major)
    constexpr int PER_WIN = dct::H * dct::D / 4;
    for (int g = blockIdx.x * blockDim.x + threadIdx.x; g < n_db * n_hb * PER_WIN; g += gridDim.x * blockDim.x) {
        const int win = g / PER_WIN, gw = g % PER_WIN;      // win = db * n_hb + hb
        const int db = win / n_hb, hb = win % n_hb;
        const int hl = gw / (dct::D / 4), dp = (gw % (dct::D / 4)) * 4;
        const int sv = dp / dct::E, dl = dp % dct::E, kb = hl / 64, kk = hl % 64;
        const int h = hb * dct::H + hl, d = db * dct::E + dl;
        float4 w4 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (h < H && d < E) w4 = *reinterpret_cast<const float4 *>(W + (size_t)h * (3 * E) + sv * E + d);
        const float wv[4] = {w4.x * scale, w4.y * scale, w4.z * scale, w4.w * scale};
        uint8_t *base = img + ((size_t)win * dct::NB + sv * 2 + kb) * dct::B_SLOT;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const __half hi = __float2half_rn(wv[q]);
            const __half lo = __float2half_rn(wv[q] - __half2float(hi));
            const uint32_t off = sw128_offset(dl + q, kk);
            *reinterpret_cast<__half *>(base + off) = hi;
            *reinterpret_cast<__half *>(base + dct::PANEL + off) = lo;
        }
    }
}

// SPARSE: a table whose slot map in sl is not NULL gets its gradient in compact form, row r of the table adding into row
// sl.<table>[r] of the [U, E] buffer passed as its gradient (sparse embedding gradients, c2v_sparse_rows).  The slot maps
// are a parameter of their own behind all the others, so that the dense instantiation keeps its parameter layout.
template <bool SPARSE = false>
__global__ void __launch_bounds__(dct::THREADS, 1)
backward_dc_tc_kernel(const EncodeArgs a, const float *__restrict__ dx, const unsigned *__restrict__ dx_absmax,
                      const uint8_t *__restrict__ wt_img, const float *__restrict__ wt_hdr,
                      float *__restrict__ g_emb_t, float *__restrict__ g_emb_p, const int sv_mask, const int n_hb,
                      const c2v_row_slots sl)
{
    const int db = (int)blockIdx.y;                     // this CTA's 128-wide window of d inside every sub-vector
    // sv_mask: which sub-vectors (bit 0 start, 1 path, 2 end) this launch handles.  The training step runs the path
    // sub-vector first (mask 2): the path table's gradient is then complete and its data-parallel reduction can overlap
    // the start / end launch (mask 5) -- see ShardedFlatAdam.early_step.
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    const uint32_t bars = base + dct::SMEM_BAR_OFF;
    // a_full[2] @0, a_empty[2] @16, b_full[2] @32, b_empty[2] @48
    const uint32_t bar_afull = bars, bar_aempty = bars + 16, bar_bfull = bars + 32, bar_bempty = bars + 48;
    __shared__ long long s_status[2];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int my_tiles = (a.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int n_sv = (sv_mask & 1) + ((sv_mask >> 1) & 1) + ((sv_mask >> 2) & 1);
    const int n_items = my_tiles * n_sv * n_hb;         // item = (row tile, sub-vector in the mask, h block): one dX stage
    long long *status = s_status;

    if (tid == 0) {
        for (int s = 0; s < 2; ++s) {
            mbar_init(bar_afull + 8 * s, 2 * dct::N_PROD_WARPS);
            mbar_init(bar_aempty + 8 * s, 2);                          // one arrival per consumer warpgroup
            mbar_init(bar_bfull + 8 * s, 1);
            mbar_init(bar_bempty + 8 * s, 2);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    float dx_scale = 1.0f;                              // power of two that lifts max |dx| just below 2^14 (see K3b)
    {
        const float mx = __uint_as_float(*dx_absmax);
        if (mx > 0.0f && mx < 3.0e38f) {
            int e;
            frexpf(mx, &e);
            int k = 14 - e;
            k = k > 100 ? 100 : (k < -100 ? -100 : k);
            dx_scale = ldexpf(1.0f, k);
        }
    }

    if (warp >= dct::PROD_WARP0 && warp < dct::W_WARP) {
        // =============================== dX PRODUCERS ===============================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 88;");
        const int pw = warp - dct::PROD_WARP0;
        const int sub_row = lane >> 4, q = lane & 15;
        uint32_t st_off[dct::ROWS_PER_PW / 2];
#pragma unroll
        for (int j = 0; j < dct::ROWS_PER_PW / 2; ++j) {
            const int r = pw * dct::ROWS_PER_PW + 2 * j + sub_row;
            st_off[j] = (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((((q >> 1) ^ (r & 7)) & 7) << 4) + (q & 1) * 8);
        }
        const float4 *dx4 = reinterpret_cast<const float4 *>(dx);
        const int H4 = a.H / 4;
        for (int vt = 0; vt < n_items; ++vt) {
            const int tl = vt / (n_sv * n_hb), h04 = (vt % n_hb) * 32;    // h block start in 16-byte pieces
            const long long row0 = ((long long)blockIdx.x + (long long)tl * gridDim.x) * dct::ROWS + pw * dct::ROWS_PER_PW;
            const int as = vt & 1;
            float4 buf[2][dct::ROWS_PER_PW / 2];
#pragma unroll
            for (int p = 0; p < 2; ++p)
#pragma unroll
                for (int j = 0; j < dct::ROWS_PER_PW / 2; ++j) {
                    const long long r = row0 + 2 * j + sub_row;
                    float4 v = (r < a.N && h04 + p * 16 + q < H4) ? ldg_nc_v4(dx4 + (size_t)r * H4 + h04 + p * 16 + q)
                                                                  : make_float4(0.f, 0.f, 0.f, 0.f);
                    v.x *= dx_scale; v.y *= dx_scale; v.z *= dx_scale; v.w *= dx_scale;
                    buf[p][j] = v;
                }
            mbar_wait(bar_aempty + 8 * as, (((uint32_t)(vt >> 1)) & 1u) ^ 1u, status);
#pragma unroll
            for (int p = 0; p < 2; ++p) {
                const uint32_t hi = base + dct::SMEM_A_OFF + as * dct::A_STAGE + p * dct::PANEL, lo = hi + 2 * dct::PANEL;
#pragma unroll
                for (int j = 0; j < dct::ROWS_PER_PW / 2; ++j) {
                    const float4 v = buf[p][j];
                    const __half2 h01 = __floats2half2_rn(v.x, v.y), h23 = __floats2half2_rn(v.z, v.w);
                    const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
                    const __half2 l01 = __floats2half2_rn(v.x - f01.x, v.y - f01.y);
                    const __half2 l23 = __floats2half2_rn(v.z - f23.x, v.w - f23.y);
                    sts_v2(hi + st_off[j], pack_h2(h01), pack_h2(h23));
                    sts_v2(lo + st_off[j], pack_h2(l01), pack_h2(l23));
                }
                fence_proxy_async_smem();             // writer side: generic-proxy stores -> visible to the tensor core's async proxy
                __syncwarp();
                if (lane == 0) mbar_arrive(bar_afull + 8 * as);
            }
        }
    } else if (warp >= dct::W_WARP) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 24;");
        // =============================== W^T PRODUCER ===============================
        if (warp == dct::W_WARP && lane == 0) {
            int it = 0;                                  // same (row tile, sub-vector, h block, k-block) order as the MMAs
            for (int tl = 0; tl < my_tiles; ++tl)
                for (int sv = 0; sv < 3; ++sv) {
                    if (!((sv_mask >> sv) & 1)) continue;
                    for (int hb = 0; hb < n_hb; ++hb) {
                        const uint8_t *win = wt_img + (size_t)(db * n_hb + hb) * dct::IMG_BYTES;
                        for (int kb = 0; kb < 2; ++kb, ++it) {
                            const int bs = it & 1;
                            mbar_wait(bar_bempty + 8 * bs, (((uint32_t)(it >> 1)) & 1u) ^ 1u, status);
                            mbar_arrive_expect_tx(bar_bfull + 8 * bs, dct::B_SLOT);
                            bulk_copy_g2s(base + dct::SMEM_B_OFF + bs * dct::B_SLOT, win + (size_t)(sv * 2 + kb) * dct::B_SLOT,
                                          dct::B_SLOT, bar_bfull + 8 * bs);
                        }
                    }
                }
        }
        __syncwarp();
    } else {
        // =============================== CONSUMERS: MMA + SCATTER ===============================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 120;");
        const int g = warp >> 2, w4 = warp & 3, m4 = lane & 3;
        const float inv = wt_hdr[0] / dx_scale;        // exact: both scales are powers of two
        int vt = 0, it = 0;
        for (int tl = 0; tl < my_tiles; ++tl) {
            long long row[2], idx[2][3];
            bool in_range[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                row[h] = ((long long)blockIdx.x + (long long)tl * gridDim.x) * dct::ROWS + 64 * g + 16 * w4 + (lane >> 2) + 8 * h;
                in_range[h] = row[h] < a.N;
                long long is = 0, ip = 0, ie = 0;
                if (in_range[h]) { is = a.starts[row[h]]; ip = a.paths[row[h]]; ie = a.ends[row[h]]; }
                idx[h][0] = (is < 0 || is >= a.T) ? 0 : is;
                idx[h][1] = (ip < 0 || ip >= a.P) ? 0 : ip;
                idx[h][2] = (ie < 0 || ie >= a.T) ? 0 : ie;
            }
#pragma unroll 1
            for (int sv = 0; sv < 3; ++sv) {
                if (!((sv_mask >> sv) & 1)) continue;
                float acc[64];
                for (int hb = 0; hb < n_hb; ++hb, ++vt) {
                    const int as = vt & 1;
                    mbar_wait(bar_afull + 8 * as, ((uint32_t)(vt >> 1)) & 1u, status);
#pragma unroll
                    for (int kb = 0; kb < 2; ++kb, ++it) {
                        const int bs = it & 1;
                        mbar_wait(bar_bfull + 8 * bs, ((uint32_t)(it >> 1)) & 1u, status);
                        const uint32_t sa = base + dct::SMEM_A_OFF + as * dct::A_STAGE + kb * dct::PANEL + g * (dct::PANEL / 2);
                        const uint32_t sb = base + dct::SMEM_B_OFF + bs * dct::B_SLOT;
                        wgmma_fence();
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            const uint64_t a_hi = wgmma_desc(sa + k * 32), a_lo = wgmma_desc(sa + 2 * dct::PANEL + k * 32);
                            const uint64_t b_hi = wgmma_desc(sb + k * 32), b_lo = wgmma_desc(sb + dct::PANEL + k * 32);
                            wgmma_m64n128<0>(acc, a_hi, b_hi, (hb | kb | k) != 0);
                            wgmma_m64n128<0>(acc, a_lo, b_hi, 1);
                            wgmma_m64n128<0>(acc, a_hi, b_lo, 1);
                        }
                        wgmma_commit();
                        wgmma_wait<0>();
                        if ((tid & 127) == 0) mbar_arrive(bar_bempty + 8 * bs);
                    }
                    if ((tid & 127) == 0) mbar_arrive(bar_aempty + 8 * as);
                }
#pragma unroll
                for (int i = 0; i < 64; ++i) fence_operand(acc[i]);
                // acc[4j + 2h + b] is row[h], column 8j + 2 (lane & 3) + b of the window: a lane quad adds 32 contiguous
                // bytes of one embedding row per instruction
                float *tab = sv == 1 ? g_emb_p : g_emb_t;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!in_range[h]) continue;
                    float *dst = tab + (size_t)idx[h][sv] * a.Et + db * dct::E;
                    if constexpr (SPARSE) {           // compact gradient: the row's slot (tables without a slot map: the row)
                        const int *slot = sv == 1 ? sl.path : sl.terminal;
                        if (slot) dst = tab + (size_t)slot[idx[h][sv]] * a.Et + db * dct::E;
                    }
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const int c = 8 * j + 2 * m4;
                        const float x = acc[4 * j + 2 * h] * inv, y = acc[4 * j + 2 * h + 1] * inv;
                        if (db * dct::E + c < a.Et && (x != 0.0f || y != 0.0f))          // padded contexts: dx == 0
                            red_add_v2(dst + c, x, y);
                    }
                }
            }
        }
    }
}

bool backward_dc_tc_ok(const EncodeArgs &a) {
    return a.Et == a.Ep && a.Et <= 2 * dct::E && a.H <= 2 * dct::H && (a.Et & 3) == 0 && (a.H & 3) == 0 &&
           (long long)a.T * (a.Et / 4) < 0xFFFFFFFFll && (long long)a.P * (a.Et / 4) < 0xFFFFFFFFll;
}
size_t backward_dc_tc_workspace_bytes() { return 1024 + 4 * dct::IMG_BYTES; }      // up to 2 x 2 window pairs

// ws: [0, 1024) header {1/scale, scale} | W^T images [db][hb]
int launch_backward_dc_tc(const EncodeArgs &a_in, const float *W, const float *dx, const unsigned *dx_absmax, void *ws,
                          float *g_emb_t, float *g_emb_p, cudaStream_t st, int sv_mask, bool build_image,
                          const c2v_row_slots *slots)
{
    EncodeArgs a = a_in;
    a.n_tiles = (int)((a.N + dct::ROWS - 1) / dct::ROWS);
    float *hdr = static_cast<float *>(ws);
    uint8_t *img = static_cast<uint8_t *>(ws) + 1024;
    const int n_hb = (a.H + dct::H - 1) / dct::H, n_db = (a.Et + dct::E - 1) / dct::E;
    unsigned *mxbits = reinterpret_cast<unsigned *>(static_cast<uint8_t *>(ws) + 512);
    if (build_image) {
        C2V_CUDA_OK(cudaMemsetAsync(mxbits, 0, 4, st));
        wt_absmax_kernel<<<48, 256, 0, st>>>(W, a.H * a.D, mxbits);
        C2V_LAUNCH_OK("wt_absmax_kernel");
        split_wt_kernel<<<48 * n_hb * n_db, 256, 0, st>>>(W, a.H, a.Et, n_hb, n_db, mxbits, img, hdr);
        C2V_LAUNCH_OK("split_wt_kernel");
    }
    if ((sv_mask & 7) == 0) return C2V_OK;
    int dev = 0, sms = 0;
    C2V_CUDA_OK(cudaGetDevice(&dev));
    C2V_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const bool sparse = slots && (slots->terminal || slots->path);
    auto kern = sparse ? backward_dc_tc_kernel<true> : backward_dc_tc_kernel<false>;
    C2V_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, dct::SMEM_BYTES));
    int grid = sms / n_db;                                 // one CTA per SM over the d windows
    if (grid > a.n_tiles) grid = a.n_tiles;
    if (grid < 1) grid = 1;
    c2v_row_slots sl = {nullptr, nullptr};
    if (sparse) sl = *slots;
    kern<<<dim3(grid, n_db), dct::THREADS, dct::SMEM_BYTES, st>>>(a, dx, dx_absmax, img, hdr, g_emb_t, g_emb_p, sv_mask & 7,
                                                                  n_hb, sl);
    C2V_LAUNCH_OK("backward_dc_tc_kernel");
    return C2V_OK;
}

}  // namespace c2v

// c2v_label_backward_tc.cu -- backward of the label head  outputs = cv . W_out^T + b  (model.py:83 under loss.backward(),
// main.py:174) on the tensor cores (wgmma).  G = d loss / d outputs [B, C] fp32 (row-major, any C):
//   LB1  dW_out[c, h] = sum_b G[b, c] cv[b, h]      M = c, N = h, K = b : both operands MN-major (the row index is K)
//        d_b[c]       = sum_b G[b, c]               (column sums, folded into LB1's producers)
//   LB2  d_cv[b, h]   = sum_c G[b, c] W_out[c, h]   M = b, N = h, K = c : A K-major (G rows), B MN-major = the forward's
//        cached W_out image ([128 c x 64 h] fp16 hi/lo tiles) streamed as it is with cp.async.bulk
// Same fp32-accurate scheme as everywhere: operands split into fp16 hi + lo, three f16 MMAs per k-step
// (hi.hi + lo.hi + hi.lo; hi.hi alone under C2V_MATMUL_TF32), fp32 accumulation in registers; G is multiplied by the power of two that lifts max |G| just
// below 2^14 before the split (mean-NLL gradients are ~1e-6) and the result by its exact inverse.
// The shared-memory image of a G tile is identical for both kernels ([128 rows(b) x 64 cols(c)] 128-byte-swizzled
// panels); only the descriptors differ (MN-major in LB1, K-major in LB2).
// Warps of both kernels: 0-7 two consumer warpgroups (warpgroup g: output rows 64g .. 64g+63 of the 128-row tile, one
// m64n64 accumulator per 64-wide block of h, NKB = ceil(H / 64) of them) | 8-15 producers (16 rows each) | 16 bulk copies.
#include <cuda_fp16.h>

#include <cstring>

#include "c2v_tc_ptx.cuh"

namespace c2v {

namespace lbt {
constexpr int ROWS = 128;
constexpr int PANEL = ROWS * 64 * 2;                  // 16 KB: [128 rows x 64 cols] fp16
constexpr int N_PROD_WARPS = 8, PROD_WARP0 = 8, BULK_WARP = 16;
constexpr int THREADS = 20 * 32;                      // warps 17-19 only donate registers
constexpr int ROWS_PER_PW = ROWS / N_PROD_WARPS;      // 16
constexpr int LD = ROWS_PER_PW / 2;                   // loads per lane and panel (two rows per instruction)
}  // namespace lbt

// byte offset of the 8-byte piece q (of 16) of row r inside a [rows x 64] fp16 128-byte-swizzled panel
__device__ __forceinline__ uint32_t lbt_st_off(int r, int q) {
    return (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((((q >> 1) ^ (r & 7)) & 7) << 4) + (q & 1) * 8);
}
__device__ __forceinline__ float lbt_scale_from_absmax(unsigned bits) {
    const float mx = __uint_as_float(bits);
    if (!(mx > 0.0f && mx < 3.0e38f)) return 1.0f;
    int e;
    frexpf(mx, &e);
    int k = 14 - e;
    k = k > 100 ? 100 : (k < -100 ? -100 : k);
    return ldexpf(1.0f, k);
}
// 4 consecutive floats of a row that may be only 4-byte aligned (C odd) and may run off the end of the row
__device__ __forceinline__ float4 lbt_load4(const float *p, long long remaining, bool vec) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (remaining >= 4 && vec) return ldg_nc_v4(reinterpret_cast<const float4 *>(p));
    if (remaining > 0) v.x = __ldg(p);
    if (remaining > 1) v.y = __ldg(p + 1);
    if (remaining > 2) v.z = __ldg(p + 2);
    if (remaining > 3) v.w = __ldg(p + 3);
    return v;
}
template <class PASS>
__device__ __forceinline__ void lbt_split_store(uint32_t hi, uint32_t lo, uint32_t off, float4 v) {
    const __half2 h01 = __floats2half2_rn(v.x, v.y), h23 = __floats2half2_rn(v.z, v.w);
    const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
    const __half2 l01 = __floats2half2_rn(v.x - f01.x, v.y - f01.y), l23 = __floats2half2_rn(v.z - f23.x, v.w - f23.y);
    sts_v2(hi + off, pack_h2(h01), pack_h2(h23));
    if constexpr (!one_pass<PASS>) sts_v2(lo + off, pack_h2(l01), pack_h2(l23));     // OnePass: no lo half
}

__global__ void lbt_absmax_kernel(const float *__restrict__ x, long long n, unsigned *__restrict__ out_bits)
{
    float m = 0.0f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        m = fmaxf(m, fabsf(x[i]));
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0 && m > 0.0f) atomicMax(out_bits, __float_as_uint(m));
}

// ------------------------------------------------------------------------------------------------------------------
// LB1: dW_out [C, H] and d_b [C].  One persistent CTA walks label tiles (128 labels); per label tile all batch tiles
// (128 bags) stream through: A = G[bags, labels] as two 64-label panels (warpgroup g multiplies panel g), B = cv[bags, 64 h]
// panels; the [128 c x HP h] accumulator is complete after the last batch tile and written out from the fragments.
// smem: 2 A stages {hi p0, hi p1, lo p0, lo p1} (128 KB) + 2 B slots {hi, lo} (64 KB) + column-sum scratch + barriers.
// ------------------------------------------------------------------------------------------------------------------
namespace lb1 {
constexpr int A_STAGE = 4 * lbt::PANEL, B_SLOT = 2 * lbt::PANEL;
constexpr int SMEM_A_OFF = 0, SMEM_B_OFF = 2 * A_STAGE, SMEM_CS_OFF = SMEM_B_OFF + 2 * B_SLOT;   // column sums [8][128] fp32
constexpr int SMEM_BAR_OFF = SMEM_CS_OFF + lbt::N_PROD_WARPS * 128 * 4;
constexpr int SMEM_BYTES = SMEM_BAR_OFF + 128 + 1024;
}  // namespace lb1

// CV_IMG: the B operand (cv) is not converted here at all: `cv_img` is the fp16 hi/lo image of cv that the label GEMM of the
// same step left in the label workspace ([128 bags x 64 h] K-major 128-byte-swizzled tiles = the very bytes an MN-major B
// tile of this GEMM needs), streamed by warp 16 with one 32 KB cp.async.bulk per (batch tile, k-block); the producers then
// only handle G.
// PASS = OnePass (C2V_MATMUL_TF32): hi.hi only; no lo panels are stored or copied.
template <bool CV_IMG, int NKB, class PASS = ThreePass>
__global__ void __launch_bounds__(lbt::THREADS, 1)
label_dw_tc_kernel(const float *__restrict__ G, const float *__restrict__ cv, int B, long long C, int H,
                   const unsigned *__restrict__ g_absmax, float *__restrict__ dW, float *__restrict__ d_bias,
                   const uint8_t *__restrict__ cv_img)
{
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    unsigned char *smem = smem_raw + (base - raw);
    float *s_cs = reinterpret_cast<float *>(smem + lb1::SMEM_CS_OFF);
    const uint32_t bars = base + lb1::SMEM_BAR_OFF;
    // a_full[2] @0, a_empty[2] @16, b_full[2] @32, b_empty[2] @48
    const uint32_t bar_afull = bars, bar_aempty = bars + 16, bar_bfull = bars + 32, bar_bempty = bars + 48;
    __shared__ long long s_status[2];
    long long *status = s_status;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n_bt = (B + 127) / 128;
    const long long n_ct = (C + 127) / 128;
    const int my_ct = (int)((n_ct - (long long)blockIdx.x + (long long)gridDim.x - 1) / (long long)gridDim.x);

    if (tid == 0) {
        for (int s = 0; s < 2; ++s) {
            mbar_init(bar_afull + 8 * s, 2 * lbt::N_PROD_WARPS);
            mbar_init(bar_aempty + 8 * s, 2);                          // one arrival per consumer warpgroup
            mbar_init(bar_bfull + 8 * s, CV_IMG ? 1 : lbt::N_PROD_WARPS);
            mbar_init(bar_bempty + 8 * s, 2);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const float g_scale = lbt_scale_from_absmax(*g_absmax);

    if (warp >= lbt::PROD_WARP0 && warp < lbt::BULK_WARP) {
        // =============================== PRODUCERS ===============================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
        const int pw = warp - lbt::PROD_WARP0;
        const int sub_row = lane >> 4, q = lane & 15;   // lanes 0-15: row 2j, lanes 16-31: row 2j+1; q = 16-B column piece
        const bool vecG = (C & 3) == 0 && (reinterpret_cast<uintptr_t>(G) & 15) == 0;
        int ita = 0, itb = 0;                          // running A-stage / B-slot counters
        for (int cl = 0; cl < my_ct; ++cl) {
            const long long ct = (long long)blockIdx.x + (long long)cl * gridDim.x;
            const long long c0 = ct * 128;
            float4 cs[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};   // column sums (unscaled)
            for (int bt = 0; bt < n_bt; ++bt, ++ita) {
                const int row0 = bt * 128 + pw * lbt::ROWS_PER_PW;
                const int as = ita & 1;
#pragma unroll
                for (int p = 0; p < 2; ++p) {
                    float4 g[lbt::LD];                   // one panel's loads in flight before the stage wait
#pragma unroll
                    for (int j = 0; j < lbt::LD; ++j) {
                        const int r = row0 + 2 * j + sub_row;
                        const long long c = c0 + p * 64 + q * 4;
                        g[j] = make_float4(0.f, 0.f, 0.f, 0.f);
                        if (r < B) g[j] = lbt_load4(G + (size_t)r * C + c, C - c, vecG);
                    }
                    if (p == 0) mbar_wait(bar_aempty + 8 * as, (((uint32_t)(ita >> 1)) & 1u) ^ 1u, status);
                    const uint32_t hi = base + lb1::SMEM_A_OFF + as * lb1::A_STAGE + p * lbt::PANEL, lo = hi + 2 * lbt::PANEL;
#pragma unroll
                    for (int j = 0; j < lbt::LD; ++j) {
                        float4 v = g[j];
                        cs[p].x += v.x; cs[p].y += v.y; cs[p].z += v.z; cs[p].w += v.w;
                        v.x *= g_scale; v.y *= g_scale; v.z *= g_scale; v.w *= g_scale;
                        lbt_split_store<PASS>(hi, lo, lbt_st_off(pw * lbt::ROWS_PER_PW + 2 * j + sub_row, q), v);
                    }
                    fence_proxy_async_smem();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bar_afull + 8 * as);
                }
#pragma unroll 1
                for (int kb = 0; kb < (CV_IMG ? 0 : NKB); ++kb, ++itb) {
                    const int bs = itb & 1;
                    float4 buf[lbt::LD];
#pragma unroll
                    for (int j = 0; j < lbt::LD; ++j) {
                        const int r = row0 + 2 * j + sub_row;
                        const int h = kb * 64 + q * 4;
                        buf[j] = (r < B && h < H) ? ldg_nc_v4(reinterpret_cast<const float4 *>(cv + (size_t)r * H + h))
                                                  : make_float4(0.f, 0.f, 0.f, 0.f);
                    }
                    mbar_wait(bar_bempty + 8 * bs, (((uint32_t)(itb >> 1)) & 1u) ^ 1u, status);
                    const uint32_t hi = base + lb1::SMEM_B_OFF + bs * lb1::B_SLOT;
#pragma unroll
                    for (int j = 0; j < lbt::LD; ++j)
                        lbt_split_store<PASS>(hi, hi + lbt::PANEL, lbt_st_off(pw * lbt::ROWS_PER_PW + 2 * j + sub_row, q), buf[j]);
                    fence_proxy_async_smem();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bar_bfull + 8 * bs);
                }
            }
            // ---- d_b of this label tile: lanes q / q+16 hold the same columns; 8 warps -> smem -> 128 threads
            if (d_bias) {
#pragma unroll
                for (int p = 0; p < 2; ++p) {
                    cs[p].x += __shfl_xor_sync(0xffffffffu, cs[p].x, 16); cs[p].y += __shfl_xor_sync(0xffffffffu, cs[p].y, 16);
                    cs[p].z += __shfl_xor_sync(0xffffffffu, cs[p].z, 16); cs[p].w += __shfl_xor_sync(0xffffffffu, cs[p].w, 16);
                    if (sub_row == 0) *reinterpret_cast<float4 *>(s_cs + pw * 128 + p * 64 + q * 4) = cs[p];
                }
                named_bar_sync(2, lbt::N_PROD_WARPS * 32);
                const int t = pw * 32 + lane;                             // 0..255
                if (t < 128) {
                    float s = 0.0f;
#pragma unroll
                    for (int w = 0; w < lbt::N_PROD_WARPS; ++w) s += s_cs[w * 128 + t];
                    if (c0 + t < C) d_bias[c0 + t] = s;
                }
                named_bar_sync(2, lbt::N_PROD_WARPS * 32);                // scratch is rewritten by the next label tile
            }
        }
    } else if (warp >= lbt::BULK_WARP) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        // =============================== cv IMAGE PRODUCER (cp.async.bulk) ===============================
        if (CV_IMG && warp == lbt::BULK_WARP && lane == 0) {
            int itb = 0;
            for (int cl = 0; cl < my_ct; ++cl)
                for (int bt = 0; bt < n_bt; ++bt)
                    for (int kb = 0; kb < NKB; ++kb, ++itb) {
                        const int bs = itb & 1;
                        mbar_wait(bar_bempty + 8 * bs, (((uint32_t)(itb >> 1)) & 1u) ^ 1u, status);
                        constexpr uint32_t bytes = one_pass<PASS> ? lbt::PANEL : lb1::B_SLOT;     // hi first in the image
                        mbar_arrive_expect_tx(bar_bfull + 8 * bs, bytes);
                        bulk_copy_g2s(base + lb1::SMEM_B_OFF + bs * lb1::B_SLOT, cv_img + ((size_t)bt * NKB + kb) * lb1::B_SLOT,
                                      bytes, bar_bfull + 8 * bs);
                    }
        }
        __syncwarp();
    } else {
        // =============================== CONSUMERS: MMA + dW_out rows ===============================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 160;");
        const int g = warp >> 2, w4 = warp & 3, m4 = lane & 3;
        const float inv = 1.0f / g_scale;
        float acc[NKB][32];
        int ita = 0, itb = 0;
        for (int cl = 0; cl < my_ct; ++cl) {
            for (int bt = 0; bt < n_bt; ++bt, ++ita) {
                const int as = ita & 1;
                mbar_wait(bar_afull + 8 * as, ((uint32_t)(ita >> 1)) & 1u, status);
                const uint32_t sa = base + lb1::SMEM_A_OFF + as * lb1::A_STAGE + g * lbt::PANEL;   // label panel g
#pragma unroll
                for (int kb = 0; kb < NKB; ++kb, ++itb) {
                    const int bs = itb & 1;
                    mbar_wait(bar_bfull + 8 * bs, ((uint32_t)(itb >> 1)) & 1u, status);
                    const uint32_t sb = base + lb1::SMEM_B_OFF + bs * lb1::B_SLOT;
                    wgmma_fence();
#pragma unroll
                    for (int k = 0; k < lbt::ROWS / 16; ++k) {
                        const uint64_t a_hi = wgmma_desc_mn(sa + k * 2048, lbt::PANEL);
                        const uint64_t a_lo = wgmma_desc_mn(sa + 2 * lbt::PANEL + k * 2048, lbt::PANEL);
                        const uint64_t b_hi = wgmma_desc_mn(sb + k * 2048, lbt::PANEL);
                        const uint64_t b_lo = wgmma_desc_mn(sb + lbt::PANEL + k * 2048, lbt::PANEL);
                        wgmma_m64n64<1, 1>(acc[kb], a_hi, b_hi, (bt | k) != 0);
                        if constexpr (one_pass<PASS>) continue;
                        wgmma_m64n64<1, 1>(acc[kb], a_lo, b_hi, 1);
                        wgmma_m64n64<1, 1>(acc[kb], a_hi, b_lo, 1);
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    if ((tid & 127) == 0) mbar_arrive(bar_bempty + 8 * bs);
                }
                if ((tid & 127) == 0) mbar_arrive(bar_aempty + 8 * as);
            }
#pragma unroll
            for (int kb = 0; kb < NKB; ++kb)
#pragma unroll
                for (int i = 0; i < 32; ++i) fence_operand(acc[kb][i]);
            // acc[kb][4j + 2hh + b] is label c0 + 64g + 16 w4 + lane/4 + 8hh, h = 64kb + 8j + 2 (lane & 3) + b
            const long long c0 = ((long long)blockIdx.x + (long long)cl * gridDim.x) * 128 + 64 * g + 16 * w4 + (lane >> 2);
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const long long c = c0 + 8 * hh;
                if (c >= C) continue;
                float *dst = dW + (size_t)c * H;
#pragma unroll
                for (int kb = 0; kb < NKB; ++kb)
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const int h = 64 * kb + 8 * j + 2 * m4;
                        if (h < H)
                            *reinterpret_cast<float2 *>(dst + h) = make_float2(acc[kb][4 * j + 2 * hh] * inv, acc[kb][4 * j + 2 * hh + 1] * inv);
                    }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------------------------
// LB2: d_cv [B, H] += G[bags, label range] . W_out[label range, :]   (split over the label dimension, fp32 atomics).
// Work item = (batch tile, label split); k-block = 64 labels: A = one K-major G panel {hi, lo} (32 KB, 3 stages; warpgroup
// g reads its 64 bags), B = rows [64 half] of the forward's W_out image tiles, NKB x {hi 8 KB, lo 8 KB} (3 stages).
// ------------------------------------------------------------------------------------------------------------------
namespace lb2 {
constexpr int MAX_STAGES = 3;
constexpr int A_STAGE = 2 * lbt::PANEL;               // hi | lo, [128 bags x 64 labels]
constexpr int B_HALF = 64 * 128;                      // 8 KB: 64 label rows x 64 h fp16
constexpr int SMEM_A_OFF = 0;
}  // namespace lb2
// the B stage is nkb x {hi, lo} x 8 KB: 3 stages of (32 + 32) KB at encode_size <= 128, 2 stages of (32 + 64) KB at 256
static inline int lb2_stages(int nkb) { return nkb <= 2 ? 3 : 2; }
static inline int lb2_smem_bytes(int nkb) { return lb2_stages(nkb) * (lb2::A_STAGE + nkb * 2 * lb2::B_HALF) + 128 + 1024; }

// DET (deterministic mode): d_cv is the slab array [n_split][B][H]; label split sp stores its partial to slab sp.
// PASS = OnePass (C2V_MATMUL_TF32): hi.hi only; the G producers store no lo panel and only the hi halves of W_out are copied.
template <int NKB, bool DET = false, class PASS = ThreePass>
__global__ void __launch_bounds__(lbt::THREADS, 1)
label_dcv_tc_kernel(const float *__restrict__ G, int B, long long C, int H, const uint8_t *__restrict__ w_img,
                    const float *__restrict__ w_hdr, const unsigned *__restrict__ g_absmax, int n_split,
                    long long kblocks_per_split, float *__restrict__ d_cv, const int S)
{
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    constexpr int b_stage = NKB * 2 * lb2::B_HALF;
    const uint32_t smem_b = base + S * lb2::A_STAGE;
    const uint32_t bars = smem_b + S * b_stage;
    // a_full[3] @0, a_empty[3] @24, b_full[3] @48, b_empty[3] @72
    const uint32_t bar_afull = bars, bar_aempty = bars + 24, bar_bfull = bars + 48, bar_bempty = bars + 72;
    __shared__ long long s_status[2];
    long long *status = s_status;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n_bt = (B + 127) / 128;
    const int n_items = n_bt * n_split;
    const int my_items = (n_items - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const long long n_kblocks = (C + 63) / 64;

    if (tid == 0) {
        for (int s = 0; s < lb2::MAX_STAGES; ++s) {
            mbar_init(bar_afull + 8 * s, lbt::N_PROD_WARPS);
            mbar_init(bar_aempty + 8 * s, 2);                          // one arrival per consumer warpgroup
            mbar_init(bar_bfull + 8 * s, 1);
            mbar_init(bar_bempty + 8 * s, 2);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const float g_scale = lbt_scale_from_absmax(*g_absmax);

    // item -> (batch tile, first k-block, number of k-blocks)
    auto item_range = [&](int il, int &bt, long long &kb0, long long &nk) {
        const int item = (int)blockIdx.x + il * (int)gridDim.x;
        bt = item / n_split;
        const int sp = item - bt * n_split;
        kb0 = (long long)sp * kblocks_per_split;
        nk = n_kblocks - kb0; if (nk > kblocks_per_split) nk = kblocks_per_split; if (nk < 0) nk = 0;
    };

    if (warp >= lbt::PROD_WARP0 && warp < lbt::BULK_WARP) {
        // =============================== G PRODUCERS (K-major panels) ===============================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
        const int pw = warp - lbt::PROD_WARP0;
        const int sub_row = lane >> 4, q = lane & 15;
        const bool vecG = (C & 3) == 0 && (reinterpret_cast<uintptr_t>(G) & 15) == 0;
        int it = 0;
        for (int il = 0; il < my_items; ++il) {
            int bt; long long kb0, nk;
            item_range(il, bt, kb0, nk);
            const int row0 = bt * 128 + pw * lbt::ROWS_PER_PW;
            for (long long kk = 0; kk < nk; ++kk, ++it) {
                const long long c = (kb0 + kk) * 64 + q * 4;
                float4 buf[lbt::LD];
#pragma unroll
                for (int j = 0; j < lbt::LD; ++j) {
                    const int r = row0 + 2 * j + sub_row;
                    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (r < B) v = lbt_load4(G + (size_t)r * C + c, C - c, vecG);
                    v.x *= g_scale; v.y *= g_scale; v.z *= g_scale; v.w *= g_scale;
                    buf[j] = v;
                }
                const int st = it % S;
                mbar_wait(bar_aempty + 8 * st, (((uint32_t)(it / S)) & 1u) ^ 1u, status);
                const uint32_t hi = base + lb2::SMEM_A_OFF + st * lb2::A_STAGE;
#pragma unroll
                for (int j = 0; j < lbt::LD; ++j)
                    lbt_split_store<PASS>(hi, hi + lbt::PANEL, lbt_st_off(pw * lbt::ROWS_PER_PW + 2 * j + sub_row, q), buf[j]);
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) mbar_arrive(bar_afull + 8 * st);
            }
        }
    } else if (warp >= lbt::BULK_WARP) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        // =============================== W_out IMAGE PRODUCER (cp.async.bulk) ===============================
        if (warp == lbt::BULK_WARP && lane == 0) {
            int it = 0;
            for (int il = 0; il < my_items; ++il) {
                int bt; long long kb0, nk;
                item_range(il, bt, kb0, nk);
                for (long long kk = 0; kk < nk; ++kk, ++it) {
                    const long long kblk = kb0 + kk;                 // 64-label block
                    const long long nt = kblk >> 1;                  // 128-label tile of the image
                    const int half = (int)(kblk & 1);
                    const int st = it % S;
                    mbar_wait(bar_bempty + 8 * st, (((uint32_t)(it / S)) & 1u) ^ 1u, status);
                    mbar_arrive_expect_tx(bar_bfull + 8 * st, (uint32_t)(one_pass<PASS> ? b_stage / 2 : b_stage));
                    for (int kb = 0; kb < NKB; ++kb) {
                        const uint8_t *src = w_img + ((size_t)nt * NKB + kb) * (size_t)(2 * lbt::PANEL) + half * lb2::B_HALF;
                        const uint32_t dst = smem_b + st * b_stage + kb * 2 * lb2::B_HALF;
                        bulk_copy_g2s(dst, src, lb2::B_HALF, bar_bfull + 8 * st);                                // hi
                        if constexpr (!one_pass<PASS>)
                            bulk_copy_g2s(dst + lb2::B_HALF, src + lbt::PANEL, lb2::B_HALF, bar_bfull + 8 * st); // lo
                    }
                }
            }
        }
        __syncwarp();
    } else {
        // =============================== CONSUMERS: MMA + atomics into d_cv ===============================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 160;");
        const int g = warp >> 2, w4 = warp & 3, m4 = lane & 3;
        const float inv = w_hdr[0] / g_scale;
        float acc[NKB][32];
        int it = 0;
        for (int il = 0; il < my_items; ++il) {
            int bt; long long kb0, nk;
            item_range(il, bt, kb0, nk);
            for (long long kk = 0; kk < nk; ++kk, ++it) {
                const int st = it % S;
                const uint32_t ph = ((uint32_t)(it / S)) & 1u;
                mbar_wait(bar_afull + 8 * st, ph, status);
                mbar_wait(bar_bfull + 8 * st, ph, status);
                const uint32_t sa = base + lb2::SMEM_A_OFF + st * lb2::A_STAGE + g * (lbt::PANEL / 2);   // bags 64g ..
                const uint32_t sb = smem_b + st * b_stage;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) {                       // 64 labels = 4 k-steps of 16
                    const uint64_t a_hi = wgmma_desc(sa + k * 32), a_lo = wgmma_desc(sa + lbt::PANEL + k * 32);
#pragma unroll
                    for (int kb = 0; kb < NKB; ++kb) {
                        // B: MN-major, 16 label rows x 128 B per k-step, one 64-column group of h per kb
                        const uint64_t b_hi = wgmma_desc_mn(sb + kb * 2 * lb2::B_HALF + k * 2048, 2 * lb2::B_HALF);
                        const uint64_t b_lo = wgmma_desc_mn(sb + kb * 2 * lb2::B_HALF + lb2::B_HALF + k * 2048, 2 * lb2::B_HALF);
                        wgmma_m64n64<0, 1>(acc[kb], a_hi, b_hi, (kk | k) != 0);
                        if constexpr (one_pass<PASS>) continue;
                        wgmma_m64n64<0, 1>(acc[kb], a_lo, b_hi, 1);
                        wgmma_m64n64<0, 1>(acc[kb], a_hi, b_lo, 1);
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
                if ((tid & 127) == 0) { mbar_arrive(bar_aempty + 8 * st); mbar_arrive(bar_bempty + 8 * st); }
            }
            if (nk > 0) {
#pragma unroll
                for (int kb = 0; kb < NKB; ++kb)
#pragma unroll
                    for (int i = 0; i < 32; ++i) fence_operand(acc[kb][i]);
                // acc[kb][4j + 2hh + b] is bag 64g + 16 w4 + lane/4 + 8hh of the tile, h = 64kb + 8j + 2 (lane & 3) + b
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    const int b = bt * 128 + 64 * g + 16 * w4 + (lane >> 2) + 8 * hh;
                    if (b >= B) continue;
                    float *dst = d_cv + (size_t)b * H;
                    if (DET) dst += (size_t)(kb0 / kblocks_per_split) * B * H;
#pragma unroll
                    for (int kb = 0; kb < NKB; ++kb)
#pragma unroll
                        for (int j = 0; j < 8; ++j) {
                            const int h = 64 * kb + 8 * j + 2 * m4;
                            if (DET && h < H)
                                *reinterpret_cast<float2 *>(dst + h) = make_float2(acc[kb][4 * j + 2 * hh] * inv, acc[kb][4 * j + 2 * hh + 1] * inv);
                            else if (h < H) red_add_v2(dst + h, acc[kb][4 * j + 2 * hh] * inv, acc[kb][4 * j + 2 * hh + 1] * inv);
                        }
                }
            }
        }
    }
}

bool label_backward_tc_ok(const c2v_dims *d)
{
    return d->encode >= 4 && d->encode <= 256 && (d->encode & 3) == 0;
}

// scratch: 256 B (word 0: bits of max |G|).  w_img / w_hdr: the label workspace's cached W_out image and header (valid).
int launch_label_backward_tc(const c2v_dims *d, const float *cv, const float *G, int B, const uint8_t *w_img,
                             const float *w_hdr, float *d_cv, float *d_w, float *d_b, unsigned *scratch, cudaStream_t st,
                             bool absmax_ready, const uint8_t *cv_img, float *dcv_slabs)
{
    const int H = d->encode, nkb = (H + 63) / 64;
    const long long C = d->label_count;
    const bool tf32 = matmul_tf32();           // the calling host thread's matmul precision (c2v_set_matmul_precision)
    int dev = 0, sms = 0;
    C2V_CUDA_OK(cudaGetDevice(&dev));
    C2V_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    if (!absmax_ready) {                       // (ready: c2v_label_dlogits left max |G| in the word while it wrote G)
        C2V_CUDA_OK(cudaMemsetAsync(scratch, 0, 4, st));
        lbt_absmax_kernel<<<sms * 4, 256, 0, st>>>(G, (long long)B * C, scratch);
        C2V_LAUNCH_OK("lbt_absmax_kernel");
    }
    if (d_w || d_b) {
        if (!d_w) { set_error("label backward (tensor cores): d_output_bias needs d_output_weight"); return C2V_EINVAL; }
        void (*kern)(const float *, const float *, int, long long, int, const unsigned *, float *, float *, const uint8_t *) =
            tf32 ? (nkb == 1 ? (cv_img ? label_dw_tc_kernel<true, 1, OnePass> : label_dw_tc_kernel<false, 1, OnePass>)
                  : nkb == 2 ? (cv_img ? label_dw_tc_kernel<true, 2, OnePass> : label_dw_tc_kernel<false, 2, OnePass>)
                  : nkb == 3 ? (cv_img ? label_dw_tc_kernel<true, 3, OnePass> : label_dw_tc_kernel<false, 3, OnePass>)
                             : (cv_img ? label_dw_tc_kernel<true, 4, OnePass> : label_dw_tc_kernel<false, 4, OnePass>))
                 : (nkb == 1 ? (cv_img ? label_dw_tc_kernel<true, 1> : label_dw_tc_kernel<false, 1>)
                  : nkb == 2 ? (cv_img ? label_dw_tc_kernel<true, 2> : label_dw_tc_kernel<false, 2>)
                  : nkb == 3 ? (cv_img ? label_dw_tc_kernel<true, 3> : label_dw_tc_kernel<false, 3>)
                             : (cv_img ? label_dw_tc_kernel<true, 4> : label_dw_tc_kernel<false, 4>));
        C2V_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, lb1::SMEM_BYTES));
        const long long n_ct = (C + 127) / 128;
        const int grid = (int)(n_ct < sms ? n_ct : sms);
        kern<<<grid, lbt::THREADS, lb1::SMEM_BYTES, st>>>(G, cv, B, C, H, scratch, d_w, d_b, cv_img);
        C2V_LAUNCH_OK("label_dw_tc_kernel");
    }
    if (d_cv) {
        if (!dcv_slabs) C2V_CUDA_OK(cudaMemsetAsync(d_cv, 0, (size_t)B * H * sizeof(float), st));
        const int smem = lb2_smem_bytes(nkb);
        void (*kern)(const float *, int, long long, int, const uint8_t *, const float *, const unsigned *, int, long long, float *,
                     int) =
            tf32 ? (dcv_slabs ? (nkb == 1 ? label_dcv_tc_kernel<1, true, OnePass> : nkb == 2 ? label_dcv_tc_kernel<2, true, OnePass>
                                 : nkb == 3 ? label_dcv_tc_kernel<3, true, OnePass> : label_dcv_tc_kernel<4, true, OnePass>)
                              : (nkb == 1 ? label_dcv_tc_kernel<1, false, OnePass> : nkb == 2 ? label_dcv_tc_kernel<2, false, OnePass>
                                 : nkb == 3 ? label_dcv_tc_kernel<3, false, OnePass> : label_dcv_tc_kernel<4, false, OnePass>))
                 : (dcv_slabs ? (nkb == 1 ? label_dcv_tc_kernel<1, true> : nkb == 2 ? label_dcv_tc_kernel<2, true>
                                 : nkb == 3 ? label_dcv_tc_kernel<3, true> : label_dcv_tc_kernel<4, true>)
                              : (nkb == 1 ? label_dcv_tc_kernel<1> : nkb == 2 ? label_dcv_tc_kernel<2>
                                 : nkb == 3 ? label_dcv_tc_kernel<3> : label_dcv_tc_kernel<4>));
        C2V_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        const int n_bt = (B + 127) / 128;
        const long long n_kblocks = (C + 63) / 64;
        long long n_split = (2LL * sms + n_bt - 1) / n_bt;            // ~2 items per SM
        if (n_split > n_kblocks) n_split = n_kblocks;
        if (dcv_slabs && n_split > kDetLabelSplits) n_split = kDetLabelSplits;
        if (n_split < 1) n_split = 1;
        const long long per = (n_kblocks + n_split - 1) / n_split;
        n_split = (n_kblocks + per - 1) / per;
        const long long n_items = (long long)n_bt * n_split;
        const int grid = (int)(n_items < sms ? n_items : sms);
        kern<<<grid, lbt::THREADS, smem, st>>>(G, B, C, H, w_img, w_hdr, scratch, (int)n_split, per, dcv_slabs ? dcv_slabs : d_cv,
                                               lb2_stages(nkb));
        C2V_LAUNCH_OK("label_dcv_tc_kernel");
        if (dcv_slabs)     // every split owns at least one label block: all n_split slabs are written
            return launch_det_slab_sum(dcv_slabs, (int)n_split, (size_t)B * H, (size_t)B * H, d_cv, false, st);
    }
    return C2V_OK;
}

}  // namespace c2v

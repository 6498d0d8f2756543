// c2v_label_tcgen05.cu -- K2: label logits  outputs = cv . W_out^T + b  (model.py:83) on the tensor cores (wgmma).
//
// Same fp32-accurate scheme as the encode kernel: both operands are split into fp16 hi + lo and
// three f16 MMAs (hi.hi + lo.hi + hi.lo) accumulate in fp32 registers (hi.hi alone under C2V_MATMUL_TF32).  W_out is scaled by a
// power of two (from its absmax) before the split; the epilogue multiplies by the exact inverse
// and adds the bias.  Plain TF32 fails the 1e-4 bar on trained weights.
//
// Three launches: absmax(W_out) -> split cv and W_out into K-major 128-byte-swizzled tile images
// ([128 rows x 64 k] fp16, hi then lo, per k-block) -> the persistent GEMM over 128x128 output tiles.
// Output-write bound (B*C*4 bytes).
#include <cuda_fp16.h>

#include <cstdlib>

#include <cstring>

#include "c2v_tc_ptx.cuh"

namespace c2v {

namespace lt {
constexpr int TM = 128, TN = 128, KB = 64;
constexpr int TILE_BYTES = 128 * KB * 2;          // 16 KB
}  // namespace lt

__host__ __device__ __forceinline__ uint32_t lt_sw128(int row, int k) {
    return (uint32_t)((row >> 3) * 1024 + (row & 7) * 128 + ((((k >> 3) ^ (row & 7)) & 7) << 4) + (k & 7) * 2);
}
__device__ __forceinline__ uint32_t lt_smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__global__ void absmax_kernel(const float *__restrict__ x, long long n, unsigned *__restrict__ out_bits)
{
    float m = 0.0f;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        m = fmaxf(m, fabsf(x[i]));
    m = warp_max(m);
    if ((threadIdx.x & 31) == 0) atomicMax(out_bits, __float_as_uint(m));   // non-negative floats order as uints
}

// X [R, K] fp32 row-major -> image: for each 128-row tile, for each k-block: {hi tile, lo tile}.
// scale_bits == nullptr: no scaling.  Rows >= R are zero-filled.  hdr[0] = 1/scale, hdr[1] = scale.
__global__ void split_rows_kernel(const float *__restrict__ X, long long R, int K, int nkb,
                                  const unsigned *__restrict__ scale_bits, uint8_t *__restrict__ img,
                                  float *__restrict__ hdr, unsigned long long *__restrict__ zero_u64, int n_zero)
{
    pdl_wait();                                   // (no-op unless launched as a programmatic dependent)
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n_zero; i += gridDim.x * blockDim.x) zero_u64[i] = 0ull;
    float scale = 1.0f;
    if (scale_bits) {
        const float mx = __uint_as_float(*scale_bits);
        if (mx > 0.0f && mx < 3.0e38f) {
            int e;
            frexpf(mx, &e);
            int k = 14 - e;
            k = k > 60 ? 60 : (k < -60 ? -60 : k);
            scale = ldexpf(1.0f, k);
        }
        if (blockIdx.x == 0 && threadIdx.x == 0) { hdr[0] = 1.0f / scale; hdr[1] = scale; }
    }
    const long long tiles = (R + 127) / 128;
    const long long total = tiles * 128 * (long long)(nkb * 16);          // float4 groups
    for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (long long)gridDim.x * blockDim.x) {
        const int k4 = (int)(g % (nkb * 16));
        const long long row = g / (nkb * 16);
        const int k = k4 * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row < R && k < K) v = *reinterpret_cast<const float4 *>(X + row * K + k);
        v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
        const __half2 h01 = __floats2half2_rn(v.x, v.y), h23 = __floats2half2_rn(v.z, v.w);
        const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
        const __half2 l01 = __floats2half2_rn(v.x - f01.x, v.y - f01.y), l23 = __floats2half2_rn(v.z - f23.x, v.w - f23.y);
        const long long tile = row >> 7;
        const int r = (int)(row & 127), kb = k / lt::KB, kk = k % lt::KB;
        uint8_t *base = img + (tile * nkb + kb) * (size_t)(2 * lt::TILE_BYTES);
        const uint32_t off = lt_sw128(r, kk);
        *reinterpret_cast<uint2 *>(base + off) = make_uint2(*reinterpret_cast<const unsigned *>(&h01), *reinterpret_cast<const unsigned *>(&h23));
        *reinterpret_cast<uint2 *>(base + lt::TILE_BYTES + off) = make_uint2(*reinterpret_cast<const unsigned *>(&l01), *reinterpret_cast<const unsigned *>(&l23));
    }
}

__device__ __forceinline__ void lt_mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok = 0;
    for (unsigned spins = 0; !ok; ++spins) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
#ifndef C2V_NO_WATCHDOG
        if (!ok && spins > (1u << 26)) __trap();
#endif
    }
}
// d (+)= A[64 x 16] . B[32 x 16]^T, both fp16 K-major in shared memory, fp32 accumulation (one warpgroup);
// d[4j + 2h + b] is row 16 (warp & 3) + lane/4 + 8h, column 8j + 2 (lane & 3) + b
__device__ __forceinline__ void lt_wgmma_m64n32(float (&d)[16], uint64_t adesc, uint64_t bdesc, int scale_d) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
// monotone float -> uint32 map, so that (key(value) << 32 | ~column) ordered as uint64 picks the largest value and,
// among equal values, the smallest column: torch.max(dim=1) semantics (main.py:285)
__device__ __forceinline__ uint32_t lt_orderable(float v) {
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float lt_from_orderable(uint32_t k) {
    return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// Tile order: groups of NT_GROUP consecutive n-tiles; inside a group m-tile major, n-tile minor.  A CTA's consecutive
// tiles then write adjacent 512-B pieces of the same 128 output rows within a few microseconds (L2 merges them into
// long DRAM bursts),
// and the W_out tiles of a group (NT_GROUP x 64 KB) are re-read from L2 by the n_mt m-tiles.
// Lane order (per_m > 0, what the launcher picks whenever n_mt * per_m CTAs cover >= 95 % of the SMs): CTA c owns m-tile
// c % n_mt for the whole launch and walks the n-tiles of slice c / n_mt of the label range one after the other.  The n_mt
// CTAs of a slice (adjacent CTA ids, same pace) ask for the same W_out tile within a few microseconds: one DRAM read and
// n_mt - 1 L2 hits, where the group order re-read the whole 100 MB image n_mt times at C = 195,299 (the 800 MB of streaming
// logits evict a group's tiles between a CTA's visits); and every CTA extends each of its
// 128 output rows by 512 contiguous bytes per tile.
struct LtTile { long long nt; int mt; };
struct LtRange { long long t_lo; int my_tiles; int mt; };         // lane order: t_lo = first n-tile, mt fixed; group order: mt = -1
__device__ __forceinline__ LtRange lt_range(long long n_tiles, int n_mt, long long n_nt, int per_m) {
    LtRange r;
    if (per_m > 0) {
        const int slice = (int)blockIdx.x / n_mt;
        r.mt = (int)blockIdx.x % n_mt;
        if (slice >= per_m) { r.t_lo = 0; r.my_tiles = 0; return r; }
        r.t_lo = n_nt * slice / per_m;
        r.my_tiles = (int)(n_nt * (slice + 1) / per_m - r.t_lo);
        return r;
    }
    r.mt = -1;
    r.t_lo = n_tiles * blockIdx.x / gridDim.x;
    r.my_tiles = (int)(n_tiles * (blockIdx.x + 1) / gridDim.x - r.t_lo);
    return r;
}
__device__ __forceinline__ LtTile lt_tile(long long t, int n_mt, long long n_nt, int group) {
    const long long per_group = (long long)group * n_mt;
    const long long g = t / per_group;
    const long long rem = t - g * per_group;
    long long gs = n_nt - g * group; if (gs > group) gs = group;           // the last group may be narrower
    LtTile r;
    r.mt = (int)(rem / gs);
    r.nt = g * group + (rem - (long long)r.mt * gs);
    return r;
}

// Loss fusion: what the epilogue adds when the caller wants the mean NLL without
// re-reading (or without ever writing) the [B, C] logits.
//   part != NULL : per (row, n-tile, 32-column block) the block's (max, sum exp(v - max)) -> part[(nt * 4 + cq) * Mpad + row],
//                  and the target logit v[row, label[row]] -> tgt[row]; merged by loss_partials_reduce / loss_finalize.
//   lse  != NULL : dlogits mode (backward): the value stored is (exp(v - lse[row]) - [col == label[row]]) * dscale
//                  instead of the logit (main.py:174 through log_softmax + NLLLoss, weights == 1).
// Angular head (model.py:71-80, the label_gemm_v2_kernel<true> instantiation): the GEMM gives dot = cv . W^T (no bias) and
// the epilogue's value becomes  s cos,  s phi(cos) at col == label[row],  cos = dot icv[row] iw[col]  (c2v_head.cu's
// semantics).  The loss / arg-max modes then run on those logits; dlogits mode stores G = d loss / d dot instead.
struct LtLoss {
    float2 *part; float *tgt; const long long *label; const float *lse; const float *dscale_ptr; float dscale; int Mpad;
    unsigned *gmax_bits;      // dlogits mode: bits of max |value stored| over the launch (what the label backward's fp16 split scales by)
    const float *icv, *iw;    // angular: 1 / max(|cv_b|, 1e-12) [M], 1 / max(|W_c|, 1e-12) [N]
    float cos_m, sin_m, s;    // angular: cos(margin), sin(margin), inverse_temp
    unsigned long long *topk; // top-k mode: per CTA 512 lists (column quarter x 128 rows) of topk_k keys, see lt_topk_insert
    int topk_k;
};
// Similarity modes (SIM != 0; the label modes pass it zeroed).  Its own parameter, behind all the others, so that the label
// instantiations keep their parameter layout.  LtLoss's icv / iw are then the row factors of sim_prep_kernel, so that the
// epilogue's value is the cosine itself.
struct LtSim {
    const long long *excl; int excl_n;        // [M, excl_n] columns that never enter row m's results (< 0: none) or NULL
    float thr; long long self_off;            // pairs: cos >= thr; self_off >= 0: row m is column self_off + m, keep col > it
    long long *pq, *pi; float *ps;            // pairs out: (qbase + row, column, cos) while the slot is < cap
    long long qbase;
    long long cap; unsigned long long *pcount; // pairs: every match adds 1 to *pcount (whatever cap is)
};
// Criterion options (the OPT instantiations, c2v_*_opts): class weights and label smoothing.  The last parameter, so that
// the other instantiations keep their parameter layout; they pass it zeroed.
//   part mode:    per (row, n-tile, 32-column block) (m, sum exp(v - m), q = sum_j w_j (m - v_j), W_b = sum_j w_j) -> part,
//                 the smoothing partial without cancellation (every term >= 0 for non-negative weights)
//   dlogits mode: G = (p - [col == label]) A_i + K_i (W p - w_j), A_i = sc u_i a_i, K_i = sc u_i eps / C, with the row
//                 coefficients a_i = (1 - eps) w[y_i], u_i and W of loss_finalize_opts_kernel (coef [2 B + 1]) and sc the
//                 upstream gradient (row_grad[i] for reduction none)
struct LtOpt {
    float4 *part; const float *weight; const float *coef; const float *row_grad; float eps_c; int B;
};

// Top-k mode (the label_gemm_v2_kernel<*, true> instantiations): a thread of the epilogue (one row, one column quarter of
// its CTA's m-tile) keeps the topk_k largest keys  lt_orderable(v) << 32 | ~col  it has seen, sorted descending, in its
// own slot of the workspace (too big for shared memory, which is full); only the upper word of the k-th key stays in a
// register.  Key order is value descending, then column ascending: torch.sort(descending=True, stable=True).
// Inserts key into lst[0..k) (empty slots hold 0, below every key) and returns the upper word of the new k-th key:
// slot i becomes max(old[i], min(key, old[i - 1])), so the loads do not wait for each other.
__device__ __forceinline__ uint32_t lt_topk_insert(unsigned long long *lst, int k, unsigned long long key) {
    unsigned long long prev = ~0ull, n = 0ull;
#pragma unroll
    for (int i = 0; i < C2V_TOPK_MAX; ++i) {
        if (i < k) {
            const unsigned long long o = lst[i];
            const unsigned long long c = key < prev ? key : prev;
            n = o > c ? o : c;
            if (n != o) lst[i] = n;
            prev = o;
        }
    }
    return (uint32_t)(n >> 32);
}
constexpr float LT_LOG2E = 1.4426950408889634f;
__device__ __forceinline__ float lt_ex2(float x) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

namespace lt2 {
constexpr int NT_GROUP = 8;
constexpr int N_EPI_WARPS = 16;                 // warp w: row quarter w & 3, column quarter w >> 2 (32 columns)
constexpr int LOAD_WARP = 16;
constexpr int THREADS = 17 * 32;
constexpr int OP_STAGES = 2;
constexpr int STAGE_BYTES = 4 * lt::TILE_BYTES;              // one k-block: {A_hi, A_lo | B_hi, B_lo}, 64 KB
constexpr int STG_LD = 36;                                   // padded fp32 row of a warp's [32 x 32] staging tile
constexpr int BAND_LD = 132;                                 // padded fp32 row of a row band's [32 x 128] staging tile (4 warps)
constexpr int STG_BYTES = N_EPI_WARPS * 32 * STG_LD * 4;     // 72 KB
constexpr int MAX_MT = 16;                                   // running arg-max table: 16 m-tiles x 128 rows x u64
constexpr int TAB_BYTES = MAX_MT * 128 * 8;
constexpr int SMEM_STG_OFF = OP_STAGES * STAGE_BYTES;
constexpr int SMEM_TAB_OFF = SMEM_STG_OFF + STG_BYTES;
constexpr int SMEM_BIAS_OFF = SMEM_TAB_OFF + TAB_BYTES;      // [16 warps][32] bias of the current tile
constexpr int SMEM_BAR_OFF = SMEM_BIAS_OFF + N_EPI_WARPS * 32 * 4;
constexpr int SMEM_BYTES = SMEM_BAR_OFF + 128 + 1024;
constexpr int SMEM_W_OFF = SMEM_BAR_OFF + 128;               // OPT only: [16 warps][32] class weights of the current tile
constexpr int SMEM_BYTES_OPT = SMEM_W_OFF + N_EPI_WARPS * 32 * 4 + 1024;
}  // namespace lt2

// K2 v2: persistent label GEMM with the arg-max folded in.  The 128 x 128 output tiles are numbered n-tile major /
// m-tile minor and cut into one contiguous range per CTA (all SMs busy for any B, C; a CTA's consecutive tiles share
// their W_out tile, which is therefore read from HBM once and re-read from L2).  Warp 16 streams {cv tile, W_out tile}
// k-block images through a 2-stage ring (one 32 KB cp.async.bulk each).  The 16 epilogue warps are four warpgroups;
// warpgroup cq issues the wgmma of the tile's columns 32 cq .. 32 cq + 31 (all 128 rows, two m64n32 accumulators in
// registers), turns the fragments into one row per thread through shared memory, then each warp (32 rows x 32 columns)
// does *1/scale + bias -> running arg-max (smem table, 64-bit atomicMax) -> padded smem tile -> row-contiguous stores.
// Bound: the logits write (B*C*4 bytes); the arg-max costs no extra pass over them.
// ANG: the angular-margin epilogue (see LtLoss); a template parameter so that the plain head compiles without it.
// TOPK: the running top-k epilogue (lt_topk_insert) instead of logits / arg-max / dlogits; needs lane order (per_m > 0,
// a CTA sees every column of its slice for its rows).  With ANG the logits are s cos without the margin: no label is read.
// SIM (with ANG, lane order, hdr unused): similarity search over a code-vector bank (c2v_knn_*), the value being the cosine
// itself (see LtSim).  SIM_KNN is the top-k mode with the columns of sm.excl left out; SIM_PAIRS writes every
// (row, column, cos) with cos >= sm.thr instead.
// OPT (loss / dlogits modes only, lt2::SMEM_BYTES_OPT of shared memory): the criterion options of LtOpt.
// PASS = OnePass (the logits / loss / dlogits modes under C2V_MATMUL_TF32): hi.hi only, and the load warp copies only the
// hi tile of each k-block of both images.  The top-k and similarity modes always run ThreePass (top-k is bound by its
// epilogue and is not faster in one pass; the similarity queries keep their fp32 contract).
constexpr int SIM_NONE = 0, SIM_KNN = 1, SIM_PAIRS = 2;
template <bool ANG, bool TOPK, int SIM = SIM_NONE, bool OPT = false, class PASS = ThreePass>
__global__ void __launch_bounds__(lt2::THREADS, 1)
label_gemm_v2_kernel(const uint8_t *__restrict__ imgA, const uint8_t *__restrict__ imgB,
                     const float *__restrict__ bias, const float *__restrict__ hdr, float *__restrict__ out,
                     int M, long long N, int nkb, int n_mt, long long n_nt, long long n_tiles,
                     unsigned long long *__restrict__ keys, unsigned *__restrict__ ticket,
                     long long *__restrict__ argmax, float *__restrict__ maxval, int dbg, const LtLoss ls, const int per_m,
                     const LtSim sm, const LtOpt op)
{
    static_assert(!OPT || (!TOPK && SIM == SIM_NONE), "criterion options belong to the loss / dlogits modes");
    static_assert(!one_pass<PASS> || (!TOPK && SIM == SIM_NONE), "top-k and the similarity queries run three passes");
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = lt_smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    unsigned char *smem = smem_raw + (base - raw);
    float *stage_all = reinterpret_cast<float *>(smem + lt2::SMEM_STG_OFF);
    unsigned long long *tab = reinterpret_cast<unsigned long long *>(smem + lt2::SMEM_TAB_OFF);
    const uint32_t bars = base + lt2::SMEM_BAR_OFF;
    // op_full[2] @0, op_empty[2] @16
    const uint32_t bar_ofull = bars, bar_oempty = bars + 16;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const LtRange rg = lt_range(n_tiles, n_mt, n_nt, per_m);
    const long long t_lo = rg.t_lo;
    const int my_tiles = rg.my_tiles;
    auto tile_of = [&](int i) {
        if (rg.mt >= 0) { LtTile r; r.nt = t_lo + i; r.mt = rg.mt; return r; }
        return lt_tile(t_lo + i, n_mt, n_nt, lt2::NT_GROUP);
    };
    const bool want_arg = keys != nullptr;

    if (tid == 0) {
        for (int s = 0; s < lt2::OP_STAGES; ++s) {
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_ofull + 8 * s));
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 4;" ::"r"(bar_oempty + 8 * s));   // one arrive per warpgroup
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (want_arg)
        for (int i = tid; i < lt2::MAX_MT * 128; i += lt2::THREADS) tab[i] = 0ull;
    __syncthreads();
    pdl_wait();                                   // everything above overlapped the tail of the cv-image kernel

    const int kb_bytes = 2 * lt::TILE_BYTES;                          // {hi, lo} of one k-block of one operand
    if (warp == lt2::LOAD_WARP) {
        if (lane == 0) {
            int it = 0;
            for (int i = 0; i < my_tiles; ++i) {
                const LtTile tt = tile_of(i);
                const long long nt = tt.nt; const int mt = tt.mt;
                for (int kb = 0; kb < nkb; ++kb, ++it) {
                    const int st = it & 1;
                    const uint32_t dst = base + st * lt2::STAGE_BYTES;
                    lt_mbar_wait(bar_oempty + 8 * st, ((uint32_t)(it >> 1) & 1u) ^ 1u);
                    constexpr int cp_bytes = one_pass<PASS> ? lt::TILE_BYTES : 2 * lt::TILE_BYTES;   // hi tile first
                    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_ofull + 8 * st), "r"((uint32_t)(2 * cp_bytes)) : "memory");
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                 ::"r"(dst), "l"(imgA + ((size_t)mt * nkb + kb) * kb_bytes), "r"((uint32_t)cp_bytes), "r"(bar_ofull + 8 * st) : "memory");
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                 ::"r"(dst + kb_bytes), "l"(imgB + ((size_t)nt * nkb + kb) * kb_bytes), "r"((uint32_t)cp_bytes), "r"(bar_ofull + 8 * st) : "memory");
                }
            }
        }
        __syncwarp();
    } else {
        // ---- epilogue: thread = output row x 32 columns.  Bounds and addresses are hoisted out of the
        //      per-element code (the epilogue is issue-bound otherwise).
        const int q = warp & 3, cq = warp >> 2;
        const float inv_scale = SIM != SIM_NONE ? 1.0f : hdr[0];
        const bool vec_ok = (N % 4 == 0);
        float *stg = stage_all + warp * 32 * lt2::STG_LD;
        float *sbias = reinterpret_cast<float *>(smem + lt2::SMEM_BIAS_OFF) + warp * 32;
        float gmax = 0.0f;                                    // dlogits mode: running max |d logit| of this thread
        // fragments -> one row per thread: the staging layout is the one the stores below use (the warp's padded tile, or
        // the row band), so every warpgroup writes only its own 32 columns
        const int xld = vec_ok ? lt2::STG_LD : lt2::BAND_LD, xcol = vec_ok ? cq * 128 * lt2::STG_LD : cq * 32;
        const int w4 = warp & 3, m4 = lane & 3;
        int it = 0;
        // bias of the NEXT tile's 32 columns is fetched one tile ahead (a dependent global load at the top of every tile
        // otherwise sits on each warp's critical path); the angular head fetches iw[col] the same way
        auto bias_of = [&](int i) {
            const float *colv = ANG ? ls.iw : bias;
            if (!colv || i >= my_tiles) return 0.0f;
            const LtTile t2 = tile_of(i);
            const long long c2 = t2.nt * lt::TN + cq * 32 + lane;
            return c2 < N ? __ldg(colv + c2) : 0.0f;
        };
        float bias_next = bias_of(0);
        // OPT: the class weights of the same columns, fetched the same way (1 without a weight vector, 0 past the last
        // column, so that the smoothing partials need no column test for W_b)
        float *sw = OPT ? reinterpret_cast<float *>(smem + lt2::SMEM_W_OFF) + warp * 32 : nullptr;
        auto weight_of = [&](int i) {
            if (i >= my_tiles) return 0.0f;
            const LtTile t2 = tile_of(i);
            const long long c2 = t2.nt * lt::TN + cq * 32 + lane;
            return c2 < N ? (op.weight ? __ldg(op.weight + c2) : 1.0f) : 0.0f;
        };
        float w_next = 0.0f;
        if constexpr (OPT) w_next = weight_of(0);
        unsigned long long *tk_list = nullptr;               // top-k: this thread's list and the upper word of its k-th key
        uint32_t tk_thr = 0;
        if constexpr (TOPK) {
            tk_list = ls.topk + ((size_t)blockIdx.x * 512 + cq * 128 + q * 32 + lane) * ls.topk_k;
            for (int j = 0; j < ls.topk_k; ++j) tk_list[j] = 0ull;
        }
        // similarity: this thread's excluded columns (0xFFFFFFFF: none), loaded once -- in lane order the row is fixed -- into
        // its slot of the arg-max table, which these modes do not use (in registers they would spill).  A column >= N lands
        // in the last tile's invalid columns (j >= n_cols), which never count anyway.
        static_assert(C2V_KNN_EXCLUDE_MAX == 4 && lt2::N_EPI_WARPS * 32 * 16 <= lt2::TAB_BYTES, "one uint4 per thread");
        if constexpr (SIM != SIM_NONE) {
            uint32_t ex[4] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
            const long long grow = (long long)rg.mt * lt::TM + q * 32 + lane;
            if (sm.excl && grow < M) {
#pragma unroll
                for (int u = 0; u < 4; ++u)
                    if (u < sm.excl_n) {
                        const long long x = sm.excl[grow * sm.excl_n + u];
                        ex[u] = (x >= 0 && x < N) ? (uint32_t)x : 0xFFFFFFFFu;
                    }
            }
            asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(base + lt2::SMEM_TAB_OFF + 16u * threadIdx.x),
                         "r"(ex[0]), "r"(ex[1]), "r"(ex[2]), "r"(ex[3]) : "memory");
        }
        auto excl_mask = [&](long long c0) {                 // bit j: column c0 + j is excluded for this thread's row
            uint32_t ex[4];
            asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(ex[0]), "=r"(ex[1]), "=r"(ex[2]), "=r"(ex[3])
                         : "r"(base + lt2::SMEM_TAB_OFF + 16u * threadIdx.x) : "memory");
            uint32_t m = 0;
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const uint32_t dl = ex[u] - (uint32_t)c0;
                m |= dl < 32u ? 1u << dl : 0u;
            }
            return m;
        };
        for (int i = 0; i < my_tiles; ++i) {
            const LtTile tt = tile_of(i);
            const long long nt = tt.nt; const int mt = tt.mt;
            const long long col0 = nt * lt::TN + cq * 32;              // first column of this warp's block
            const long long row0 = (long long)mt * lt::TM + q * 32;    // first row
            const int n_cols = (int)(N - col0 < 32 ? N - col0 : 32);   // valid columns / rows of the block (may be <= 0)
            const int n_rows = (int)(M - row0 < 32 ? M - row0 : 32);
            // bias of this warp's 32 columns: one element per lane -> smem -> broadcast float4 reads
            sbias[lane] = bias_next;
            if constexpr (OPT) sw[lane] = w_next;
            __syncwarp();
            bias_next = bias_of(i + 1);
            if constexpr (OPT) w_next = weight_of(i + 1);
            float icv_r = 0.0f;                                        // angular: 1 / |cv| of this thread's row (thread = row)
            if constexpr (ANG) icv_r = row0 + lane < M ? __ldg(ls.icv + row0 + lane) : 0.0f;
            float d[2][16];
            for (int kb = 0; kb < nkb; ++kb, ++it) {
                const int st = it & 1;
                lt_mbar_wait(bar_ofull + 8 * st, (uint32_t)(it >> 1) & 1u);
                const uint32_t sa = base + st * lt2::STAGE_BYTES, sb = sa + kb_bytes + cq * 32 * 128;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < lt::KB / 16; ++k) {
                    const uint64_t b_hi = wgmma_desc(sb + k * 32), b_lo = wgmma_desc(sb + lt::TILE_BYTES + k * 32);
#pragma unroll
                    for (int hh = 0; hh < 2; ++hh) {
                        const uint64_t a_hi = wgmma_desc(sa + hh * 8192 + k * 32), a_lo = wgmma_desc(sa + lt::TILE_BYTES + hh * 8192 + k * 32);
                        lt_wgmma_m64n32(d[hh], a_hi, b_hi, (kb | k) != 0);
                        if constexpr (one_pass<PASS>) continue;
                        lt_wgmma_m64n32(d[hh], a_lo, b_hi, 1);
                        lt_wgmma_m64n32(d[hh], a_hi, b_lo, 1);
                    }
                }
                wgmma_commit();
                wgmma_wait<0>();
                if ((tid & 127) == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar_oempty + 8 * st) : "memory");
            }
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int j = 0; j < 16; ++j) fence_operand(d[hh][j]);
            named_bar_sync(5 + cq, 128);          // every warp of this warpgroup is done with the previous tile's staging
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int rr = 64 * hh + 16 * w4 + (lane >> 2) + 8 * h;
                        *reinterpret_cast<float2 *>(stage_all + rr * xld + xcol + 8 * j + 2 * m4) = make_float2(d[hh][4 * j + 2 * h], d[hh][4 * j + 2 * h + 1]);
                    }
            named_bar_sync(5 + cq, 128);
            float r[32];
            {
                const float *src = stage_all + (q * 32 + lane) * xld + xcol;
#pragma unroll
                for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4 *>(r + j) = *reinterpret_cast<const float4 *>(src + j);
            }
            float v[32];
            float cos_t = 0.0f;                  // angular: cosine at this row's target column, when it lies in this block
            if constexpr (!ANG) {
#pragma unroll
                for (int j = 0; j < 32; j += 4) {                                                   // model.py:83
                    const float4 b4 = *reinterpret_cast<const float4 *>(sbias + j);
                    v[j] = fmaf(r[j], inv_scale, b4.x); v[j + 1] = fmaf(r[j + 1], inv_scale, b4.y);
                    v[j + 2] = fmaf(r[j + 2], inv_scale, b4.z); v[j + 3] = fmaf(r[j + 3], inv_scale, b4.w);
                }
            } else {                                                                                // model.py:71-80
#pragma unroll
                for (int j = 0; j < 32; j += 4) {                   // cos = dot icv iw (sbias holds iw of these columns)
                    const float4 w4 = *reinterpret_cast<const float4 *>(sbias + j);
                    v[j] = r[j] * inv_scale * icv_r * w4.x; v[j + 1] = r[j + 1] * inv_scale * icv_r * w4.y;
                    v[j + 2] = r[j + 2] * inv_scale * icv_r * w4.z; v[j + 3] = r[j + 3] * inv_scale * icv_r * w4.w;
                }
                if constexpr (SIM != SIM_NONE) {                                    // the cosine itself
                } else if constexpr (TOPK) {                                        // label-free: s cos, no margin
#pragma unroll
                    for (int j = 0; j < 32; ++j) v[j] *= ls.s;
                } else {
                    const long long grow = row0 + lane;
                    const long long tj = (grow < M ? ls.label[grow] : -1) - col0;
                    const int tji = (tj >= 0 && tj < n_cols) ? (int)tj : -1;
                    float phi = 0.0f;
                    if (__any_sync(0xffffffffu, tji >= 0)) {
                        // the PTX select chain of the loss partials below: a dynamic v[tj] would put v[] in local memory
#pragma unroll
                        for (int j = 0; j < 32; ++j)
                            asm volatile("{\n\t.reg .pred p;\n\tsetp.eq.s32 p, %2, %3;\n\tselp.f32 %0, %1, %0, p;\n\t}"
                                         : "+f"(cos_t) : "f"(v[j]), "r"(tji), "r"(j));
                        // phi(c) = c > 0 ? c cos_m - sqrt(1 - c^2) sin_m : c, for the target element only
                        phi = cos_t > 0.0f ? cos_t * ls.cos_m - sqrtf(1.0f - cos_t * cos_t) * ls.sin_m : cos_t;
                    }
#pragma unroll
                    for (int j = 0; j < 32; ++j) v[j] = (j == tji ? phi : v[j]) * ls.s;
                }
            }
            if (SIM != SIM_PAIRS && (ls.part || ls.lse)) {
                const long long grow = row0 + lane;                                     // this thread's output row
                const long long lab = (grow < M && ls.label) ? ls.label[grow] : -1;
                const long long tj = lab - col0;                                        // label's column inside this block
                if (ls.part) {
                    float m = -INFINITY, ssum = 0.0f;
#pragma unroll
                    for (int j = 0; j < 32; ++j) m = fmaxf(m, j < n_cols ? v[j] : -INFINITY);
                    const float mb = m * LT_LOG2E;
#pragma unroll
                    for (int j = 0; j < 32; ++j) ssum += j < n_cols ? lt_ex2(fmaf(v[j], LT_LOG2E, -mb)) : 0.0f;
                    if constexpr (OPT) {
                        float qs = 0.0f, wb = 0.0f;
#pragma unroll
                        for (int j = 0; j < 32; j += 4) {
                            const float4 w4 = *reinterpret_cast<const float4 *>(sw + j);
                            const float wj[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
                            for (int u = 0; u < 4; ++u) {
                                qs += j + u < n_cols ? wj[u] * (m - v[j + u]) : 0.0f;
                                wb += wj[u];
                            }
                        }
                        op.part[(size_t)(nt * 4 + cq) * ls.Mpad + grow] = make_float4(m, n_cols > 0 ? ssum : 0.0f, qs, wb);
                    } else {
                        ls.part[(size_t)(nt * 4 + cq) * ls.Mpad + grow] = make_float2(m, n_cols > 0 ? ssum : 0.0f);
                    }
                    if (__any_sync(0xffffffffu, tj >= 0 && tj < n_cols)) {
                        // select chain in PTX: written in C++ the compiler turns it into v[tj], a dynamically indexed read
                        // that puts all of v[] in local memory -- 8 x STL.128 per thread and tile in EVERY mode of this
                        // kernel (64 KB of local stores per tile and SM, as much as the logits themselves)
                        float t = 0.0f;
                        const int tji = (int)tj;
#pragma unroll
                        for (int j = 0; j < 32; ++j)
                            asm volatile("{\n\t.reg .pred p;\n\tsetp.eq.s32 p, %2, %3;\n\tselp.f32 %0, %1, %0, p;\n\t}"
                                         : "+f"(t) : "f"(v[j]), "r"(tji), "r"(j));
                        if (tj >= 0 && tj < n_cols) ls.tgt[grow] = t;
                    }
                }
                if (!TOPK && ls.lse) {                                                  // dlogits (overwrites v)
                    const float lb = (grow < M ? ls.lse[grow] : 0.0f) * LT_LOG2E;
                    const float sc = ls.dscale_ptr ? ls.dscale * *ls.dscale_ptr : ls.dscale;
                    if constexpr (OPT) {
                        // d logit = (p - [j == y]) A + K (W p - w_j); K == 0 (no smoothing) leaves the first term's bits
                        const bool in = grow < M;
                        const float up = op.row_grad ? ls.dscale * (in ? op.row_grad[grow] : 0.0f) : sc;
                        const float ur = up * (in ? op.coef[op.B + grow] : 0.0f);
                        const float A = ur * (in ? op.coef[grow] : 0.0f), K = ur * op.eps_c, Wt = op.coef[2 * op.B];
                        const float tf = ANG && cos_t > 0.0f ? ls.cos_m + ls.sin_m * cos_t / sqrtf(1.0f - cos_t * cos_t) : 1.0f;
#pragma unroll
                        for (int j = 0; j < 32; j += 4) {
                            const float4 w4 = *reinterpret_cast<const float4 *>(sw + j);
                            const float wj[4] = {w4.x, w4.y, w4.z, w4.w};
                            float4 iw4 = make_float4(0.f, 0.f, 0.f, 0.f);
                            if constexpr (ANG) iw4 = *reinterpret_cast<const float4 *>(sbias + j);
                            const float iwj[4] = {iw4.x, iw4.y, iw4.z, iw4.w};
#pragma unroll
                            for (int u = 0; u < 4; ++u) {
                                const bool t = j + u == (int)tj;
                                const float p = lt_ex2(fmaf(v[j + u], LT_LOG2E, -lb));
                                const float g = fmaf(K, fmaf(Wt, p, -wj[u]), (p - (t ? 1.0f : 0.0f)) * A);
                                if constexpr (!ANG) {
                                    v[j + u] = g;
                                } else {                          // G = d loss / d dot, as below
                                    float dcos = g * ls.s;
                                    if (t) dcos *= tf;
                                    v[j + u] = dcos * icv_r * iwj[u];
                                }
                            }
                        }
                    } else if constexpr (!ANG) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) v[j] = (lt_ex2(fmaf(v[j], LT_LOG2E, -lb)) - ((j == (int)tj) ? 1.0f : 0.0f)) * sc;
                    } else {
                        // G = d loss / d dot: dcos = s d_logit (x phi'(cos) at the target when cos > 0), G = dcos icv iw
                        const float tf = cos_t > 0.0f ? ls.cos_m + ls.sin_m * cos_t / sqrtf(1.0f - cos_t * cos_t) : 1.0f;
#pragma unroll
                        for (int j = 0; j < 32; j += 4) {
                            const float4 w4 = *reinterpret_cast<const float4 *>(sbias + j);
                            const float iwj[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
                            for (int u = 0; u < 4; ++u) {
                                const bool t = j + u == (int)tj;
                                float dcos = (lt_ex2(fmaf(v[j + u], LT_LOG2E, -lb)) - (t ? 1.0f : 0.0f)) * sc * ls.s;
                                if (t) dcos *= tf;
                                v[j + u] = dcos * icv_r * iwj[u];
                            }
                        }
                    }
                    if (ls.gmax_bits && grow < M) {
#pragma unroll
                        for (int j = 0; j < 32; ++j) gmax = fmaxf(gmax, j < n_cols ? fabsf(v[j]) : 0.0f);
                    }
                }
            }
            if constexpr (TOPK) {
                // candidates: keys above the k-th one (columns arrive in increasing order, so an equal value never
                // displaces an earlier column).  v + 0: -0 ranks as +0, as torch compares them equal.
                uint32_t cand = 0;
                if (lane < n_rows) {
#pragma unroll
                    for (int j = 0; j < 32; ++j) {
                        const uint32_t h = lt_orderable(v[j] + 0.0f);
                        v[j] = __uint_as_float(h);
                        cand |= (j < n_cols && h > tk_thr) ? (1u << j) : 0u;
                    }
                }
                if (cand) {
                    // this row's keys go back to its own staging slot (read above; the warpgroup barrier at the top of the
                    // next tile orders the reuse), so that the insert loop can index them
                    uint32_t *ks = reinterpret_cast<uint32_t *>(stage_all + (q * 32 + lane) * xld + xcol);
#pragma unroll
                    for (int j = 0; j < 32; j += 4)
                        *reinterpret_cast<uint4 *>(ks + j) = make_uint4(__float_as_uint(v[j]), __float_as_uint(v[j + 1]),
                                                                        __float_as_uint(v[j + 2]), __float_as_uint(v[j + 3]));
                    do {
                        const int j = __ffs(cand) - 1;
                        cand &= cand - 1;
                        const uint32_t h = ks[j];
                        // an excluded column never enters the list (checked here, on the rare candidates, not per element)
                        if (h > tk_thr && (SIM != SIM_KNN || !((excl_mask(col0) >> j) & 1u)))
                            tk_thr = lt_topk_insert(tk_list, ls.topk_k, ((unsigned long long)h << 32) |
                                                                            (unsigned long long)(0xFFFFFFFFu - (uint32_t)(col0 + j)));
                    } while (cand);
                }
                __syncwarp();
                continue;
            }
            if constexpr (SIM == SIM_PAIRS) {
                // the row's matches in this block; one atomic per warp reserves the slots of all 32 rows (exclusive scan of
                // the per-thread counts), and the count grows by every match even where the slots run out
                const long long grow = row0 + lane;
                uint32_t hit = 0;
                if (lane < n_rows) {
                    const long long lim = sm.self_off >= 0 ? sm.self_off + grow : -1;
#pragma unroll
                    for (int j = 0; j < 32; ++j) hit |= (j < n_cols && v[j] >= sm.thr && col0 + j > lim) ? (1u << j) : 0u;
                    hit &= ~excl_mask(col0);
                }
                const int nh = __popc(hit);
                int incl = nh;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const int t = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += t;
                }
                const int tot = __shfl_sync(0xffffffffu, incl, 31);
                if (tot) {
                    unsigned long long base = 0;
                    if (lane == 31) base = atomicAdd(sm.pcount, (unsigned long long)tot);
                    long long slot = (long long)__shfl_sync(0xffffffffu, base, 31) + (incl - nh);
                    if (hit) {
                        // the row's values go back to its own staging slot (read above), so that the loop can index them
                        float *vs = stage_all + (q * 32 + lane) * xld + xcol;
#pragma unroll
                        for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4 *>(vs + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
                        do {
                            const int j = __ffs(hit) - 1;
                            hit &= hit - 1;
                            if (slot < sm.cap) { sm.pq[slot] = sm.qbase + grow; sm.pi[slot] = col0 + j; sm.ps[slot] = vs[j]; }
                            ++slot;
                        } while (hit);
                    }
                }
                __syncwarp();
                continue;
            }
            if (want_arg && lane < n_rows && n_cols > 0 && !C2V_EXPT(dbg, 2)) {
                float m = -INFINITY;
                if (n_cols == 32) {
#pragma unroll
                    for (int j = 0; j < 32; ++j) m = fmaxf(m, v[j]);
                } else {
#pragma unroll
                    for (int j = 0; j < 32; ++j) m = fmaxf(m, j < n_cols ? v[j] : -INFINITY);
                }
                unsigned long long *slot = tab + mt * 128 + q * 32 + lane;
                const uint32_t mk = lt_orderable(m);
                if (mk >= (uint32_t)(*reinterpret_cast<volatile unsigned long long *>(slot) >> 32)) {
                    int jm = 31;
#pragma unroll
                    for (int j = 31; j >= 0; --j) jm = (v[j] == m && j < n_cols) ? j : jm;        // first maximum
                    atomicMax(slot, ((unsigned long long)mk << 32) | (unsigned long long)(0xFFFFFFFFu - (uint32_t)(col0 + jm)));
                }
            }
            if (out == nullptr) { __syncwarp(); continue; }   // loss-only mode: the logits are never written
            if (!vec_ok && !C2V_EXPT(dbg, 7)) {
                // Rows that are only 4-byte aligned (label_count % 4 != 0, e.g. top11's 195,299): the four column-quarter
                // warps of a row band stage the whole [32 rows x 128 columns] band, then every warp writes 8 rows of it in
                // segments that start on 128-byte boundaries of GLOBAL memory (5 store instructions per row instead of 4;
                // only the tile's two edge sectors per row stay partial).  Per-warp 128-B pieces at the row's own misalignment
                // would write every sector in two halves.
                float *band = stage_all + q * (32 * lt2::BAND_LD);
#pragma unroll
                for (int j = 0; j < 32; j += 4)
                    *reinterpret_cast<float4 *>(band + lane * lt2::BAND_LD + cq * 32 + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
                asm volatile("bar.sync %0, 128;" ::"r"(1 + q) : "memory");
                const long long base_col = nt * lt::TN;
                const int tile_cols = (int)(N - base_col < lt::TN ? N - base_col : lt::TN);
                if (!C2V_EXPT(dbg, 1)) {
#pragma unroll 1
                    for (int rr = cq * 8; rr < cq * 8 + 8; ++rr) {
                        const long long grow = (long long)mt * lt::TM + q * 32 + rr;
                        if (grow >= M) break;
                        float *grow_p = out + (size_t)grow * N + base_col;
                        const int a = (int)(((size_t)grow * N + base_col) & 31);        // floats past a 128-byte boundary
                        const float *sp = band + rr * lt2::BAND_LD;
#pragma unroll
                        for (int sg = 0; sg < 5; ++sg) {
                            const int col = sg * 32 - a + lane;
                            if (col >= 0 && col < tile_cols) grow_p[col] = sp[col];
                        }
                    }
                }
                asm volatile("bar.sync %0, 128;" ::"r"(1 + q) : "memory");     // the band is restaged by the next tile
                continue;
            }
            // registers -> padded smem tile (thread = row), then row-contiguous stores
#pragma unroll
            for (int j = 0; j < 32; j += 4)
                *reinterpret_cast<float4 *>(stg + lane * lt2::STG_LD + j) = make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
            __syncwarp();
            if (C2V_EXPT(dbg, 4)) {          // timing experiment: same bytes, but every warp block as one contiguous 4 KB run
                float *gp = out + ((size_t)(t_lo + i) * 16 + warp) * 1024 + lane * 4;
#pragma unroll
                for (int it = 0; it < 8; ++it)
                    *reinterpret_cast<float4 *>(gp + it * 128) = *reinterpret_cast<const float4 *>(stg + (it * 4 + (lane >> 3)) * lt2::STG_LD + (lane & 7) * 4);
            } else if (n_rows > 0 && n_cols > 0 && !C2V_EXPT(dbg, 1)) {
                if (vec_ok && n_cols == 32) {
                    const int rr0 = lane >> 3, c4 = (lane & 7) * 4;          // 4 rows x 128 B per store instruction
                    float *gp = out + (size_t)(row0 + rr0) * N + col0 + c4;
                    const float *sp = stg + rr0 * lt2::STG_LD + c4;
                    const size_t gstep = (size_t)4 * N;
#pragma unroll
                    for (int it = 0; it < 8; ++it) {
                        if (it * 4 + rr0 < n_rows) *reinterpret_cast<float4 *>(gp) = *reinterpret_cast<const float4 *>(sp + it * 4 * lt2::STG_LD);
                        gp += gstep;
                    }
                } else if (lane < n_cols) {                                  // one <= 128-B row segment per store instruction
                    float *gp = out + (size_t)row0 * N + col0 + lane;
                    const float *sp = stg + lane;
#pragma unroll
                    for (int rr = 0; rr < 32; ++rr) {
                        if (rr < n_rows) *gp = sp[rr * lt2::STG_LD];
                        gp += N;
                    }
                }
            }
            __syncwarp();                         // staging tile is rewritten by the next tile
        }
        if (ls.lse && ls.gmax_bits) {                 // one atomic per warp and launch (non-negative floats order as uints)
            gmax = warp_max(gmax);
            if (lane == 0 && gmax > 0.0f && gmax < 3.0e38f) atomicMax(ls.gmax_bits, __float_as_uint(gmax));
        }
    }
    __syncthreads();
    if (want_arg) {
        // flush this CTA's table, then the last CTA to arrive decodes keys -> (argmax, maxval)
        __shared__ unsigned s_last;
        for (int i = tid; i < n_mt * 128; i += lt2::THREADS) {
            const unsigned long long k = tab[i];
            if (k != 0ull && i < M) atomicMax(keys + i, k);
        }
        __threadfence();
        __syncthreads();
        if (tid == 0) s_last = atomicAdd(ticket, 1u) == gridDim.x - 1 ? 1u : 0u;
        __syncthreads();
        if (s_last) {
            __threadfence();
            for (int b = tid; b < M; b += lt2::THREADS) {
                const unsigned long long k = *reinterpret_cast<volatile unsigned long long *>(keys + b);
                if (argmax) argmax[b] = (long long)(0xFFFFFFFFu - (uint32_t)(k & 0xFFFFFFFFull));
                if (maxval) maxval[b] = lt_from_orderable((uint32_t)(k >> 32));
            }
        }
    }
}

// ---- merging the loss partials: (max, sum exp) pairs are merged online-softmax style ----------------------------------
__device__ __forceinline__ void lt_merge(float &M, float &S, float m, float sv) {
    if (m > M) { S = S * __expf(M - m) + sv; M = m; }          // (M = -inf, S = 0 start: exp(-inf) = 0)
    else if (m > -INFINITY) S += sv * __expf(m - M);
}
constexpr int LT_PSPLIT = 16;
// grid (Mpad / 32, LT_PSPLIT), 256 threads: lane = row, the 8 warps stride over this CTA's share of the partial index
__global__ void __launch_bounds__(256)
loss_partials_reduce_kernel(const float2 *__restrict__ part, int P, int Mpad, float2 *__restrict__ part2)
{
    __shared__ float2 sh[8][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int row = blockIdx.x * 32 + lane;
    const int p0 = (int)((long long)P * blockIdx.y / gridDim.y), p1 = (int)((long long)P * (blockIdx.y + 1) / gridDim.y);
    float M = -INFINITY, S = 0.0f;
    for (int p = p0 + warp; p < p1; p += 8) {
        const float2 v = part[(size_t)p * Mpad + row];
        lt_merge(M, S, v.x, v.y);
    }
    sh[warp][lane] = make_float2(M, S);
    __syncthreads();
    if (warp == 0) {
        for (int w = 1; w < 8; ++w) lt_merge(M, S, sh[w][lane].x, sh[w][lane].y);      // fixed order: deterministic
        part2[(size_t)blockIdx.y * Mpad + row] = make_float2(M, S);
    }
}
// one CTA: lse[b] = M + log S, loss = mean_b (lse[b] - target logit[b])   (main.py:251-264 with weights == 1)
__global__ void __launch_bounds__(1024)
loss_finalize_kernel(const float2 *__restrict__ part2, int nsplit, int Mpad, const float *__restrict__ tgt, int B,
                     float *__restrict__ lse, float *__restrict__ loss)
{
    __shared__ float red[32];
    float acc = 0.0f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        float M = -INFINITY, S = 0.0f;
        for (int k = 0; k < nsplit; ++k) { const float2 v = part2[(size_t)k * Mpad + b]; lt_merge(M, S, v.x, v.y); }
        const float l = M + logf(S);
        if (lse) lse[b] = l;
        acc += l - tgt[b];
    }
    acc = warp_sum(acc);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x < 32) {
        float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.0f;
        v = warp_sum(v);
        if (threadIdx.x == 0 && loss) *loss = v / (float)B;
    }
}

// ---- the same with the criterion options: (max, sum exp, q, W_b) partials (see LtOpt) --------------------------------
// A merge to the larger max M adds W_b (M - m_b) to the q of the side whose max was smaller: every term stays >= 0.
// (S, M) are merged with lt_merge's exact operations, so that lse is the same number as without options.
__device__ __forceinline__ void lt_merge4(float4 &a, const float4 b) {
    if (b.x > a.x) {
        const float q = a.x > -INFINITY ? fmaf(a.w, b.x - a.x, a.z) : a.z;   // (no column merged yet: W = 0, q = 0)
        a.y = a.y * __expf(a.x - b.x) + b.y; a.x = b.x;
        a.z = q + b.z; a.w += b.w;
    } else if (b.x > -INFINITY) {
        a.y += b.y * __expf(b.x - a.x);
        a.z += fmaf(b.w, a.x - b.x, b.z); a.w += b.w;
    }
}
__global__ void __launch_bounds__(256)
loss_partials_reduce_opts_kernel(const float4 *__restrict__ part, int P, int Mpad, float4 *__restrict__ part2)
{
    __shared__ float4 sh[8][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int row = blockIdx.x * 32 + lane;
    const int p0 = (int)((long long)P * blockIdx.y / gridDim.y), p1 = (int)((long long)P * (blockIdx.y + 1) / gridDim.y);
    float4 acc = make_float4(-INFINITY, 0.0f, 0.0f, 0.0f);
    for (int p = p0 + warp; p < p1; p += 8) lt_merge4(acc, part[(size_t)p * Mpad + row]);
    sh[warp][lane] = acc;
    __syncthreads();
    if (warp == 0) {
        for (int w = 1; w < 8; ++w) lt_merge4(acc, sh[w][lane]);                        // fixed order: deterministic
        part2[(size_t)blockIdx.y * Mpad + row] = acc;
    }
}
// one CTA, the reductions in loss_finalize_kernel's fixed order.  Per row i (y = label[i], w_y = weight[y] or 1; an
// ignored row, label == ignore_index, has w_y = 0 and row term 0):
//   lse_i = M + log S,  smooth_i = sum_j w_j (lse_i - z_ij) = q + W log S
//   row_i = (1 - eps) w_y (lse_i - z_iy) + (eps / C) smooth_i,   den = sum_i w_y
// loss: mean sum_i row_i / den, sum sum_i row_i, none row_i [B].  coef [2 B + 1] for the dlogits mode:
// a_i = (1 - eps) w_y, u_i = 0 if ignored else (1 / den for mean, 1 otherwise), then W.
// A label outside [0, C) that is not ignore_index has no target logit (tgt stays NaN): its row is NaN, as without
// options, and it adds nothing to den.
__global__ void __launch_bounds__(1024)
loss_finalize_opts_kernel(const float4 *__restrict__ part2, int nsplit, int Mpad, const float *__restrict__ tgt,
                          const long long *__restrict__ label, int B, long long C, const float *__restrict__ weight,
                          long long ignore_index, float eps, float eps_c, int reduction, float *__restrict__ lse,
                          float *__restrict__ loss, float *__restrict__ coef)
{
    __shared__ float red[32], red_den[32], s_den;
    float acc = 0.0f, dacc = 0.0f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        float4 a = make_float4(-INFINITY, 0.0f, 0.0f, 0.0f);
        for (int k = 0; k < nsplit; ++k) lt_merge4(a, part2[(size_t)k * Mpad + b]);
        const float ls = logf(a.y), l = a.x + ls;
        if (lse) lse[b] = l;
        const long long y = label[b];
        const bool ign = y == ignore_index, valid = y >= 0 && y < C;
        const float wy = (ign || !valid) ? 0.0f : (weight ? weight[y] : 1.0f);
        const float ab = (1.0f - eps) * wy;
        const float row = ign ? 0.0f : fmaf(eps_c, fmaf(a.w, ls, a.z), ab * (l - tgt[b]));
        if (reduction == C2V_REDUCTION_NONE && loss) loss[b] = row;
        acc += row;
        dacc += wy;
        if (coef) {
            coef[b] = ab;
            if (b == 0) coef[2 * B] = a.w;
        }
    }
    acc = warp_sum(acc);
    dacc = warp_sum(dacc);
    if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = acc; red_den[threadIdx.x >> 5] = dacc; }
    __syncthreads();
    if (threadIdx.x < 32) {
        const bool on = threadIdx.x < (blockDim.x >> 5);
        const float v = warp_sum(on ? red[threadIdx.x] : 0.0f), den = warp_sum(on ? red_den[threadIdx.x] : 0.0f);
        if (threadIdx.x == 0) {
            s_den = den;
            if (loss && reduction == C2V_REDUCTION_MEAN) *loss = v / den;       // every row ignored: 0 / 0 = NaN, as torch
            else if (loss && reduction == C2V_REDUCTION_SUM) *loss = v;
        }
    }
    if (!coef) return;
    __syncthreads();
    const float u = reduction == C2V_REDUCTION_MEAN ? 1.0f / s_den : 1.0f;
    for (int b = threadIdx.x; b < B; b += blockDim.x) coef[B + b] = label[b] == ignore_index ? 0.0f : u;
}

// ---- top-k: merging the per-thread lists of label_gemm_v2_kernel<*, true> --------------------------------------------
constexpr int LT_TOPK_MAX_CTAS = 256;               // grid cap of the top-k GEMM: bounds its workspace independently of the device
// one warp per row b: the row's 4 per_m sorted lists (list l = 4 slice + column quarter, written by CTA slice * n_mt + mt)
// are merged k-way -- every lane holds the best head of its lists l = lane, lane + 32, ...; k rounds of a warp maximum.
// part2 != NULL: lse from the row's (max, sum exp) partials and prob = exp(v - lse).
__global__ void __launch_bounds__(256)
topk_merge_kernel(const unsigned long long *__restrict__ lists, int k, int M, int n_mt, int per_m,
                  const float2 *__restrict__ part2, int Mpad, long long *__restrict__ idx, float *__restrict__ val,
                  float *__restrict__ prob)
{
    __shared__ unsigned char heads[8][4 * LT_TOPK_MAX_CTAS];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int b = blockIdx.x * 8 + w;
    if (b >= M) return;
    const int L = 4 * per_m, mt = b >> 7, r = b & 127;
    unsigned char *hd = heads[w];
    for (int l = lane; l < L; l += 32) hd[l] = 0;
    unsigned long long best = 0ull;
    int bl = -1;
    auto rescan = [&]() {
        best = 0ull; bl = -1;
        for (int l = lane; l < L; l += 32) {
            const int h = hd[l];
            const unsigned long long key = h < k ? lists[((size_t)((l >> 2) * n_mt + mt) * 512 + (l & 3) * 128 + r) * k + h] : 0ull;
            if (key > best) { best = key; bl = l; }
        }
    };
    rescan();
    float lse = 0.0f;
    if (prob) {
        float Mx = -INFINITY, S = 0.0f;
        if (lane < LT_PSPLIT) { const float2 pr = part2[(size_t)lane * Mpad + b]; Mx = pr.x; S = pr.y; }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float m2 = __shfl_xor_sync(0xffffffffu, Mx, o), s2 = __shfl_xor_sync(0xffffffffu, S, o);
            lt_merge(Mx, S, m2, s2);
        }
        lse = __shfl_sync(0xffffffffu, Mx + logf(S), 0);
    }
    for (int i = 0; i < k; ++i) {
        unsigned long long top = best;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long t = __shfl_xor_sync(0xffffffffu, top, o);
            top = t > top ? t : top;
        }
        if (lane == 0) {
            const float v = lt_from_orderable((uint32_t)(top >> 32));
            const size_t o = (size_t)b * k + i;
            idx[o] = (long long)(0xFFFFFFFFu - (uint32_t)(top & 0xFFFFFFFFull));
            val[o] = v;
            if (prob) prob[o] = expf(v - lse);
        }
        if (bl >= 0 && best == top) { hd[bl] += 1; rescan(); }          // keys are unique (one column each): one winner
        __syncwarp();
    }
}

// K (= encode_size) is zero-padded to a multiple of 64 inside the operand images
bool label_tcgen05_shape_ok(const c2v_dims *d) { return d->encode >= 4 && d->encode <= 256 && (d->encode & 3) == 0; }

// ticket (first 64 bytes) + arg-max keys [B] u64.  This region sits AFTER the W_out image: the image is reused across calls
// while the weights are unchanged (C2V_FLAG_REUSE_PREP), so its offset must not depend on the batch size (a ragged last
// batch of an evaluation pass has a different B).
static size_t lt_keys_bytes(int B) { return (64 + (size_t)B * 8 + 1023) / 1024 * 1024; }

// loss partials (behind the cv image): part [nt * 4][Mpad] float2 | part2 [LT_PSPLIT][Mpad] float2 | tgt [Mpad] float
static size_t lt_loss_bytes(int B, long long C)
{
    const size_t Mpad = (size_t)(B + 127) / 128 * 128, nt = (size_t)((C + 127) / 128);
    return (nt * 4 + LT_PSPLIT) * Mpad * sizeof(float2) + Mpad * sizeof(float) + 1024;
}
// criterion options (c2v_*_opts): part4 [nt * 4][Mpad] float4 | part4_2 [LT_PSPLIT][Mpad] float4, in a region of its own
// so that the label workspace keeps its layout
size_t label_loss_opts_bytes(const c2v_dims *d, int B)
{
    const size_t Mpad = (size_t)(B + 127) / 128 * 128, nt = (size_t)((d->label_count + 127) / 128);
    return (nt * 4 + LT_PSPLIT) * Mpad * sizeof(float4) + 1024;
}
size_t label_tcgen05_workspace_bytes(const c2v_dims *d, int B)
{
    const size_t nkb = (size_t)(d->encode + 63) / 64;
    const size_t mt = (size_t)(B + 127) / 128, nt = (size_t)(d->label_count + 127) / 128;
    return 1024 + lt_keys_bytes(B) + (mt + nt) * nkb * 2 * lt::TILE_BYTES + lt_loss_bytes(B, d->label_count);
}

// top-k region, behind the label workspace (whose layout it leaves alone): the GEMM's lists, 512 x k keys per CTA |
// inv_norms [B + C] of the angular head
static size_t lt_topk_lists_bytes(const c2v_dims *d, int B, int k)
{
    const long long n_tiles = (long long)((B + 127) / 128) * ((d->label_count + 127) / 128);
    const long long ctas = n_tiles < LT_TOPK_MAX_CTAS ? n_tiles : LT_TOPK_MAX_CTAS;
    return align_up((size_t)ctas * 512 * (size_t)k * 8, 1024);
}
size_t label_topk_workspace_bytes(const c2v_dims *d, int B, int k)
{
    return align_up(label_tcgen05_workspace_bytes(d, B), 1024) + lt_topk_lists_bytes(d, B, k) +
           align_up((size_t)(B + d->label_count) * sizeof(float), 1024);
}
float *label_topk_inv_norms(const c2v_dims *d, int B, int k, void *ws)
{
    return reinterpret_cast<float *>(static_cast<uint8_t *>(ws) + align_up(label_tcgen05_workspace_bytes(d, B), 1024) +
                                     lt_topk_lists_bytes(d, B, k));
}

int launch_loss_argmax(const float *out, const long long *label, int B, long long C, float *loss,
                       long long *argmax, float *maxval, float *d_out, cudaStream_t st);

// argmax / maxval (torch.max(dim=1), main.py:285) are folded into the GEMM epilogue (label_gemm_v2_kernel) for up to
// 16 m-tiles (B <= 2048); beyond that they are a second pass over the logits.
int launch_label_tcgen05_ex(const c2v_dims *d, const float *cv, int B, const float *Wout, const float *bias,
                            float *out, long long *argmax, float *maxval, void *ws, size_t ws_bytes, bool reuse_prep,
                            cudaStream_t st, const LabelLossArgs *la);

// The cached W_out image of a label workspace (built here unless reuse_prep): what the tensor-core label backward streams.
int label_w_image(const c2v_dims *d, const float *Wout, int B, void *ws, size_t ws_bytes, bool reuse_prep, cudaStream_t st,
                  const uint8_t **img, const float **hdr, unsigned **scratch, const uint8_t **cv_img)
{
    if (!label_tcgen05_shape_ok(d) || !ws || ws_bytes < label_tcgen05_workspace_bytes(d, B)) {
        set_error("label backward: workspace missing or too small");
        return C2V_EWORKSPACE;
    }
    const int H = d->encode, nkb = (H + 63) / 64;
    const long long C = d->label_count;
    uint8_t *p = static_cast<uint8_t *>(ws);
    float *h = reinterpret_cast<float *>(p);
    unsigned *mxbits = reinterpret_cast<unsigned *>(p + 256);
    uint8_t *imgB = p + 1024;
    if (!reuse_prep) {
        int dev = 0, sms = 0;
        C2V_CUDA_OK(cudaGetDevice(&dev));
        C2V_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        C2V_CUDA_OK(cudaMemsetAsync(mxbits, 0, 4, st));
        absmax_kernel<<<sms * 4, 256, 0, st>>>(Wout, C * H, mxbits);
        C2V_LAUNCH_OK("absmax_kernel");
        split_rows_kernel<<<sms * 8, 256, 0, st>>>(Wout, C, H, nkb, mxbits, imgB, h, nullptr, 0);
        C2V_LAUNCH_OK("split_rows_kernel");
    }
    *img = imgB; *hdr = h; *scratch = reinterpret_cast<unsigned *>(p + 768);
    // where launch_label_tcgen05_ex keeps the fp16 image of the code vectors of its last call with this B (same layout math)
    if (cv_img) *cv_img = imgB + (size_t)((C + 127) / 128) * nkb * 2 * lt::TILE_BYTES + lt_keys_bytes(B);
    return C2V_OK;
}

// What the last label GEMM launched from this host thread left in its workspace: the fp16 image of `cv` (every call) and, in
// dlogits mode, max |d logit|.  c2v_label_backward_ws only believes C2V_FLAG_GRAD_ABSMAX_READY when this record matches its
// own workspace / code_vector / B -- a wrong flag then costs the skipped shortcuts, not the result.
static thread_local struct { const void *ws; const float *cv; int B; bool dlogits; } g_label_last = {nullptr, nullptr, 0, false};
bool label_ws_holds_dlogits_of(const void *ws, const float *cv, int B)
{
    return g_label_last.dlogits && g_label_last.ws == ws && g_label_last.cv == cv && g_label_last.B == B;
}

// la != NULL: la->loss (mean NLL) / la->lse [B] are produced from the fused partials (out may then be NULL: the logits
// are never written); la->dlogits_lse != NULL: `out` receives d(loss)/d(logits) instead of the logits.
int launch_label_tcgen05_ex(const c2v_dims *d, const float *cv, int B, const float *Wout, const float *bias,
                            float *out, long long *argmax, float *maxval, void *ws, size_t ws_bytes, bool reuse_prep,
                            cudaStream_t st, const LabelLossArgs *la)
{
    if (!label_tcgen05_shape_ok(d)) {
        set_error("tcgen05 label GEMM needs encode_size %% 4 == 0 and <= 256 (got %d)", d->encode);
        return C2V_EUNSUPPORTED;
    }
    const int H = d->encode, nkb = (H + 63) / 64;
    const long long C = d->label_count;
    const bool topk = la && la->topk_k > 0;
    const size_t ws_need = topk ? label_topk_workspace_bytes(d, B, la->topk_k) : label_tcgen05_workspace_bytes(d, B);
    if (!ws || ws_bytes < ws_need) {
        set_error("label workspace too small: %zu < %zu", ws_bytes, ws_need);
        return C2V_EWORKSPACE;
    }
    g_label_last.ws = ws; g_label_last.cv = cv; g_label_last.B = B; g_label_last.dlogits = la && la->dlogits_lse;
    uint8_t *p = static_cast<uint8_t *>(ws);
    float *hdr = reinterpret_cast<float *>(p);
    unsigned *mxbits = reinterpret_cast<unsigned *>(p + 256);

    const size_t mt = (size_t)(B + 127) / 128, nt = (size_t)((C + 127) / 128);
    // W_out image first (reusable across calls while the weights are unchanged), then the cv image
    uint8_t *imgB = p + 1024;                                           // batch-size independent offset
    uint8_t *key_region = imgB + nt * nkb * 2 * lt::TILE_BYTES;
    unsigned *ticket = reinterpret_cast<unsigned *>(key_region);
    unsigned long long *keys = reinterpret_cast<unsigned long long *>(key_region + 64);
    uint8_t *imgA = key_region + lt_keys_bytes(B);
    const int Mpad = (int)mt * 128;
    float2 *part = reinterpret_cast<float2 *>(imgA + mt * nkb * 2 * lt::TILE_BYTES);
    float2 *part2 = part + nt * 4 * (size_t)Mpad;
    float *tgt = reinterpret_cast<float *>(part2 + (size_t)LT_PSPLIT * Mpad);
    LtLoss ls;
    memset(&ls, 0, sizeof(ls));
    ls.Mpad = Mpad;
    const bool want_loss = la && (la->loss || la->lse_out);
    if (want_loss) {
        if (!la->label) { set_error("label loss: label is NULL"); return C2V_EINVAL; }
        ls.part = part; ls.tgt = tgt; ls.label = la->label;
        // a label outside [0, C) leaves its target logit unwritten: NaN then makes the loss NaN (the reference's NLLLoss
        // raises "Target out of bounds")
        C2V_CUDA_OK(cudaMemsetAsync(tgt, 0xFF, (size_t)Mpad * sizeof(float), st));
    }
    if (la && la->dlogits_lse) {
        if (!la->label || !out) { set_error("label dlogits: label / output is NULL"); return C2V_EINVAL; }
        ls.lse = la->dlogits_lse; ls.label = la->label; ls.dscale = la->dscale; ls.dscale_ptr = la->dscale_ptr;
        // max |d logit| for the label backward (c2v_label_backward_ws with C2V_FLAG_GRAD_ABSMAX_READY skips its own pass
        // over the [B, C] gradient); same word label_w_image hands to the backward as `scratch`
        ls.gmax_bits = reinterpret_cast<unsigned *>(p + 768);
        C2V_CUDA_OK(cudaMemsetAsync(ls.gmax_bits, 0, 4, st));
    }
    const bool angular = la && la->inv_norms;
    if (angular) {
        if (!la->label && !topk) { set_error("angular label head: label is NULL"); return C2V_EINVAL; }
        ls.label = topk ? nullptr : la->label;
        ls.icv = la->inv_norms; ls.iw = la->inv_norms + B;
        ls.cos_m = la->cos_m; ls.sin_m = la->sin_m; ls.s = la->inverse_temp;
        bias = nullptr;                                                 // the angular head has none
    }
    if (topk) {
        if (!la->topk_idx || !la->topk_val || out || argmax || maxval || want_loss || la->dlogits_lse) {
            set_error("label top-k: indices / values missing, or combined with another output");
            return C2V_EINVAL;
        }
        ls.topk = reinterpret_cast<unsigned long long *>(p + align_up(label_tcgen05_workspace_bytes(d, B), 1024));
        ls.topk_k = la->topk_k;
        if (la->topk_prob) ls.part = part;                              // (max, sum exp) partials, no label / target
    }
    const LossOptArgs *opt = la ? la->opts : nullptr;
    LtOpt op;
    memset(&op, 0, sizeof(op));
    float4 *part4 = nullptr, *part4_2 = nullptr;
    if (opt) {
        if (topk || !opt->coef || (want_loss && !opt->part)) {
            set_error("label loss options: top-k mode, or coefficients / partials missing");
            return C2V_EINVAL;
        }
        op.weight = opt->weight; op.coef = opt->coef; op.row_grad = opt->row_grad; op.B = B;
        op.eps_c = (float)((double)opt->eps / (double)C);
        if (want_loss) {
            part4 = static_cast<float4 *>(opt->part);
            part4_2 = part4 + nt * 4 * (size_t)Mpad;
            op.part = part4;
            ls.part = reinterpret_cast<float2 *>(part4);          // (selects the loss mode; the OPT epilogue writes op.part)
        }
    }
    // the matmul precision of the calling host thread picks the instantiation (c2v_set_matmul_precision); top-k always
    // runs three passes
    auto *kern = topk ? (angular ? label_gemm_v2_kernel<true, true> : label_gemm_v2_kernel<false, true>)
               : matmul_tf32()
        ? (opt ? (angular ? label_gemm_v2_kernel<true, false, SIM_NONE, true, OnePass> : label_gemm_v2_kernel<false, false, SIM_NONE, true, OnePass>)
               : (angular ? label_gemm_v2_kernel<true, false, SIM_NONE, false, OnePass> : label_gemm_v2_kernel<false, false, SIM_NONE, false, OnePass>))
        : (opt ? (angular ? label_gemm_v2_kernel<true, false, SIM_NONE, true> : label_gemm_v2_kernel<false, false, SIM_NONE, true>)
               : (angular ? label_gemm_v2_kernel<true, false> : label_gemm_v2_kernel<false, false>));
    const int smem_bytes = opt ? lt2::SMEM_BYTES_OPT : lt2::SMEM_BYTES;
    const bool want_arg = argmax || maxval;
    const bool fused_arg = want_arg && mt <= (size_t)lt2::MAX_MT;
    int dev = 0, sms = 0;
    C2V_CUDA_OK(cudaGetDevice(&dev));
    C2V_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));

    if (!reuse_prep) {
        C2V_CUDA_OK(cudaMemsetAsync(mxbits, 0, 4, st));
        absmax_kernel<<<sms * 4, 256, 0, st>>>(Wout, C * H, mxbits);
        C2V_LAUNCH_OK("absmax_kernel");
        split_rows_kernel<<<sms * 8, 256, 0, st>>>(Wout, C, H, nkb, mxbits, imgB, hdr, nullptr, 0);
        C2V_LAUNCH_OK("split_rows_kernel");
    }
    // cv image (+ zeroes the ticket and the arg-max keys, which sit contiguously in key_region)
    C2V_CUDA_OK(launch_pdl(split_rows_kernel, dim3((unsigned)((mt * 128 * nkb * 16 + 255) / 256)), dim3(256), 0, st, cv,
                           (long long)B, H, nkb, (const unsigned *)nullptr, imgA, hdr,
                           reinterpret_cast<unsigned long long *>(key_region), fused_arg ? 8 + B : 0));
    C2V_COUNT_LAUNCH();

    C2V_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
    const long long n_tiles = (long long)mt * (long long)nt;
    int grid = (int)(n_tiles < sms ? n_tiles : sms);
    // tile order (see lt_range): lanes when that keeps >= 95 % of the CTAs busy, else groups; C2V_LABEL_ORDER=groups|lanes forces one
    int per_m = (mt <= (size_t)grid) ? grid / (int)mt : 0;
    if (per_m > 0 && (long long)per_m * (long long)mt * 100 < 95ll * grid) per_m = 0;
    if (const char *ord = getenv("C2V_LABEL_ORDER")) {
        if (!strcmp(ord, "groups")) per_m = 0;
        else if (!strcmp(ord, "lanes") && mt <= (size_t)grid) per_m = grid / (int)mt;
    }
    if (topk) {                                   // always lane order: each list then sees every column of its slice
        if (grid > LT_TOPK_MAX_CTAS) grid = LT_TOPK_MAX_CTAS;
        per_m = grid / (int)mt;
        if (per_m < 1) { set_error("label top-k: %d SMs for %zu m-tiles", sms, mt); return C2V_EUNSUPPORTED; }
    }
    C2V_CUDA_OK(launch_pdl(kern, dim3((unsigned)grid), dim3(lt2::THREADS), (size_t)smem_bytes, st,
                           (const uint8_t *)imgA, (const uint8_t *)imgB, bias, (const float *)hdr, out, B, C, nkb, (int)mt,
                           (long long)nt, n_tiles, fused_arg ? keys : (unsigned long long *)nullptr, ticket,
                           fused_arg ? argmax : (long long *)nullptr, fused_arg ? maxval : (float *)nullptr,
                           getenv("C2V_K2_FLAGS") ? atoi(getenv("C2V_K2_FLAGS")) : 0, ls, per_m, LtSim{}, op));
    C2V_LAUNCH_OK("label_gemm_v2_kernel");
    if (want_loss && opt) {
        loss_partials_reduce_opts_kernel<<<dim3((unsigned)(Mpad / 32), LT_PSPLIT), 256, 0, st>>>(part4, (int)(nt * 4), Mpad,
                                                                                               part4_2);
        C2V_LAUNCH_OK("loss_partials_reduce_opts_kernel");
        loss_finalize_opts_kernel<<<1, 1024, 0, st>>>(part4_2, LT_PSPLIT, Mpad, tgt, la->label, B, C, opt->weight,
                                                      opt->ignore_index, opt->eps, op.eps_c, opt->reduction, la->lse_out,
                                                      la->loss, opt->coef);
        C2V_LAUNCH_OK("loss_finalize_opts_kernel");
    } else if (want_loss) {
        loss_partials_reduce_kernel<<<dim3((unsigned)(Mpad / 32), LT_PSPLIT), 256, 0, st>>>(part, (int)(nt * 4), Mpad, part2);
        C2V_LAUNCH_OK("loss_partials_reduce_kernel");
        loss_finalize_kernel<<<1, 1024, 0, st>>>(part2, LT_PSPLIT, Mpad, tgt, B, la->lse_out, la->loss);
        C2V_LAUNCH_OK("loss_finalize_kernel");
    }
    if (topk) {
        if (la->topk_prob) {
            loss_partials_reduce_kernel<<<dim3((unsigned)(Mpad / 32), LT_PSPLIT), 256, 0, st>>>(part, (int)(nt * 4), Mpad, part2);
            C2V_LAUNCH_OK("loss_partials_reduce_kernel");
        }
        topk_merge_kernel<<<(unsigned)((B + 7) / 8), 256, 0, st>>>(ls.topk, la->topk_k, B, (int)mt, per_m,
                                                                  la->topk_prob ? part2 : nullptr, Mpad, la->topk_idx,
                                                                  la->topk_val, la->topk_prob);
        C2V_LAUNCH_OK("topk_merge_kernel");
    }
    if (want_arg && !fused_arg) {
        if (!out) { set_error("label loss without logits: arg-max needs B <= %d", lt2::MAX_MT * 128); return C2V_EUNSUPPORTED; }
        return launch_loss_argmax(out, nullptr, B, C, nullptr, argmax, maxval, nullptr, st);
    }
    return C2V_OK;
}

// ---- similarity search over a code-vector bank (c2v_knn_*) -----------------------------------------------------------
// Rows -> the GEMM operand image (split_rows_kernel's layout), each row scaled by its own power of two 2^k so that its
// largest element lands in [2^13, 2^14) (fp16's range is used in full whatever the row's magnitude), and
// fac[r] = 1 / max(|x_r 2^k|, 1e-12 2^k) = 2^-k / max(|x_r|, 1e-12).  Then cos(q, b) = (q 2^kq . b 2^kb) fac_q fac_b, with
// F.normalize's clamp; a zero row has fac = 1e12 and a zero dot product, so similarity 0.  One warp per row of the
// 128-row padded range (rows >= R are zero).  H % 4 == 0 and H <= 256: two float4 groups per lane.
__global__ void __launch_bounds__(256)
sim_prep_kernel(const float *__restrict__ X, long long R, int H, int nkb, uint8_t *__restrict__ img, float *__restrict__ fac)
{
    const int lane = threadIdx.x & 31;
    const long long rows = (R + 127) / 128 * 128;
    const long long wstride = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += wstride) {
        float4 v[2];
        float m = 0.0f;
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int k = (lane + 32 * u) * 4;
            v[u] = (row < R && k < H) ? *reinterpret_cast<const float4 *>(X + row * H + k) : make_float4(0.f, 0.f, 0.f, 0.f);
            m = fmaxf(m, fmaxf(fmaxf(fabsf(v[u].x), fabsf(v[u].y)), fmaxf(fabsf(v[u].z), fabsf(v[u].w))));
        }
        m = warp_max(m);
        int e = 14;                                            // zero or non-finite rows: scale 1
        if (m > 0.0f && m <= 3.4e38f) frexpf(m, &e);
        const int ks = 14 - e > 126 ? 126 : (14 - e < -126 ? -126 : 14 - e);
        const float sc = ldexpf(1.0f, ks);
        float ss = 0.0f;
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            v[u].x *= sc; v[u].y *= sc; v[u].z *= sc; v[u].w *= sc;
            ss += v[u].x * v[u].x + v[u].y * v[u].y + v[u].z * v[u].z + v[u].w * v[u].w;
        }
        ss = warp_sum(ss);
        if (lane == 0 && row < R) fac[row] = 1.0f / fmaxf(sqrtf(ss), 1e-12f * sc);
        const long long tile = row >> 7;
        const int r = (int)(row & 127);
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int k = (lane + 32 * u) * 4;
            if (k >= nkb * lt::KB) continue;
            const __half2 h01 = __floats2half2_rn(v[u].x, v[u].y), h23 = __floats2half2_rn(v[u].z, v[u].w);
            const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
            const __half2 l01 = __floats2half2_rn(v[u].x - f01.x, v[u].y - f01.y);
            const __half2 l23 = __floats2half2_rn(v[u].z - f23.x, v[u].w - f23.y);
            uint8_t *base = img + (tile * nkb + k / lt::KB) * (size_t)(2 * lt::TILE_BYTES);
            const uint32_t off = lt_sw128(r, k % lt::KB);
            *reinterpret_cast<uint2 *>(base + off) = make_uint2(*reinterpret_cast<const unsigned *>(&h01), *reinterpret_cast<const unsigned *>(&h23));
            *reinterpret_cast<uint2 *>(base + lt::TILE_BYTES + off) = make_uint2(*reinterpret_cast<const unsigned *>(&l01), *reinterpret_cast<const unsigned *>(&l23));
        }
    }
}

// prep workspace (the bank's image, then fac [N]): depends on N and H only, so one prep serves every query chunk
size_t knn_prep_bytes(long long N, int H)
{
    const size_t nkb = (size_t)(H + 63) / 64, nt = (size_t)((N + 127) / 128);
    return nt * nkb * 2 * lt::TILE_BYTES + align_up((size_t)N * sizeof(float), 1024);
}
// call workspace: the query image, fac [Q], then (top-k) 512 lists of k keys per CTA of the GEMM
size_t knn_query_bytes(long long N, int H, int Q, int k)
{
    const size_t nkb = (size_t)(H + 63) / 64, mt = (size_t)(Q + 127) / 128;
    const long long n_tiles = (long long)mt * ((N + 127) / 128);
    const size_t ctas = (size_t)(n_tiles < LT_TOPK_MAX_CTAS ? n_tiles : LT_TOPK_MAX_CTAS);
    return mt * nkb * 2 * lt::TILE_BYTES + align_up((size_t)Q * sizeof(float), 1024) + align_up(ctas * 512 * (size_t)k * 8, 1024);
}

static int launch_sim_prep(const float *X, long long R, int H, uint8_t *img, float *fac, int sms, cudaStream_t st)
{
    const long long blocks = ((R + 127) / 128 * 128 + 7) / 8;             // 8 warps (rows) per block
    sim_prep_kernel<<<(unsigned)(blocks < sms * 32ll ? blocks : sms * 32ll), 256, 0, st>>>(X, R, H, (H + 63) / 64, img, fac);
    C2V_LAUNCH_OK("sim_prep_kernel");
    return C2V_OK;
}

static int knn_sms(int *sms)
{
    int dev = 0;
    C2V_CUDA_OK(cudaGetDevice(&dev));
    C2V_CUDA_OK(cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev));
    return C2V_OK;
}

int launch_knn_prepare(const float *bank, long long N, int H, void *prep, cudaStream_t st)
{
    int sms = 0;
    const int rc = knn_sms(&sms);
    if (rc != C2V_OK) return rc;
    uint8_t *img = static_cast<uint8_t *>(prep);
    const size_t nt = (size_t)((N + 127) / 128), nkb = (size_t)(H + 63) / 64;
    return launch_sim_prep(bank, N, H, img, reinterpret_cast<float *>(img + nt * nkb * 2 * lt::TILE_BYTES), sms, st);
}

// The arguments were checked by the caller (c2v_knn_topk / c2v_knn_pairs): Q <= 2048, H % 4 == 0, H <= 256, N < 2^32 - 1,
// workspaces of knn_prep_bytes / knn_query_bytes.
int launch_knn(const KnnArgs &a, cudaStream_t st)
{
    int sms = 0;
    int rc = knn_sms(&sms);
    if (rc != C2V_OK) return rc;
    const int H = a.H, nkb = (H + 63) / 64;
    const long long N = a.N;
    const size_t mt = (size_t)(a.Q + 127) / 128, nt = (size_t)((N + 127) / 128);
    uint8_t *imgB = static_cast<uint8_t *>(a.prep);
    const float *fb = reinterpret_cast<const float *>(imgB + nt * nkb * 2 * lt::TILE_BYTES);
    uint8_t *imgA = static_cast<uint8_t *>(a.ws);
    float *fq = reinterpret_cast<float *>(imgA + mt * nkb * 2 * lt::TILE_BYTES);
    unsigned long long *lists = reinterpret_cast<unsigned long long *>(reinterpret_cast<uint8_t *>(fq) +
                                                                       align_up((size_t)a.Q * sizeof(float), 1024));
    if (!a.reuse_prep && (rc = launch_knn_prepare(a.bank, N, H, a.prep, st)) != C2V_OK) return rc;
    if ((rc = launch_sim_prep(a.queries, a.Q, H, imgA, fq, sms, st)) != C2V_OK) return rc;

    LtLoss ls;
    memset(&ls, 0, sizeof(ls));
    ls.icv = fq; ls.iw = fb;
    LtSim sm = {};
    sm.excl = a.exclude; sm.excl_n = a.exclude ? a.X : 0;
    const bool topk = a.k > 0;
    if (topk) {
        ls.topk = lists; ls.topk_k = a.k;
    } else {
        sm.thr = a.threshold; sm.self_off = a.self_offset; sm.cap = a.capacity; sm.qbase = a.query_base;
        sm.pq = a.pair_query; sm.pi = a.pair_index; sm.ps = a.pair_sim;
        sm.pcount = reinterpret_cast<unsigned long long *>(a.count);
    }
    auto *kern = topk ? label_gemm_v2_kernel<true, true, SIM_KNN> : label_gemm_v2_kernel<true, false, SIM_PAIRS>;
    C2V_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, lt2::SMEM_BYTES));
    const long long n_tiles = (long long)mt * (long long)nt;
    int grid = (int)(n_tiles < sms ? n_tiles : sms);
    if (grid > LT_TOPK_MAX_CTAS) grid = LT_TOPK_MAX_CTAS;
    const int per_m = grid / (int)mt;                       // lane order: a CTA keeps one m-tile, so its rows are fixed
    if (per_m < 1) { set_error("similarity search: %d SMs for %zu m-tiles", sms, mt); return C2V_EUNSUPPORTED; }
    C2V_CUDA_OK(launch_pdl(kern, dim3((unsigned)grid), dim3(lt2::THREADS), (size_t)lt2::SMEM_BYTES, st, (const uint8_t *)imgA,
                           (const uint8_t *)imgB, (const float *)nullptr, (const float *)nullptr, (float *)nullptr, a.Q, N, nkb,
                           (int)mt, (long long)nt, n_tiles, (unsigned long long *)nullptr, (unsigned *)nullptr,
                           (long long *)nullptr, (float *)nullptr, 0, ls, per_m, sm, LtOpt{}));
    C2V_LAUNCH_OK("label_gemm_v2_kernel");
    if (topk) {
        topk_merge_kernel<<<(unsigned)((a.Q + 7) / 8), 256, 0, st>>>(lists, a.k, a.Q, (int)mt, per_m, nullptr, 0,
                                                                     a.indices, a.sims, nullptr);
        C2V_LAUNCH_OK("topk_merge_kernel");
    }
    return C2V_OK;
}

}  // namespace c2v

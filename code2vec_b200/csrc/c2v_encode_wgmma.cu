// c2v_encode_wgmma.cu -- K1h: the fused gather + encode + attention kernel on the Hopper tensor cores (sm_90a, wgmma).
//
// What it replaces: model.py:48-69 + get_attention (model.py:90-96) of the reference.
//
// Numerics.  The reference contraction x = c . W^T is fp32; plain TF32/BF16 miss the 1e-4 parity bar.
// Both operands are split into fp16 hi + fp16 lo (a = a_hi + a_lo exactly to ~2^-22) and three f16 MMAs with fp32
// accumulation are issued per k-step:  a_hi.w_hi + a_lo.w_hi + a_hi.w_lo  (the dropped a_lo.w_lo term is 2^-22
// relative).  Under C2V_MATMUL_TF32 the OnePass instantiations issue a_hi.w_hi alone (TF32-class).  W is pre-multiplied
// by a power of two so its lo part stays out of the fp16 subnormals; the epilogue folds the exact inverse into the
// LayerNorm scale.
//
// Shapes: terminal_embed == path_embed = E, E % 4 == 0; (E <= 128 and encode_size in {100, 128}) or (E <= 256 and
// encode_size == 256).  Every sub-vector is padded to EP = 128 (256) k and the encode size to HP = 128 (256) n.
//
// Structure (one persistent CTA per SM, 20 warps, warp-specialised, tiles of 128 context rows):
//   warps 0-7   two consumer warpgroups: warpgroup g issues the wgmma of tile rows 64g .. 64g+63 (accumulator
//               [64 x HP] fp32 in registers) and runs the epilogue straight from the accumulator fragments:
//               LayerNorm, tanh, dropout, score, per-16-row online-softmax partials of the weighted sum
//   warps 8-15  A producers: 128-bit gathers of the fp32 embedding rows, hi/lo fp16 split in registers,
//               st.shared into the K-major 128-byte-swizzled operand layout
//   warp 16     W producer: one cp.async.bulk per k-block of the pre-split, pre-swizzled weight image
//   warps 17-19 idle (register donors)
// A ring of mbarrier-guarded stages carries {A_hi, A_lo, W_hi, W_lo} k-blocks.
#include <cstdlib>

#include "c2v_tc_ptx.cuh"

namespace c2v {

template <bool WIDE>
struct WgCfg {
    static constexpr int ROWS = 128;                          // context rows per tile (two warpgroups x 64)
    static constexpr int EP = WIDE ? 256 : 128;               // padded sub-vector width (k per start / path / end)
    static constexpr int HP = WIDE ? 256 : 128;               // padded encode size = MMA N
    static constexpr int KB = 64, NQ = EP / KB, NKB = 3 * NQ; // k-blocks per sub-vector / per tile
    static constexpr int STAGES = WIDE ? 2 : 3;
    static constexpr int A_TILE = ROWS * KB * 2;              // one [128 x 64] fp16 tile: 16 KB
    static constexpr int W_TILE = HP * KB * 2;                // one [HP x 64] fp16 tile: 16 / 32 KB
    static constexpr int W_KB_BYTES = 2 * W_TILE;             // {hi, lo} of one k-block of W, contiguous in HBM
    static constexpr int STAGE_BYTES = 2 * A_TILE + W_KB_BYTES;
    static constexpr int N_PROD_WARPS = 8, PROD_WARP0 = 8, MISC_WARP0 = 16;
    static constexpr int THREADS = (MISC_WARP0 + 4) * 32;     // 640
    static constexpr int ROWS_PER_PW = ROWS / N_PROD_WARPS;   // 16 rows of every tile per producer warp
    static constexpr int LDG_PER_ITEM = ROWS_PER_PW / 2;      // 8 x LDG.128 (two 256-byte half rows each)
    static constexpr int NACC = HP / 2;                       // accumulator registers per consumer thread
    static constexpr int VROWS = 16;                          // rows per softmax partial (one consumer warp)
    static constexpr int SMEM_VEC_OFF = STAGES * STAGE_BYTES;
    static constexpr int SMEM_BAR_OFF = SMEM_VEC_OFF + 3 * HP * 4;
    static constexpr int SMEM_BYTES = SMEM_BAR_OFF + 64 + 1024;   // + alignment pad
    static_assert(SMEM_BYTES <= 232448, "shared memory budget (227 KB per block)");
};
constexpr float kTwoLog2e = 2.8853900817779268f;

bool tcgen05_shape_ok(const c2v_dims *d)
{
    const int E = d->terminal_embed, H = d->encode;
    if (d->path_embed != E || E < 4 || (E & 3)) return false;
    const bool narrow = E <= 128 && (H == 100 || H == 128), wide = E <= 256 && H == 256;
    if (!narrow && !wide) return false;
    const long long row_bytes = (long long)E * 4;
    return d->terminal_count * row_bytes < (1ll << 32) && d->path_count * row_bytes < (1ll << 32);
}

// ------------------------------------------------------------------------------------
// weight preparation: W [H, 3E] fp32 -> 3*NQ k-block images {hi tile, lo tile} of [HP n x 64 k] fp16 in the exact
// shared-memory layout (K-major, 128-byte swizzle), scaled by 2^k; EP = HP = 128 (NQ = 2) or 256 (NQ = 4).  Sub-vector
// sv (start / path / end) owns k-blocks NQ*sv .. NQ*sv + NQ-1; k >= E and n >= H are zero padding.
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
split_w_kernel(const float *__restrict__ W, uint8_t *__restrict__ img, float *__restrict__ hdr, int E, int H, int EP, int HP)
{
    // Several CTAs (the image is rebuilt every training step).  Every CTA finds max |W| over the whole matrix itself
    // (<= 768 KB, L2 hits after the first CTA): no second launch, no atomics, no pre-zeroed word.  Then one item = 4
    // consecutive k of one row n of the PADDED [HP][3 EP] matrix (zeros beyond E / H), i.e. 8 contiguous bytes of the
    // hi tile and of the lo tile: every byte of the image is written once.
    __shared__ float red[32];
    const int tid = threadIdx.x;
    const int D = 3 * E, NQ = EP / 64;
    const int tile_bytes = HP * 64 * 2, kb_bytes = 2 * tile_bytes;
    const bool vec = (reinterpret_cast<uintptr_t>(W) & 15) == 0;       // E % 4 == 0 on this path: rows are 16-B multiples
    float mx = 0.0f;
    if (vec) {
        const float4 *W4 = reinterpret_cast<const float4 *>(W);
        for (int i = tid; i < H * D / 4; i += 1024) {
            const float4 v = W4[i];
            mx = fmaxf(mx, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
        }
    } else {
        for (int i = tid; i < H * D; i += 1024) mx = fmaxf(mx, fabsf(W[i]));
    }
    mx = warp_max(mx);
    if ((tid & 31) == 0) red[tid >> 5] = mx;
    __syncthreads();
    mx = red[0];
    for (int i = 1; i < 32; ++i) mx = fmaxf(mx, red[i]);
    // largest power of two with max|W| * scale < 2^14 (fp16 max is 65504)
    float scale = 1.0f;
    if (mx > 0.0f && mx < 3.0e38f) {
        int e;
        frexpf(mx, &e);                       // mx = f * 2^e, f in [0.5, 1)
        int k = 14 - e;
        k = k > 60 ? 60 : (k < -60 ? -60 : k);
        scale = ldexpf(1.0f, k);
    }
    if (blockIdx.x == 0 && tid == 0) { hdr[0] = 1.0f / scale; hdr[1] = scale; }
    const int per_row = 3 * EP / 4;
    for (int g = blockIdx.x * 1024 + tid; g < HP * per_row; g += gridDim.x * 1024) {
        const int n = g / per_row, kp = (g % per_row) * 4;
        const int sv = kp / EP, e = kp % EP;
        float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
        if (n < H && e < E) {
            const float *src = W + (size_t)n * D + sv * E + e;
            w = vec ? *reinterpret_cast<const float4 *>(src) : make_float4(src[0], src[1], src[2], src[3]);
        }
        w.x *= scale; w.y *= scale; w.z *= scale; w.w *= scale;
        const __half2 h01 = __floats2half2_rn(w.x, w.y), h23 = __floats2half2_rn(w.z, w.w);
        const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
        const __half2 l01 = __floats2half2_rn(w.x - f01.x, w.y - f01.y), l23 = __floats2half2_rn(w.z - f23.x, w.w - f23.y);
        const int kb = NQ * sv + e / 64, kk = e % 64;
        uint8_t *dst = img + (size_t)kb * kb_bytes + sw128_offset(n, kk);
        *reinterpret_cast<uint2 *>(dst) = make_uint2(pack_h2(h01), pack_h2(h23));
        *reinterpret_cast<uint2 *>(dst + tile_bytes) = make_uint2(pack_h2(l01), pack_h2(l23));
    }
}

int launch_split_w_tcgen05(const c2v_dims *d, const float *W, EncodeWorkspace &ws, cudaStream_t st)
{
    const int P = (d->encode > 128 || d->terminal_embed > 128) ? 256 : 128;
    split_w_kernel<<<P == 256 ? 24 : 12, 1024, 0, st>>>(W, reinterpret_cast<uint8_t *>(ws.w_hi), ws.prep_hdr, d->terminal_embed, d->encode, P, P);
    C2V_LAUNCH_OK("split_w_kernel");
    return C2V_OK;
}

// ------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------
// PASS: ThreePass (fp32-accurate) or OnePass (C2V_MATMUL_TF32: a_hi.w_hi only; the A producers store no lo tile and the
// W producer copies only the hi tile of each k-block of the image)
template <bool DROPOUT, int HV, bool PACKED = false, bool SEED_DEV = false, class PASS = ThreePass>
__global__ void __launch_bounds__(WgCfg<(HV > 128)>::THREADS, 1)
encode_wgmma_kernel(const EncodeArgs a)
{
    constexpr bool WIDE = HV > 128;
    using C = WgCfg<WIDE>;
    extern __shared__ unsigned char smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;                  // 128-byte-swizzled tiles need 1024-B alignment
    unsigned char *smem = smem_raw + (base - raw);
    float *s_vec = reinterpret_cast<float *>(smem + C::SMEM_VEC_OFF);      // gamma' | beta' | attn
    const uint32_t bar_full = base + C::SMEM_BAR_OFF, bar_empty = bar_full + 8 * C::STAGES;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int my_tiles = (a.n_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
    const int n_items = my_tiles * C::NKB;
    long long *status = a.ws.status;

    if (tid == 0) {
        for (int s = 0; s < C::STAGES; ++s) {
            mbar_init(bar_full + 8 * s, C::N_PROD_WARPS + 1);      // 8 producer warps + the W copy's arrive
            mbar_init(bar_empty + 8 * s, 2);                        // one arrive per consumer warpgroup
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    pdl_wait();              // barrier init above overlaps the previous kernel's tail
    // LayerNorm affine pre-multiplied by 2*log2(e) so tanh needs no extra multiply; columns >= a.H get 0
    for (int i = tid; i < 3 * C::HP; i += C::THREADS) {
        const int which = i / C::HP, c = i % C::HP;
        float v = 0.0f;
        if (c < a.H) v = which == 0 ? a.ln_g[c] * kTwoLog2e : which == 1 ? a.ln_b[c] * kTwoLog2e : a.attn[c];
        s_vec[i] = v;
    }
    __syncthreads();

    if (warp < C::PROD_WARP0) {
        // =============================== CONSUMERS (MMA + epilogue) ===============================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 160;");
        const int g = warp >> 2, w4 = warp & 3;
        const int m4 = lane & 3;
        const float inv_scale = a.ws.prep_hdr[0];
        constexpr float inv_h = 1.0f / (float)HV;
        float acc[C::NACC];
        int it = 0;
        for (int tl = 0; tl < my_tiles; ++tl) {
            const int tile = (int)blockIdx.x + tl * (int)gridDim.x;
#pragma unroll 1
            for (int kb = 0; kb < C::NKB; ++kb, ++it) {
                const int stage = it % C::STAGES;
                mbar_wait(bar_full + 8 * stage, (uint32_t)(it / C::STAGES) & 1u, status);
                const uint32_t sa = base + stage * C::STAGE_BYTES + g * (C::A_TILE / 2);   // this warpgroup's 64 rows
                const uint32_t sw = base + stage * C::STAGE_BYTES + 2 * C::A_TILE;
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < C::KB / 16; ++k) {
                    const uint64_t a_hi = wgmma_desc(sa + k * 32), a_lo = wgmma_desc(sa + C::A_TILE + k * 32);
                    const uint64_t w_hi = wgmma_desc(sw + k * 32), w_lo = wgmma_desc(sw + C::W_TILE + k * 32);
                    const int first = (kb | k) == 0;
                    wgmma_m64n128<0>(acc, a_hi, w_hi, !first);
                    if (WIDE) wgmma_m64n128<64 % C::NACC>(acc, a_hi, w_hi + (16384 >> 4), !first);
                    if constexpr (one_pass<PASS>) continue;
                    wgmma_m64n128<0>(acc, a_lo, w_hi, 1);
                    if (WIDE) wgmma_m64n128<64 % C::NACC>(acc, a_lo, w_hi + (16384 >> 4), 1);
                    wgmma_m64n128<0>(acc, a_hi, w_lo, 1);
                    if (WIDE) wgmma_m64n128<64 % C::NACC>(acc, a_hi, w_lo + (16384 >> 4), 1);
                }
                wgmma_commit();
                // keep one k-block of MMAs in flight; the one before it has retired and its stage can be refilled
                wgmma_wait<1>();
                if (kb > 0 && (tid & 127) == 0) mbar_arrive(bar_empty + 8 * ((it - 1) % C::STAGES));
            }
            wgmma_wait<0>();
#pragma unroll
            for (int i = 0; i < C::NACC; ++i) fence_operand(acc[i]);
            if ((tid & 127) == 0) mbar_arrive(bar_empty + 8 * ((it - 1) % C::STAGES));

            // ---- epilogue.  Fragment layout of the m64 accumulator: acc[4j + 2h + b] is row 16 w4 + lane/4 + 8h of
            //      this warpgroup's 64 rows, column 8j + 2 (lane & 3) + b.  A row's columns live in one lane quad.
            long long row[2], bag_r[2] = {0, 0};
            bool in_range[2];
            float nrm[2], shift[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                row[h] = (long long)tile * C::ROWS + 64 * g + 16 * w4 + (lane >> 2) + 8 * h;
                in_range[h] = row[h] < a.N;
                if (PACKED) bag_r[h] = in_range[h] ? bag_of_row<true>(a, row[h]) : 0;     // rows past N: any valid bag, unused
                // LayerNorm (model.py:55-56) in two passes over the accumulator registers, as the CUDA-core encode and
                // the backward compute it: the one-pass E[x^2] - mean^2 loses ~2^-24 mean^2 / var relative, which misses
                // the 1e-4 bar once |mean| / std reaches a few tens.  Padding columns (c >= HV) are exactly 0 and stay
                // out of the sum of squares.
                float s = 0.f, q = 0.f;
#pragma unroll
                for (int j = 0; j < C::HP / 8; ++j) s += acc[4 * j + 2 * h] + acc[4 * j + 2 * h + 1];
                s += __shfl_xor_sync(0xffffffffu, s, 1); s += __shfl_xor_sync(0xffffffffu, s, 2);
                const float mean = s * inv_h;
#pragma unroll
                for (int j = 0; j < C::HP / 8; ++j) {
                    const bool col = 8 * j + 2 * m4 < HV;
                    const float d0 = col ? acc[4 * j + 2 * h] - mean : 0.f, d1 = col ? acc[4 * j + 2 * h + 1] - mean : 0.f;
                    q = fmaf(d0, d0, fmaf(d1, d1, q));
                }
                q += __shfl_xor_sync(0xffffffffu, q, 1); q += __shfl_xor_sync(0xffffffffu, q, 2);
                const float var = q * inv_h * inv_scale * inv_scale;
                nrm[h] = inv_scale / sqrtf(var + C2V_LN_EPS);
                shift[h] = -mean * nrm[h];
            }
            if (a.stash_x) {       // training forward: keep x = c . W^T for the backward (no recompute)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!in_range[h]) continue;
                    float *dst = a.stash_x + (size_t)row[h] * a.H;
#pragma unroll
                    for (int j = 0; j < C::HP / 8; ++j) {
                        const int c = 8 * j + 2 * m4;
                        if (c < HV)
                            *reinterpret_cast<float2 *>(dst + c) = make_float2(acc[4 * j + 2 * h] * inv_scale, acc[4 * j + 2 * h + 1] * inv_scale);
                    }
                }
            }
            // tanh (model.py:57), dropout (model.py:60-61), score h.a (model.py:92-93); h overwrites the accumulator
            float u[2] = {0.f, 0.f};
#pragma unroll
            for (int j = 0; j < C::HP / 8; ++j) {
                const int c = 8 * j + 2 * m4;
                const float2 gm = *reinterpret_cast<const float2 *>(s_vec + c);
                const float2 bt = *reinterpret_cast<const float2 *>(s_vec + C::HP + c);
                const float2 at = *reinterpret_cast<const float2 *>(s_vec + 2 * C::HP + c);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    float y0 = tanh_from_scaled(fmaf(fmaf(acc[4 * j + 2 * h], nrm[h], shift[h]), gm.x, bt.x));
                    float y1 = tanh_from_scaled(fmaf(fmaf(acc[4 * j + 2 * h + 1], nrm[h], shift[h]), gm.y, bt.y));
                    if (DROPOUT) {
                        const uint4 bits = dropout_bits(dropout_key<SEED_DEV>(a), PACKED ? dropout_row<true>(a, row[h], bag_r[h]) : row[h], c >> 2);
                        y0 *= dropout_mul((m4 & 1) ? bits.z : bits.x, a.drop_p, a.drop_scale);
                        y1 *= dropout_mul((m4 & 1) ? bits.w : bits.y, a.drop_p, a.drop_scale);
                    }
                    acc[4 * j + 2 * h] = y0; acc[4 * j + 2 * h + 1] = y1;
                    u[h] = fmaf(y0, at.x, fmaf(y1, at.y, u[h]));
                }
            }
            float z[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                u[h] += __shfl_xor_sync(0xffffffffu, u[h], 1);
                u[h] += __shfl_xor_sync(0xffffffffu, u[h], 2);
                const long long st_idx = in_range[h] ? a.starts[row[h]] : 0;    // model.py:64 mask = starts > 0
                z[h] = (in_range[h] && st_idx > 0) ? u[h] : C2V_NINF;           // model.py:93
                if (m4 == 0 && in_range[h]) a.attention[row[h]] = z[h];
            }

            // per-(warp, bag) online-softmax partial -> slot (vtile + bag)
            const long long vrow0 = (long long)tile * C::ROWS + 64 * g + 16 * w4;
            if (vrow0 < a.N) {
                const long long vt = vrow0 / C::VROWS;
                long long last = vrow0 + C::VROWS - 1; if (last > a.N - 1) last = a.N - 1;
                // packed: up to 16 bags per slice (one per row); every bag in [bag_lo, bag_hi] has a row here (lengths >= 1)
                const long long bag_lo = bag_of_row<PACKED>(a, vrow0), bag_hi = bag_of_row<PACKED>(a, last);
                for (long long bag = bag_lo; bag <= bag_hi; ++bag) {
                    const bool seg0 = in_range[0] && (PACKED ? bag_r[0] : row[0] / a.L) == bag;
                    const bool seg1 = in_range[1] && (PACKED ? bag_r[1] : row[1] / a.L) == bag;
                    const float m = warp_max(fmaxf(seg0 ? z[0] : -INFINITY, seg1 ? z[1] : -INFINITY));
                    const float e0 = seg0 ? __expf(z[0] - m) : 0.0f, e1 = seg1 ? __expf(z[1] - m) : 0.0f;
                    const size_t slot = (size_t)(vt + bag);
                    float *pv = a.ws.part_v + slot * a.H;
                    // a row of another bag is selected out, not multiplied by 0: its h may be NaN (an inf / NaN
                    // embedding entry), and 0 * NaN would spread into this bag's code vector
#pragma unroll
                    for (int j = 0; j < C::HP / 8; ++j) {
                        float v0 = fmaf(e0, seg0 ? acc[4 * j] : 0.0f, seg1 ? e1 * acc[4 * j + 2] : 0.0f);
                        float v1 = fmaf(e0, seg0 ? acc[4 * j + 1] : 0.0f, seg1 ? e1 * acc[4 * j + 3] : 0.0f);
#pragma unroll
                        for (int o = 4; o < 32; o <<= 1) {
                            v0 += __shfl_xor_sync(0xffffffffu, v0, o);
                            v1 += __shfl_xor_sync(0xffffffffu, v1, o);
                        }
                        const int c = 8 * j + 2 * m4;
                        if (lane < 4 && c < HV) *reinterpret_cast<float2 *>(pv + c) = make_float2(v0, v1);
                    }
                    const float ssum = warp_sum(m4 == 0 ? e0 + e1 : 0.0f);
                    if (lane == 0) { a.ws.part_m[slot] = m; a.ws.part_s[slot] = ssum; }
                }
            }
        }
    } else if (warp < C::MISC_WARP0) {
        // =============================== A PRODUCERS ===============================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 56;");
        const int pw = warp - C::PROD_WARP0;         // rows 16*pw .. 16*pw+15 of every tile
        const int sub_row = lane >> 4;               // which of the 2 rows of a load this lane serves
        const int q = lane & 15;                     // 16-byte column of the 256-byte half row
        const float4 *tab_t = reinterpret_cast<const float4 *>(a.emb_t);
        const float4 *tab_p = reinterpret_cast<const float4 *>(a.emb_p);
        const uint32_t row_f4 = (uint32_t)(a.Et / 4);
        uint32_t off_s = 0, off_p = 0, off_e = 0;    // row offsets (float4 units) of this lane's row of the tile
        int it = 0;
        for (int tl = 0; tl < my_tiles; ++tl) {
            {
                long long s = 0, p = 0, e = 0;
                const long long r = ((long long)blockIdx.x + (long long)tl * gridDim.x) * C::ROWS + pw * C::ROWS_PER_PW + q;
                if (r < a.N) { s = a.starts[r]; p = a.paths[r]; e = a.ends[r]; }
                int bad = 0;
                if (s < 0 || s >= a.T) { s = 0; ++bad; }
                if (p < 0 || p >= a.P) { p = 0; ++bad; }
                if (e < 0 || e >= a.T) { e = 0; ++bad; }
                if (bad && sub_row == 0) atomicAdd((unsigned long long *)status, (unsigned long long)bad);
                off_s = (uint32_t)s * row_f4; off_p = (uint32_t)p * row_f4; off_e = (uint32_t)e * row_f4;
            }
#pragma unroll 1
            for (int kb = 0; kb < C::NKB; ++kb, ++it) {
                const int sv = kb / C::NQ;                                  // 0 start, 1 path, 2 end (model.py:51)
                const float4 *tab = sv == 1 ? tab_p : tab_t;
                const uint32_t off = sv == 0 ? off_s : (sv == 1 ? off_p : off_e);
                const uint32_t col = (uint32_t)((kb % C::NQ) * 16 + q);      // float4 column of the embedding row
                const bool valid = col < row_f4;                             // k >= E: zero padding
                float4 buf[C::LDG_PER_ITEM];
#pragma unroll
                for (int j = 0; j < C::LDG_PER_ITEM; ++j) {
                    const uint32_t o = __shfl_sync(0xffffffffu, off, 2 * j + sub_row);
                    buf[j] = valid ? ldg_nc_v4(tab + (size_t)o + col) : make_float4(0.f, 0.f, 0.f, 0.f);
                }
                const int stage = it % C::STAGES;
                mbar_wait(bar_empty + 8 * stage, ((uint32_t)(it / C::STAGES) & 1u) ^ 1u, status);
                const uint32_t a_hi = base + stage * C::STAGE_BYTES, a_lo = a_hi + C::A_TILE;
#pragma unroll
                for (int j = 0; j < C::LDG_PER_ITEM; ++j) {
                    const int r = pw * C::ROWS_PER_PW + 2 * j + sub_row;
                    const uint32_t so = (uint32_t)((r >> 3) * 1024 + (r & 7) * 128 + ((((q >> 1) ^ (r & 7)) & 7) << 4) + (q & 1) * 8);
                    const float4 v = buf[j];
                    const __half2 h01 = __floats2half2_rn(v.x, v.y), h23 = __floats2half2_rn(v.z, v.w);
                    const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
                    sts_v2(a_hi + so, pack_h2(h01), pack_h2(h23));
                    if constexpr (one_pass<PASS>) continue;
                    sts_v2(a_lo + so, pack_h2(__floats2half2_rn(v.x - f01.x, v.y - f01.y)),
                           pack_h2(__floats2half2_rn(v.z - f23.x, v.w - f23.y)));
                }
                fence_proxy_async_smem();    // generic-proxy stores -> visible to the tensor cores (async proxy)
                __syncwarp();
                if (lane == 0) mbar_arrive(bar_full + 8 * stage);
            }
        }
    } else {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (warp == C::MISC_WARP0 && lane == 0) {
            // =============================== W PRODUCER ===============================
            const uint8_t *img = reinterpret_cast<const uint8_t *>(a.ws.w_hi);
            int kb = 0;
            for (int it = 0; it < n_items; ++it) {
                const int stage = it % C::STAGES;
                mbar_wait(bar_empty + 8 * stage, ((uint32_t)(it / C::STAGES) & 1u) ^ 1u, status);
                constexpr uint32_t bytes = one_pass<PASS> ? C::W_TILE : C::W_KB_BYTES;     // hi tile first in the image
                mbar_arrive_expect_tx(bar_full + 8 * stage, bytes);
                bulk_copy_g2s(base + stage * C::STAGE_BYTES + 2 * C::A_TILE, img + (size_t)kb * C::W_KB_BYTES, bytes,
                              bar_full + 8 * stage);
                if (++kb == C::NKB) kb = 0;
            }
        }
        __syncwarp();
    }
}

template <bool WIDE>
static int launch_wg(void (*kern)(const EncodeArgs), const EncodeArgs &a, cudaStream_t st)
{
    using C = WgCfg<WIDE>;
    int dev = 0, sms = 0;
    C2V_CUDA_OK(cudaGetDevice(&dev));
    C2V_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    C2V_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES));
    int grid = a.n_tiles < sms ? a.n_tiles : sms;
    if (grid < 1) grid = 1;
    C2V_CUDA_OK(launch_pdl(kern, dim3((unsigned)grid), dim3(C::THREADS), (size_t)C::SMEM_BYTES, st, a));
    C2V_COUNT_LAUNCH();
    return C2V_OK;
}

template <bool PACKED, class PASS>
static int launch_encode_wg(const EncodeArgs &a, cudaStream_t st)
{
    const bool drop = a.drop_p > 0.0f, dev_key = drop && a.seed_dev;
    if (a.H == 256)
        return launch_wg<true>(dev_key ? encode_wgmma_kernel<true, 256, PACKED, true, PASS>
                               : drop ? encode_wgmma_kernel<true, 256, PACKED, false, PASS>
                                      : encode_wgmma_kernel<false, 256, PACKED, false, PASS>, a, st);
    if (a.H == 128)
        return launch_wg<false>(dev_key ? encode_wgmma_kernel<true, 128, PACKED, true, PASS>
                                : drop ? encode_wgmma_kernel<true, 128, PACKED, false, PASS>
                                       : encode_wgmma_kernel<false, 128, PACKED, false, PASS>, a, st);
    if (a.H == 100)
        return launch_wg<false>(dev_key ? encode_wgmma_kernel<true, 100, PACKED, true, PASS>
                                : drop ? encode_wgmma_kernel<true, 100, PACKED, false, PASS>
                                       : encode_wgmma_kernel<false, 100, PACKED, false, PASS>, a, st);
    set_error("encode_wgmma_kernel: encode_size %d not supported (100, 128 or 256)", a.H);
    return C2V_EUNSUPPORTED;
}

// the matmul precision of the calling host thread picks the instantiations (c2v_set_matmul_precision)
int launch_encode_tcgen05(const EncodeArgs &a, cudaStream_t st)
{
    if (matmul_tf32())
        return a.bag_off ? launch_encode_wg<true, OnePass>(a, st) : launch_encode_wg<false, OnePass>(a, st);
    return a.bag_off ? launch_encode_wg<true, ThreePass>(a, st) : launch_encode_wg<false, ThreePass>(a, st);
}

}  // namespace c2v

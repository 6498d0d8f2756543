// c2v_adam.cu -- fused flat-buffer Adam: the optimizer side of the training step.
// torch.optim.Adam(model.parameters(), lr, betas, weight_decay) of main.py:138 + optimizer.step() (:175) +
// optimizer.zero_grad() (:171) for ALL parameters in one launch over flat fp32 buffers: reads p, g, m, v once, writes
// p, m, v and the zeroed gradient (ready for the next backward), and folds the 1/world of the data-parallel mean into
// the gradient read (the all_reduce then is a plain sum).  Dense on purpose: momentum keeps moving embedding rows that
// received no gradient, so a row-sparse Adam would not be the reference's optimizer.  That row-sparse Adam
// (torch.optim.SparseAdam, for tables with sparse gradients) is sparse_adam_step_kernel at the end of this file, opt-in.
// Same operation order as torch's single-tensor Adam (amsgrad=False, maximize=False):
//   g += wd * p;  m += (g - m) * (1 - b1);  v = v * b2 + (1 - b2) * g * g;
//   p -= (lr / (1 - b1^t)) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
#include <cstring>

#include "c2v_common.cuh"

namespace c2v {

__global__ void __launch_bounds__(256)
adam_step_kernel(float4 *__restrict__ p, float4 *__restrict__ g, float4 *__restrict__ m, float4 *__restrict__ v,
                 long long n4, float *__restrict__ pt, float *__restrict__ gt, float *__restrict__ mt, float *__restrict__ vt,
                 int tail, float step_size, float one_minus_b1, float b2, float one_minus_b2, float inv_sqrt_bc2, float eps,
                 float wd, float gscale, int zero_grad)
{
    auto upd = [&](float &pp, float &gg, float &mm, float &vv) {
        float gr = gg * gscale;
        if (wd != 0.0f) gr = fmaf(wd, pp, gr);
        mm = mm + (gr - mm) * one_minus_b1;                 // exp_avg.lerp_(grad, 1 - beta1)
        vv = vv * b2 + one_minus_b2 * gr * gr;              // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
        const float denom = sqrtf(vv) * inv_sqrt_bc2 + eps;
        pp = pp - step_size * (mm / denom);                 // param.addcdiv_(exp_avg, denom, value=-step_size)
        if (zero_grad) gg = 0.0f;
    };
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        float4 P = p[i], G = g[i], M = m[i], V = v[i];
        upd(P.x, G.x, M.x, V.x); upd(P.y, G.y, M.y, V.y); upd(P.z, G.z, M.z, V.z); upd(P.w, G.w, M.w, V.w);
        p[i] = P; m[i] = M; v[i] = V;
        if (zero_grad) g[i] = G;
    }
    if (blockIdx.x == 0 && (int)threadIdx.x < tail) {
        const int i = threadIdx.x;
        float P = pt[i], G = gt[i], M = mt[i], V = vt[i];
        upd(P, G, M, V);
        pt[i] = P; mt[i] = M; vt[i] = V;
        if (zero_grad) gt[i] = G;
    }
}

// ------------------------------------------------------------------------------------------------------------------
// Sharded step over NVLink (data-parallel training + section 5 "later option"): ONE kernel per rank does
// the gradient reduction, the optimizer and the parameter broadcast for the rank's 1/world slice of the flat buffers:
//   g  = sum over ranks of grad[slice]      multimem.ld_reduce.add.f32 through the NVSwitch multicast mapping
//                                           (in-switch reduction, NVLS) or fixed-order loads from the peers' buffers
//   Adam on (p, m, v)[slice]                m, v exist only on the owner of the slice (1/world of the optimizer state)
//   p' -> every rank's parameter buffer     multimem.st (one store, the switch replicates it) or world peer stores
// and, while the NVLink traffic is in flight, zeroes the rank's OTHER gradient bucket (the buckets alternate between
// steps: peers may still be reading this step's bucket, nobody reads the other one).  The caller brackets the launch
// with two cross-GPU barriers (all gradients complete before / all parameter stores landed after).
// ------------------------------------------------------------------------------------------------------------------
struct AdamPeers { float *param[16]; const float *grad[16]; };

__device__ __forceinline__ float4 mm_ld_reduce_add(const float *mc) {
    float4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(mc) : "memory");
    return v;
}
__device__ __forceinline__ void mm_st(float *mc, float4 v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};"
                 ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// 128-thread CTAs (<= 64 registers): 8 K registers per CTA, so that the kernel can share SMs with the persistent tensor-core
// backward kernels (22 warps x 72-80 registers leave ~9-15 K of the 64 K registers) when it runs on a side stream.
template <bool MULTIMEM>
__global__ void __launch_bounds__(128)
adam_step_sharded_kernel(const float *__restrict__ p_local, float *__restrict__ p_mc, const float *__restrict__ g_mc,
                         const AdamPeers peers, int world, float4 *__restrict__ m, float4 *__restrict__ v,
                         long long slice_begin, long long slice_n4, float4 *__restrict__ zero_buf, long long zero_n4,
                         float step_size, float one_minus_b1, float b2, float one_minus_b2, float inv_sqrt_bc2, float eps,
                         float wd, float gscale)
{
    auto upd = [&](float &pp, float gg, float &mm, float &vv) {
        float gr = gg * gscale;
        if (wd != 0.0f) gr = fmaf(wd, pp, gr);
        mm = mm + (gr - mm) * one_minus_b1;
        vv = vv * b2 + one_minus_b2 * gr * gr;
        const float denom = sqrtf(vv) * inv_sqrt_bc2 + eps;
        pp = pp - step_size * (mm / denom);
    };
    // Every 4th CTA only zero-fills the other gradient bucket (local HBM stores), the rest do the NVLink work, two 16-byte
    // pieces per thread and iteration so that twice the bytes are in flight per thread (the in-switch reduction has a
    // round trip of several microseconds): both halves of the step run side by side instead of one after the other.
    const int n_zero_cta = zero_n4 > 0 ? (int)gridDim.x / 4 : 0;
    const bool zero_role = n_zero_cta > 0 && (blockIdx.x & 3) == 3;
    if (zero_role) {
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        const long long zstride = (long long)n_zero_cta * blockDim.x;
        for (long long i = (long long)(blockIdx.x >> 2) * blockDim.x + threadIdx.x; i < zero_n4; i += zstride) zero_buf[i] = z;
        return;
    }
    const int wb = (int)blockIdx.x - (n_zero_cta > 0 ? (int)(blockIdx.x + 1) / 4 : 0);
    const long long stride = (long long)((int)gridDim.x - n_zero_cta) * blockDim.x, t0 = (long long)wb * blockDim.x + threadIdx.x;
    for (long long i0 = t0; i0 < slice_n4; i0 += 2 * stride) {
        const long long i1 = i0 + stride;
        const bool two = i1 < slice_n4;
        const long long e0 = slice_begin + 4 * i0, e1 = slice_begin + 4 * (two ? i1 : i0);   // element offsets in the flat buffers
        float4 G0, G1;
        if (MULTIMEM) { G0 = mm_ld_reduce_add(g_mc + e0); G1 = two ? mm_ld_reduce_add(g_mc + e1) : G0; }
        else {
            G0 = G1 = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int r = 0; r < world; ++r) {                   // fixed rank order: every replica of the sum is bit-identical
                const float4 x0 = *reinterpret_cast<const float4 *>(peers.grad[r] + e0);
                const float4 x1 = *reinterpret_cast<const float4 *>(peers.grad[r] + e1);
                G0.x += x0.x; G0.y += x0.y; G0.z += x0.z; G0.w += x0.w;
                G1.x += x1.x; G1.y += x1.y; G1.z += x1.z; G1.w += x1.w;
            }
        }
        float4 P0 = *reinterpret_cast<const float4 *>(p_local + e0), M0 = m[i0], V0 = v[i0];
        float4 P1 = *reinterpret_cast<const float4 *>(p_local + e1), M1 = m[two ? i1 : i0], V1 = v[two ? i1 : i0];
        upd(P0.x, G0.x, M0.x, V0.x); upd(P0.y, G0.y, M0.y, V0.y); upd(P0.z, G0.z, M0.z, V0.z); upd(P0.w, G0.w, M0.w, V0.w);
        m[i0] = M0; v[i0] = V0;
        if (MULTIMEM) mm_st(p_mc + e0, P0);
        else
            for (int r = 0; r < world; ++r) *reinterpret_cast<float4 *>(peers.param[r] + e0) = P0;
        if (two) {
            upd(P1.x, G1.x, M1.x, V1.x); upd(P1.y, G1.y, M1.y, V1.y); upd(P1.z, G1.z, M1.z, V1.z); upd(P1.w, G1.w, M1.w, V1.w);
            m[i1] = M1; v[i1] = V1;
            if (MULTIMEM) mm_st(p_mc + e1, P1);
            else
                for (int r = 0; r < world; ++r) *reinterpret_cast<float4 *>(peers.param[r] + e1) = P1;
        }
    }
    __threadfence_system();
}

// ------------------------------------------------------------------------------------------------------------------
// The same step driven by bulk-async copies (TMA) instead of thousands of threads: four warps per CTA, 28 KB of shared
// memory.  Purpose: run on a side stream NEXT TO the persistent tensor-core backward kernels, which own every SM
// (22 warps x 72-80 registers, 197 KB of shared memory) and leave room for exactly this much -- the thread-per-element
// kernel above cannot get enough CTAs resident beside them to keep NVLink busy.  Per chunk: lane 0 issues one
// cp.async.bulk per rank (peer gradient slice -> shared memory, completion on an mbarrier; 2 stages = the bytes in flight),
// the warp sums the `world` copies in rank order, runs Adam on the chunk (p, m, v are local: plain vector loads / stores),
// writes the new parameters into the stage's first buffer and lane 0 issues one bulk store per rank (shared -> peer
// parameter buffer).  Peer pointers only (no multicast): region 0 of ShardedFlatAdam (early_step).
// ------------------------------------------------------------------------------------------------------------------
constexpr int AB_STAGES = 2, AB_STAGE_BYTES = 14 * 1024;

__device__ __forceinline__ uint32_t ab_smem(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

constexpr int AB_THREADS = 128;          // 4 warps x <= 48 registers = 6 K registers: fits beside the tensor-core backward kernels

__global__ void __launch_bounds__(AB_THREADS)
adam_step_bulk_kernel(const float *__restrict__ p_local, const AdamPeers peers, int world, float *__restrict__ m,
                      float *__restrict__ v, long long slice_begin, long long slice_n, int chunk,
                      float step_size, float one_minus_b1, float b2, float one_minus_b2, float inv_sqrt_bc2, float eps,
                      float wd, float gscale)
{
    extern __shared__ __align__(128) unsigned char ab_raw[];
    __shared__ __align__(8) unsigned long long ab_bar[AB_STAGES];
    const int tid = threadIdx.x;
    const long long n_chunks = (slice_n + chunk - 1) / chunk;
    const long long my_chunks = (n_chunks - (long long)blockIdx.x + (long long)gridDim.x - 1) / (long long)gridDim.x;
    if (tid == 0) {
        for (int s = 0; s < AB_STAGES; ++s)
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(ab_smem(&ab_bar[s])));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    auto issue = [&](long long k) {                               // thread 0: loads of this CTA's k-th chunk into stage k & 1
        const long long c = (long long)blockIdx.x + k * gridDim.x;
        const long long off = c * chunk;
        const int len = (int)((slice_n - off) < chunk ? (slice_n - off) : chunk);
        const uint32_t bytes = (uint32_t)len * 4u;
        const int st = (int)(k & 1);
        const uint32_t bar = ab_smem(&ab_bar[st]);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes * (uint32_t)world) : "memory");
        for (int r = 0; r < world; ++r) {
            const uint32_t dst = ab_smem(ab_raw + (size_t)st * AB_STAGE_BYTES + (size_t)r * chunk * 4);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(dst), "l"(peers.grad[r] + slice_begin + off), "r"(bytes), "r"(bar) : "memory");
        }
    };
    auto upd = [&](float &pp, float gg, float &mm, float &vv) {
        float gr = gg * gscale;
        if (wd != 0.0f) gr = fmaf(wd, pp, gr);
        mm = mm + (gr - mm) * one_minus_b1;
        vv = vv * b2 + one_minus_b2 * gr * gr;
        const float denom = sqrtf(vv) * inv_sqrt_bc2 + eps;
        pp = pp - step_size * (mm / denom);
    };
    if (tid == 0 && my_chunks > 0) issue(0);
    for (long long k = 0; k < my_chunks; ++k) {
        const int st = (int)(k & 1);
        if (tid == 0 && k + 1 < my_chunks) {
            // the other stage's first buffer was the source of chunk k-1's bulk stores: wait until those have READ it
            asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
            issue(k + 1);
        }
        const long long c = (long long)blockIdx.x + k * gridDim.x;
        const long long off = c * chunk;
        const int len = (int)((slice_n - off) < chunk ? (slice_n - off) : chunk);
        // p, m, v of this thread's first piece are local HBM: fetch them while the peers' gradients are still in flight
        const int i0 = tid * 4;
        float4 P0 = make_float4(0.f, 0.f, 0.f, 0.f), M0 = P0, V0 = P0;
        if (i0 < len) {
            P0 = *reinterpret_cast<const float4 *>(p_local + slice_begin + off + i0);
            M0 = *reinterpret_cast<const float4 *>(m + off + i0); V0 = *reinterpret_cast<const float4 *>(v + off + i0);
        }
        {   // wait for this stage's loads
            const uint32_t bar = ab_smem(&ab_bar[st]), parity = (uint32_t)(k >> 1) & 1u;
            uint32_t ok = 0;
            while (!ok) {
                asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                             : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
            }
        }
        float *stage = reinterpret_cast<float *>(ab_raw + (size_t)st * AB_STAGE_BYTES);
        for (int i = i0; i < len; i += 4 * AB_THREADS) {          // len is a multiple of 4 (slices are)
            float4 G = *reinterpret_cast<const float4 *>(stage + i);
            for (int r = 1; r < world; ++r) {                      // rank order: replicas of the sum are bit-identical
                const float4 x = *reinterpret_cast<const float4 *>(stage + (size_t)r * chunk + i);
                G.x += x.x; G.y += x.y; G.z += x.z; G.w += x.w;
            }
            const long long e = off + i;                           // offset inside the slice
            float4 P, M, V;
            if (i == i0) { P = P0; M = M0; V = V0; }
            else {
                P = *reinterpret_cast<const float4 *>(p_local + slice_begin + e);
                M = *reinterpret_cast<const float4 *>(m + e); V = *reinterpret_cast<const float4 *>(v + e);
            }
            upd(P.x, G.x, M.x, V.x); upd(P.y, G.y, M.y, V.y); upd(P.z, G.z, M.z, V.z); upd(P.w, G.w, M.w, V.w);
            *reinterpret_cast<float4 *>(m + e) = M; *reinterpret_cast<float4 *>(v + e) = V;
            *reinterpret_cast<float4 *>(stage + i) = P;            // rank 0's buffer becomes the output staging
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");    // generic-proxy stores -> visible to the bulk stores
        __syncthreads();
        if (tid == 0) {
            const uint32_t src = ab_smem(stage), bytes = (uint32_t)len * 4u;
            for (int r = 0; r < world; ++r)
                asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                             ::"l"(peers.param[r] + slice_begin + off), "r"(src), "r"(bytes) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
    }
    if (tid == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // all stores performed before the kernel ends
    __syncthreads();
    __threadfence_system();
}

// ------------------------------------------------------------------------------------------------------------------
// torch.optim._functional.sparse_adam on the rows of a coalesced gradient, every operation rounded as torch rounds it
// (the _rn intrinsics keep nvcc from contracting a multiply and an add into one fma).  One warp per gradient row.
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
sparse_adam_step_kernel(float *__restrict__ p, float *__restrict__ m, float *__restrict__ v, const float *__restrict__ g,
                        const long long *__restrict__ rows, long long U, long long n_rows, int E, float neg_step_size,
                        float one_minus_b1, float one_minus_b2, float eps)
{
    const int lane = threadIdx.x & 31;
    const long long n_warps = (long long)gridDim.x * (blockDim.x >> 5);
    for (long long i = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); i < U; i += n_warps) {
        const long long r = rows[i];
        if (r < 0 || r >= n_rows) continue;
        const float *gi = g + (size_t)i * E;
        float *pr = p + (size_t)r * E, *mr = m + (size_t)r * E, *vr = v + (size_t)r * E;
        for (int c = lane; c < E; c += 32) {
            const float gg = gi[c], m0 = mr[c], v0 = vr[c];
            const float u1 = __fmul_rn(__fsub_rn(gg, m0), one_minus_b1);              // (g - m) * (1 - b1)
            const float u2 = __fmul_rn(__fsub_rn(__fmul_rn(gg, gg), v0), one_minus_b2); // (g^2 - v) * (1 - b2)
            mr[c] = __fadd_rn(m0, u1);
            vr[c] = __fadd_rn(v0, u2);
            const float numer = __fadd_rn(u1, m0);
            const float denom = __fadd_rn(__fsqrt_rn(__fadd_rn(u2, v0)), eps);
            pr[c] = __fadd_rn(pr[c], __fmul_rn(neg_step_size, __fdiv_rn(numer, denom)));
        }
    }
}

}  // namespace c2v

using namespace c2v;

static bool misaligned(const void *ptr, uintptr_t a) { return (reinterpret_cast<uintptr_t>(ptr) & (a - 1)) != 0; }

extern "C" int c2v_adam_step(float *param, float *grad, float *exp_avg, float *exp_avg_sq, int64_t n, float lr,
                             float beta1, float beta2, float eps, float weight_decay, int64_t step, float grad_scale,
                             int32_t zero_grad, void *stream)
{
    if (!param || !grad || !exp_avg || !exp_avg_sq || n < 1 || step < 1) {
        set_error("c2v_adam_step: bad argument");
        return C2V_EINVAL;
    }
    if ((reinterpret_cast<uintptr_t>(param) | reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(exp_avg) |
         reinterpret_cast<uintptr_t>(exp_avg_sq)) & 15) {
        set_error("c2v_adam_step: buffers must be 16-byte aligned");
        return C2V_EINVAL;
    }
    const double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);
    const float step_size = (float)((double)lr / bc1);
    const float inv_sqrt_bc2 = (float)(1.0 / sqrt(bc2));
    const long long n4 = n / 4;
    const int tail = (int)(n % 4);
    int dev = 0, sms = 0;
    C2V_CUDA_OK(cudaGetDevice(&dev));
    C2V_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    long long blocks = (n4 + 255) / 256;
    if (blocks > (long long)sms * 16) blocks = (long long)sms * 16;
    if (blocks < 1) blocks = 1;
    adam_step_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<float4 *>(param), reinterpret_cast<float4 *>(grad), reinterpret_cast<float4 *>(exp_avg),
        reinterpret_cast<float4 *>(exp_avg_sq), n4, param + n4 * 4, grad + n4 * 4, exp_avg + n4 * 4, exp_avg_sq + n4 * 4, tail,
        step_size, 1.0f - beta1, beta2, 1.0f - beta2, inv_sqrt_bc2, eps, weight_decay, grad_scale, zero_grad);
    C2V_LAUNCH_OK("adam_step_kernel");
    return C2V_OK;
}

extern "C" int c2v_adam_step_sharded(const float *param_local, float *param_multicast, const float *grad_multicast,
                                     float *const *param_peers, const float *const *grad_peers, int32_t world,
                                     float *exp_avg_slice, float *exp_avg_sq_slice, int64_t slice_begin, int64_t slice_n,
                                     float *zero_buffer, int64_t zero_n, float lr, float beta1, float beta2, float eps,
                                     float weight_decay, int64_t step, float grad_scale, void *stream)
{
    if (!param_local || !exp_avg_slice || !exp_avg_sq_slice || slice_n < 0 || slice_begin < 0 || step < 1 || world < 1 ||
        world > 16) {
        set_error("c2v_adam_step_sharded: bad argument");
        return C2V_EINVAL;
    }
    const bool mm = param_multicast != nullptr && grad_multicast != nullptr;
    if (!mm && (!param_peers || !grad_peers)) {
        set_error("c2v_adam_step_sharded: needs either the multicast pointers or the peer pointer tables");
        return C2V_EINVAL;
    }
    if ((slice_begin | slice_n | zero_n) & 3) {
        set_error("c2v_adam_step_sharded: slice_begin, slice_n and zero_n must be multiples of 4 elements");
        return C2V_EINVAL;
    }
    AdamPeers peers;
    memset(&peers, 0, sizeof(peers));
    uintptr_t align = reinterpret_cast<uintptr_t>(param_local) | reinterpret_cast<uintptr_t>(exp_avg_slice) |
                      reinterpret_cast<uintptr_t>(exp_avg_sq_slice) | reinterpret_cast<uintptr_t>(zero_buffer) |
                      reinterpret_cast<uintptr_t>(param_multicast) | reinterpret_cast<uintptr_t>(grad_multicast);
    if (!mm)
        for (int r = 0; r < world; ++r) {
            if (!param_peers[r] || !grad_peers[r]) { set_error("c2v_adam_step_sharded: NULL peer pointer %d", r); return C2V_EINVAL; }
            peers.param[r] = param_peers[r]; peers.grad[r] = grad_peers[r];
            align |= reinterpret_cast<uintptr_t>(param_peers[r]) | reinterpret_cast<uintptr_t>(grad_peers[r]);
        }
    if (align & 15) { set_error("c2v_adam_step_sharded: buffers must be 16-byte aligned"); return C2V_EINVAL; }
    const double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);
    const float step_size = (float)((double)lr / bc1);
    const float inv_sqrt_bc2 = (float)(1.0 / sqrt(bc2));
    int dev = 0, sms = 0;
    C2V_CUDA_OK(cudaGetDevice(&dev));
    C2V_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const long long n4 = slice_n / 4, z4 = zero_buffer ? zero_n / 4 : 0;
    long long blocks = ((n4 > z4 ? n4 : z4) + 127) / 128;
    if (blocks > (long long)sms * 16) blocks = (long long)sms * 16;
    if (blocks < 4) blocks = 4;
    blocks = blocks / 4 * 4;                                  // every 4th CTA zero-fills
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (mm)
        adam_step_sharded_kernel<true><<<(unsigned)blocks, 128, 0, st>>>(
            param_local, param_multicast, grad_multicast, peers, world, reinterpret_cast<float4 *>(exp_avg_slice),
            reinterpret_cast<float4 *>(exp_avg_sq_slice), slice_begin, n4, reinterpret_cast<float4 *>(zero_buffer), z4,
            step_size, 1.0f - beta1, beta2, 1.0f - beta2, inv_sqrt_bc2, eps, weight_decay, grad_scale);
    else
        adam_step_sharded_kernel<false><<<(unsigned)blocks, 128, 0, st>>>(
            param_local, param_multicast, grad_multicast, peers, world, reinterpret_cast<float4 *>(exp_avg_slice),
            reinterpret_cast<float4 *>(exp_avg_sq_slice), slice_begin, n4, reinterpret_cast<float4 *>(zero_buffer), z4,
            step_size, 1.0f - beta1, beta2, 1.0f - beta2, inv_sqrt_bc2, eps, weight_decay, grad_scale);
    C2V_LAUNCH_OK("adam_step_sharded_kernel");
    return C2V_OK;
}

extern "C" int c2v_adam_step_sharded_bulk(const float *param_local, float *const *param_peers, const float *const *grad_peers,
                                          int32_t world, float *exp_avg_slice, float *exp_avg_sq_slice, int64_t slice_begin,
                                          int64_t slice_n, float lr, float beta1, float beta2, float eps, float weight_decay,
                                          int64_t step, float grad_scale, int32_t max_ctas, void *stream)
{
    if (!param_local || !param_peers || !grad_peers || !exp_avg_slice || !exp_avg_sq_slice || slice_n < 0 || slice_begin < 0 ||
        step < 1 || world < 1 || world > 16 || ((slice_begin | slice_n) & 3)) {
        set_error("c2v_adam_step_sharded_bulk: bad argument");
        return C2V_EINVAL;
    }
    AdamPeers peers;
    memset(&peers, 0, sizeof(peers));
    uintptr_t align = reinterpret_cast<uintptr_t>(param_local) | reinterpret_cast<uintptr_t>(exp_avg_slice) |
                      reinterpret_cast<uintptr_t>(exp_avg_sq_slice);
    for (int r = 0; r < world; ++r) {
        if (!param_peers[r] || !grad_peers[r]) { set_error("c2v_adam_step_sharded_bulk: NULL peer pointer %d", r); return C2V_EINVAL; }
        peers.param[r] = param_peers[r]; peers.grad[r] = grad_peers[r];
        align |= reinterpret_cast<uintptr_t>(param_peers[r]) | reinterpret_cast<uintptr_t>(grad_peers[r]);
    }
    if (align & 15) { set_error("c2v_adam_step_sharded_bulk: buffers must be 16-byte aligned"); return C2V_EINVAL; }
    if (slice_n == 0) return C2V_OK;
    const double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);
    const float step_size = (float)((double)lr / bc1);
    const float inv_sqrt_bc2 = (float)(1.0 / sqrt(bc2));
    int dev = 0, sms = 0;
    C2V_CUDA_OK(cudaGetDevice(&dev));
    C2V_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const int chunk = AB_STAGE_BYTES / 4 / world / 4 * 4;          // floats per rank and stage (16-byte multiple)
    const long long n_chunks = (slice_n + chunk - 1) / chunk;
    long long grid = max_ctas > 0 ? max_ctas : sms;
    if (grid > n_chunks) grid = n_chunks;
    const int smem = AB_STAGES * AB_STAGE_BYTES;
    C2V_CUDA_OK(cudaFuncSetAttribute(adam_step_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    adam_step_bulk_kernel<<<(unsigned)grid, AB_THREADS, smem, static_cast<cudaStream_t>(stream)>>>(
        param_local, peers, world, exp_avg_slice, exp_avg_sq_slice, slice_begin, slice_n, chunk, step_size, 1.0f - beta1, beta2,
        1.0f - beta2, inv_sqrt_bc2, eps, weight_decay, grad_scale);
    C2V_LAUNCH_OK("adam_step_bulk_kernel");
    return C2V_OK;
}

extern "C" int c2v_sparse_adam_step(float *param, float *exp_avg, float *exp_avg_sq, const float *values,
                                    const int64_t *rows, int64_t U, int64_t n_rows, int32_t E, double lr, double beta1,
                                    double beta2, double eps, int64_t step, void *stream)
{
    if (U < 0 || n_rows < 1 || E < 1 || E > 65536 || step < 1) {
        set_error("c2v_sparse_adam_step: bad argument (U = %lld, n_rows = %lld, E = %d, step = %lld)", (long long)U,
                  (long long)n_rows, E, (long long)step);
        return C2V_EINVAL;
    }
    if (!param || !exp_avg || !exp_avg_sq || (U > 0 && (!values || !rows))) {
        set_error("c2v_sparse_adam_step: NULL pointer argument");
        return C2V_EINVAL;
    }
    if (misaligned(param, 4) || misaligned(exp_avg, 4) || misaligned(exp_avg_sq, 4) || misaligned(values, 4) ||
        misaligned(rows, 8)) {
        set_error("c2v_sparse_adam_step: misaligned pointer (float buffers: 4 bytes, rows: 8)");
        return C2V_EINVAL;
    }
    if (U == 0) return C2V_OK;
    // torch: step_size = lr * sqrt(1 - b2^t) / (1 - b1^t) and the 1 - b factors in double, applied to float tensors
    const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
    const double step_size = lr * sqrt(bc2) / bc1;
    int dev = 0, sms = 0;
    C2V_CUDA_OK(cudaGetDevice(&dev));
    C2V_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    long long blocks = (U + 7) / 8;
    if (blocks > (long long)sms * 8) blocks = (long long)sms * 8;
    sparse_adam_step_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        param, exp_avg, exp_avg_sq, values, reinterpret_cast<const long long *>(rows), U, n_rows, E, (float)(-step_size),
        (float)(1.0 - beta1), (float)(1.0 - beta2), (float)eps);
    C2V_LAUNCH_OK("sparse_adam_step_kernel");
    return C2V_OK;
}

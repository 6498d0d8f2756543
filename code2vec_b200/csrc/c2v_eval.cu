// c2v_eval.cu -- evaluation metrics of the eval pass (main.py:267-297) as integer counts on the device.
//
// One warp per row.  The warp finds the first rank of the label among the row's k predictions (a ballot per 32 ranks),
// then compares the subtoken lists E = S(label) and P = S(best prediction) across its lanes: lane l checks entries
// l, l + 32, ... of P against all of E (tp) and of E against all of P (fn), so lists of any length work.  Lane 0 adds
// the per-class counts with integer atomics and keeps the row's scalar counts in registers; the block adds its warps'
// counts in shared memory and issues one integer atomic per counter.  Every count is an integer, so the result does not
// depend on the batch split, the row order or the launch order.
#include "c2v_common.cuh"

namespace c2v {

namespace evalk {
constexpr int THREADS = 256, WARPS = THREADS / 32;
constexpr int SHARED_RANKS = 1024;          // rank-hit counters kept in shared memory; deeper ranks go straight to global
constexpr int NSCALAR = 8;                  // n, skipped, tp, fp, fn and the three fixed-point sums
}

__device__ __forceinline__ unsigned long long fx_ratio(unsigned long long num, unsigned long long den)
{
    return den ? (num << 32) / den : 0ull;    // floor(num / den * 2^32); 0 for 0 / 0
}

// how many entries of a[0..na) occur in b[0..nb), counted across the warp (entries of a split over the lanes); a 32-bit
// count: a list holds fewer than 2^31 entries
__device__ __forceinline__ long long warp_count_in(const int *__restrict__ a, long long na, const int *__restrict__ b,
                                                   long long nb, int lane)
{
    int c = 0;
    for (long long i = lane; i < na; i += 32) {
        const int v = a[i];
        bool found = false;
        for (long long j = 0; j < nb && !found; ++j) found = b[j] == v;
        c += found;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    return c;
}

__global__ void __launch_bounds__(evalk::THREADS)
eval_accumulate_kernel(const long long *__restrict__ label, const long long *__restrict__ pred, int B, int k, long long C,
                       const long long *__restrict__ sub_off, const int *__restrict__ sub_ids,
                       unsigned long long *__restrict__ counters, unsigned long long *__restrict__ class_counts)
{
    extern __shared__ unsigned long long s_hits[];                 // min(k, SHARED_RANKS)
    __shared__ unsigned long long s_scalar[evalk::WARPS][evalk::NSCALAR];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int shared_k = min(k, evalk::SHARED_RANKS);
    for (int i = threadIdx.x; i < shared_k; i += blockDim.x) s_hits[i] = 0;
    __syncthreads();

    // lane 0's counts: n, skipped, tp, fp, fn, sum prec, sum rec, sum f1 (fixed point, units of 2^-32)
    unsigned long long acc[evalk::NSCALAR] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (long long row = (long long)blockIdx.x * evalk::WARPS + warp; row < B; row += (long long)gridDim.x * evalk::WARPS) {
        const long long y = label[row];
        if (y < 0 || y >= C) {                                     // unlabelled (-1) or ignore_index: skipped
            acc[1] += 1;
            continue;
        }
        const long long *p = pred + row * k;
        int rank = -1;
        for (int base = 0; base < k; base += 32) {
            const int j = base + lane;
            const unsigned hit = __ballot_sync(0xffffffffu, j < k && p[j] == y);
            if (hit) { rank = base + __ffs(hit) - 1; break; }
        }
        const long long p0 = p[0];
        const bool p0_ok = p0 >= 0 && p0 < C;
        const long long e_lo = sub_off[y], e_n = sub_off[y + 1] - e_lo;
        const long long q_lo = p0_ok ? sub_off[p0] : 0, q_n = p0_ok ? sub_off[p0 + 1] - q_lo : 0;
        const long long tp = warp_count_in(sub_ids + q_lo, q_n, sub_ids + e_lo, e_n, lane);
        const long long fn = e_n - warp_count_in(sub_ids + e_lo, e_n, sub_ids + q_lo, q_n, lane);
        if (lane == 0) {
            const unsigned long long utp = tp, ufp = q_n - tp, ufn = fn;
            acc[0] += 1;
            acc[2] += utp; acc[3] += ufp; acc[4] += ufn;
            acc[5] += fx_ratio(utp, utp + ufp);
            acc[6] += fx_ratio(utp, utp + ufn);
            acc[7] += fx_ratio(2 * utp, 2 * utp + ufp + ufn);
            if (rank >= 0) {
                if (rank < shared_k) atomicAdd(&s_hits[rank], 1ull);
                else atomicAdd(&counters[2 + rank], 1ull);
            }
            atomicAdd(&class_counts[y], 1ull);                     // true
            if (p0_ok) atomicAdd(&class_counts[C + p0], 1ull);     // pred
            if (p0 == y) atomicAdd(&class_counts[2 * C + y], 1ull);   // hit
        }
    }
    if (lane == 0) {
#pragma unroll
        for (int i = 0; i < evalk::NSCALAR; ++i) s_scalar[warp][i] = acc[i];
    }
    __syncthreads();
    if (threadIdx.x < evalk::NSCALAR) {
        unsigned long long s = 0;
#pragma unroll
        for (int w = 0; w < evalk::WARPS; ++w) s += s_scalar[w][threadIdx.x];
        // counter index: n 0, skipped 1, then tp / fp / fn / sums behind the k rank hits
        const int at = threadIdx.x < 2 ? threadIdx.x : 2 + k + (threadIdx.x - 2);
        if (s) atomicAdd(&counters[at], s);
    }
    for (int i = threadIdx.x; i < shared_k; i += blockDim.x)
        if (s_hits[i]) atomicAdd(&counters[2 + i], s_hits[i]);
}

}  // namespace c2v

using namespace c2v;

extern "C" int c2v_eval_accumulate(const int64_t *label, const int64_t *pred, int32_t B, int32_t k, int64_t C,
                                   const int64_t *subtoken_offsets, const int32_t *subtoken_ids, int64_t *counters,
                                   int64_t *class_counts, void *stream)
{
    const char *null_arg = !label ? "label" : !pred ? "pred" : !subtoken_offsets ? "subtoken_offsets" :
                           !subtoken_ids ? "subtoken_ids" : !counters ? "counters" : !class_counts ? "class_counts" : nullptr;
    if (null_arg) {
        set_error("c2v_eval_accumulate: %s is NULL", null_arg);
        return C2V_EINVAL;
    }
    if (B < 1) {
        set_error("c2v_eval_accumulate: B = %d < 1", (int)B);
        return C2V_EINVAL;
    }
    if (C < 1) {
        set_error("c2v_eval_accumulate: C = %lld < 1", (long long)C);
        return C2V_EINVAL;
    }
    if (k < 1 || k > C) {
        set_error("c2v_eval_accumulate: k = %d outside [1, C = %lld]", (int)k, (long long)C);
        return C2V_EINVAL;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    long long blocks = ((long long)B + evalk::WARPS - 1) / evalk::WARPS;
    if (blocks > 4096) blocks = 4096;
    const size_t smem = (size_t)min((int)k, evalk::SHARED_RANKS) * sizeof(unsigned long long);
    eval_accumulate_kernel<<<(unsigned)blocks, evalk::THREADS, smem, st>>>(
        reinterpret_cast<const long long *>(label), reinterpret_cast<const long long *>(pred), (int)B, (int)k, (long long)C,
        reinterpret_cast<const long long *>(subtoken_offsets), reinterpret_cast<const int *>(subtoken_ids),
        reinterpret_cast<unsigned long long *>(counters), reinterpret_cast<unsigned long long *>(class_counts));
    C2V_LAUNCH_OK("eval_accumulate_kernel");
    return C2V_OK;
}

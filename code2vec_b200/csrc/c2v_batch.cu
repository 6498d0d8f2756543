// c2v_batch.cu -- on-GPU batch construction for the method-name task: the device-side counterpart of
// DatasetBuilder.build_data (/root/reference/model/dataset_builder.py:112-150, infer_method branch) +
// pad_inputs (:212-219).  The corpus stays in HBM as CSR (offsets [n_items + 1] int64, contexts
// [total][3] int32 = start, path, end); one CTA builds one row of the [B, L] int64 index tensors the encode kernel
// reads: a uniformly random subset of min(n, L) contexts of the method (the reference shuffles and truncates),
// @method_0 -> @question (:136-143), zero-padded suffix.  Randomness is a counter-based hash of (seed, item, j), so
// the result is a pure function of its arguments; oracle/batch_oracle.py is the bit-exact CPU restatement.
//
// Variable-name task (build_batch_vars_kernel, dataset_builder.py:152-204, infer_variable branch): the unit is an
// (item, @var_k) pair; its bag is the contexts of the item that touch @var_k (start or end), with @var_k -> @question,
// every other @var_* token mapped through the per-item permutation of `variable_indexes` when shuffle_variable_indexes
// is set (:166-168, identity otherwise), truncated to a uniformly random subset of max_path_length (:193-195).
#include "c2v_common.cuh"

namespace c2v {

__device__ __forceinline__ unsigned long long bb_mix64(unsigned long long x) {      // splitmix64 finalizer
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}
__device__ __forceinline__ unsigned bb_key(unsigned long long base, long long j) {
    return (unsigned)(bb_mix64(base ^ ((unsigned long long)j * 0x8CB92BA72F3D8DD7ull)) >> 32);
}

// exclusive prefix sum of one flag per thread over a 256-thread CTA; returns this thread's offset, *total = CTA sum
__device__ __forceinline__ int bb_block_scan(int flag, int *s_warp, int *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    const int in_warp = __popc(bal & ((1u << lane) - 1u));
    if (lane == 0) s_warp[warp] = __popc(bal);
    __syncthreads();
    int before = 0, sum = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) { const int c = s_warp[w]; before += w < warp ? c : 0; sum += c; }
    __syncthreads();
    *total = sum;
    return before + in_warp;
}

// PACKED: bag b goes to rows bag_off[b] .. bag_off[b+1]-1 (its length: min(n, L), 1 for an empty or unknown item)
// instead of row b of the [B, L] tensors; the same contexts, without the zero suffix.
template <bool PACKED = false>
__global__ void __launch_bounds__(256)
build_batch_kernel(const long long *__restrict__ offsets, const int *__restrict__ ctx, long long n_items,
                   const long long *__restrict__ item_ids, const long long *__restrict__ item_labels, int L,
                   unsigned long long seed, long long method_token, long long question_token,
                   long long *__restrict__ starts, long long *__restrict__ paths, long long *__restrict__ ends,
                   long long *__restrict__ label, const long long *__restrict__ bag_off)
{
    __shared__ unsigned hist[256];
    __shared__ int s_warp[8];
    __shared__ unsigned s_prefix, s_k;
    const int b = blockIdx.x, tid = threadIdx.x;
    const long long item = item_ids[b];
    const long long row0 = PACKED ? bag_off[b] : (long long)b * L;
    long long *rs = starts + row0, *rp = paths + row0, *re = ends + row0;
    if (PACKED) {                                            // the host-computed length, clamped into [0, L]
        const long long len = bag_off[b + 1] - row0;
        L = len < 0 ? 0 : (len > L ? L : (int)len);
    }
    if (item < 0 || item >= n_items) {                      // not a method of this corpus: an all-pad bag
        for (int j = tid; j < L; j += 256) { rs[j] = 0; rp[j] = 0; re[j] = 0; }
        if (label && tid == 0) label[b] = 0;
        return;
    }
    if (label && tid == 0) label[b] = item_labels ? item_labels[item] : 0;
    const long long lo = offsets[item];
    const long long n = offsets[item + 1] - lo;
    auto emit = [&](int pos, long long j) {                 // dataset_builder.py:135-143
        const int *c = ctx + (lo + j) * 3;
        long long s = c[0], p = c[1], e = c[2];
        if (s == method_token) s = question_token;
        if (e == method_token) e = question_token;
        rs[pos] = s; rp[pos] = p; re[pos] = e;
    };
    if (n <= L) {                                            // everything, stored order, zero suffix (:145-147)
        for (int j = tid; j < L; j += 256) {
            if (j < n) emit(j, j);
            else { rs[j] = 0; rp[j] = 0; re[j] = 0; }
        }
        return;
    }
    // ---- n > L: the L smallest (key, j).  Radix select of the L-th smallest key, most significant byte first.
    const unsigned long long base = bb_mix64(seed ^ ((unsigned long long)item * 0xD1B54A32D192ED03ull));
    if (tid == 0) { s_prefix = 0u; s_k = (unsigned)L; }
    unsigned mask = 0u;
    for (int pass = 3; pass >= 0; --pass) {
        hist[tid] = 0u;
        __syncthreads();
        const unsigned prefix = s_prefix;
        for (long long j = tid; j < n; j += 256) {
            const unsigned key = bb_key(base, j);
            if ((key & mask) == prefix) atomicAdd(&hist[(key >> (8 * pass)) & 255u], 1u);
        }
        __syncthreads();
        if (tid == 0) {
            unsigned k = s_k, cum = 0u, d = 0u;
            for (; d < 255u; ++d) {
                if (cum + hist[d] >= k) break;
                cum += hist[d];
            }
            s_k = k - cum;                                   // rank of the wanted key inside bucket d
            s_prefix = prefix | (d << (8 * pass));
        }
        mask |= 0xFFu << (8 * pass);
        __syncthreads();
    }
    const unsigned T = s_prefix;                             // key of the L-th smallest element
    const int need_eq = (int)s_k;                            // how many of the keys == T belong to the L smallest
    int base_pos = 0, base_eq = 0;
    for (long long j0 = 0; j0 < n; j0 += 256) {              // compaction in stored order
        const long long j = j0 + tid;
        const unsigned key = j < n ? bb_key(base, j) : 0xFFFFFFFFu;
        const int is_eq = (j < n && key == T) ? 1 : 0;
        int tot_eq, tot_take;
        const int eq_rank = base_eq + bb_block_scan(is_eq, s_warp, &tot_eq);
        const int take = (j < n && (key < T || (is_eq && eq_rank < need_eq))) ? 1 : 0;
        const int pos = base_pos + bb_block_scan(take, s_warp, &tot_take);
        if (take) emit(pos, j);
        base_eq += tot_eq; base_pos += tot_take;
    }
}

// ---- variable-name task ---------------------------------------------------------------------------------------------
constexpr int BB_MAX_VARS = 2048;      // |variable_indexes| (dataset/: 62, top11: 390)

// context c (start, path, end) belongs to the bag of variable v when its start or end is v.
// The count kernel and the builder both call this: a disagreement would silently give a bag of another length.
__device__ __forceinline__ bool bb_var_match(const int *c, long long v) { return c[0] == v || c[2] == v; }

// one warp per unit: counts[u] = the number of contexts of unit_item[u] that match unit_var[u] (0 for an unknown item)
__global__ void __launch_bounds__(256)
count_unit_contexts_kernel(const long long *__restrict__ offsets, const int *__restrict__ ctx, long long n_items,
                           const long long *__restrict__ unit_item, const long long *__restrict__ unit_var,
                           long long n_units, long long *__restrict__ counts)
{
    const long long u = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (u >= n_units) return;
    const long long item = unit_item[u];
    long long cnt = 0;
    if (item >= 0 && item < n_items) {
        const long long lo = offsets[item], n = offsets[item + 1] - lo, v = unit_var[u];
        for (long long j = lane; j < n; j += 32) cnt += bb_var_match(ctx + (lo + j) * 3, v) ? 1 : 0;
    }
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) counts[u] = cnt;
}

// PACKED: bag b goes to rows bag_off[b] .. bag_off[b+1]-1 (its length: min(n_match, L), 1 for a unit without a match or
// an unknown unit) instead of row b of the [B, L] tensors.  The selection still runs on L = max_path_length.
template <bool PACKED = false>
__global__ void __launch_bounds__(256)
build_batch_vars_kernel(const long long *__restrict__ offsets, const int *__restrict__ ctx, long long n_items,
                        const long long *__restrict__ unit_item, const long long *__restrict__ unit_var,
                        const long long *__restrict__ unit_label, long long n_units,
                        const long long *__restrict__ unit_ids, int L, unsigned long long seed, long long question_token,
                        const int *__restrict__ var_pos, long long T, const long long *__restrict__ variable_indexes,
                        int n_vars, int shuffle,
                        long long *__restrict__ starts, long long *__restrict__ paths, long long *__restrict__ ends,
                        long long *__restrict__ label, const long long *__restrict__ bag_off)
{
    __shared__ unsigned hist[256];
    __shared__ int s_warp[8];
    __shared__ unsigned s_prefix, s_k;
    __shared__ int s_nmatch;
    __shared__ unsigned s_vkey[BB_MAX_VARS];
    __shared__ unsigned short s_sigma[BB_MAX_VARS];
    const int b = blockIdx.x, tid = threadIdx.x;
    const long long unit = unit_ids[b];
    const long long row0 = PACKED ? bag_off[b] : (long long)b * L;
    long long *rs = starts + row0, *rp = paths + row0, *re = ends + row0;
    int cap = L;                                             // rows this bag may write
    if (PACKED) {                                            // the host-computed length, clamped into [0, L]
        const long long len = bag_off[b + 1] - row0;
        cap = len < 0 ? 0 : (len > L ? L : (int)len);
    }
    const long long item = (unit >= 0 && unit < n_units) ? unit_item[unit] : -1;
    if (item < 0 || item >= n_items) {                      // not a unit of this corpus: an all-pad bag
        for (int j = tid; j < cap; j += 256) { rs[j] = 0; rp[j] = 0; re[j] = 0; }
        if (label && tid == 0) label[b] = 0;
        return;
    }
    const long long v = unit_var[unit];
    if (label && tid == 0) label[b] = unit_label ? unit_label[unit] : 0;
    const long long lo = offsets[item];
    const long long n = offsets[item + 1] - lo;
    // per-item permutation of the variable indexes (dataset_builder.py:166-168): position i of `variable_indexes` maps to
    // variable_indexes[sigma(i)], sigma = argsort of the keys hash(seed, item, i) (ties by i)
    const bool permute = shuffle != 0 && var_pos != nullptr && n_vars > 1;
    if (permute) {
        const unsigned long long vbase = bb_mix64(seed ^ 0xA5A5A5A55A5A5A5Aull ^ ((unsigned long long)item * 0xD1B54A32D192ED03ull));
        for (int i = tid; i < n_vars; i += 256) s_vkey[i] = bb_key(vbase, i);
        __syncthreads();
        for (int i = tid; i < n_vars; i += 256) {
            const unsigned ki = s_vkey[i];
            int rank = 0;
            for (int j = 0; j < n_vars; ++j) { const unsigned kj = s_vkey[j]; rank += (kj < ki || (kj == ki && j < i)) ? 1 : 0; }
            s_sigma[rank] = (unsigned short)i;
        }
        __syncthreads();
    }
    auto remap = [&](long long t) -> long long {            // dataset_builder.py:181-184 / :190-193
        if (t == v) return question_token;
        if (permute && t >= 0 && t < T) {
            const int pos = var_pos[t];
            if (pos >= 0) return variable_indexes[s_sigma[pos]];
        }
        return t;
    };
    auto match = [&](long long j) { return bb_var_match(ctx + (lo + j) * 3, v); };
    auto emit = [&](int pos, long long j) {
        const int *c = ctx + (lo + j) * 3;
        rs[pos] = remap(c[0]); rp[pos] = c[1]; re[pos] = remap(c[2]);
    };
    // ---- number of matching contexts
    if (tid == 0) s_nmatch = 0;
    __syncthreads();
    {
        int cnt = 0;
        for (long long j = tid; j < n; j += 256) cnt += match(j) ? 1 : 0;
        for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        if ((tid & 31) == 0 && cnt) atomicAdd(&s_nmatch, cnt);
    }
    __syncthreads();
    const int n_match = s_nmatch;
    unsigned Tkey = 0xFFFFFFFFu;
    int need_eq = 0x7fffffff;
    const unsigned long long base = bb_mix64(seed ^ ((unsigned long long)item * 0xD1B54A32D192ED03ull) ^
                                             ((unsigned long long)v * 0x9E3779B97F4A7C15ull));
    if (n_match > L) {                                       // radix select of the L-th smallest key among the matches
        if (tid == 0) { s_prefix = 0u; s_k = (unsigned)L; }
        unsigned mask = 0u;
        for (int pass = 3; pass >= 0; --pass) {
            hist[tid] = 0u;
            __syncthreads();
            const unsigned prefix = s_prefix;
            for (long long j = tid; j < n; j += 256) {
                if (!match(j)) continue;
                const unsigned key = bb_key(base, j);
                if ((key & mask) == prefix) atomicAdd(&hist[(key >> (8 * pass)) & 255u], 1u);
            }
            __syncthreads();
            if (tid == 0) {
                unsigned k = s_k, cum = 0u, d = 0u;
                for (; d < 255u; ++d) {
                    if (cum + hist[d] >= k) break;
                    cum += hist[d];
                }
                s_k = k - cum;
                s_prefix = prefix | (d << (8 * pass));
            }
            mask |= 0xFFu << (8 * pass);
            __syncthreads();
        }
        Tkey = s_prefix; need_eq = (int)s_k;
    }
    int base_pos = 0, base_eq = 0;
    for (long long j0 = 0; j0 < n; j0 += 256) {              // compaction in stored order
        const long long j = j0 + tid;
        const bool m = j < n && match(j);
        const unsigned key = (m && n_match > L) ? bb_key(base, j) : 0u;
        const int is_eq = (m && n_match > L && key == Tkey) ? 1 : 0;
        int tot_eq, tot_take;
        const int eq_rank = base_eq + bb_block_scan(is_eq, s_warp, &tot_eq);
        const int take = (m && (n_match <= L || key < Tkey || (is_eq && eq_rank < need_eq))) ? 1 : 0;
        const int pos = base_pos + bb_block_scan(take, s_warp, &tot_take);
        if (take && (!PACKED || pos < cap)) emit(pos, j);
        base_eq += tot_eq; base_pos += tot_take;
    }
    const int filled = n_match < L ? n_match : L;
    for (int j = filled + tid; j < cap; j += 256) { rs[j] = 0; rp[j] = 0; re[j] = 0; }   // pad_inputs (:212-219)
}

}  // namespace c2v

using namespace c2v;

extern "C" int c2v_build_batch(const int64_t *offsets, const int32_t *contexts, int64_t n_items,
                               const int64_t *item_ids, const int64_t *item_labels, int32_t B, int32_t L,
                               uint64_t seed, int64_t method_token, int64_t question_token, int64_t *starts,
                               int64_t *paths, int64_t *ends, int64_t *label, void *stream)
{
    if (!offsets || !contexts || !item_ids || !starts || !paths || !ends || n_items < 1 || B < 1 || L < 1) {
        set_error("c2v_build_batch: bad argument");
        return C2V_EINVAL;
    }
    build_batch_kernel<<<(unsigned)B, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const long long *>(offsets), contexts, n_items, reinterpret_cast<const long long *>(item_ids),
        reinterpret_cast<const long long *>(item_labels), L, seed, method_token, question_token,
        reinterpret_cast<long long *>(starts), reinterpret_cast<long long *>(paths), reinterpret_cast<long long *>(ends),
        reinterpret_cast<long long *>(label), nullptr);
    C2V_LAUNCH_OK("build_batch_kernel");
    return C2V_OK;
}

extern "C" int c2v_build_batch_packed(const int64_t *offsets, const int32_t *contexts, int64_t n_items,
                                      const int64_t *item_ids, const int64_t *item_labels, int32_t B, int32_t L,
                                      uint64_t seed, int64_t method_token, int64_t question_token, const int64_t *bag_offsets,
                                      int64_t *starts, int64_t *paths, int64_t *ends, int64_t *label, void *stream)
{
    if (!offsets || !contexts || !item_ids || !bag_offsets || !starts || !paths || !ends || n_items < 1 || B < 1 || L < 1) {
        set_error("c2v_build_batch_packed: bad argument (NULL pointer, n_items < 1, B < 1 or L < 1)");
        return C2V_EINVAL;
    }
    build_batch_kernel<true><<<(unsigned)B, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const long long *>(offsets), contexts, n_items, reinterpret_cast<const long long *>(item_ids),
        reinterpret_cast<const long long *>(item_labels), L, seed, method_token, question_token,
        reinterpret_cast<long long *>(starts), reinterpret_cast<long long *>(paths), reinterpret_cast<long long *>(ends),
        reinterpret_cast<long long *>(label), reinterpret_cast<const long long *>(bag_offsets));
    C2V_LAUNCH_OK("build_batch_kernel<packed>");
    return C2V_OK;
}

// argument checks of both variable-name builders, before any CUDA call
static int vars_args_ok(const char *fn, const int64_t *offsets, const int32_t *contexts, int64_t n_items,
                        const int64_t *unit_item, const int64_t *unit_var, int64_t n_units, const int64_t *unit_ids,
                        int32_t B, int32_t L, const int32_t *var_pos, const int64_t *variable_indexes, int32_t n_vars,
                        int32_t shuffle_variable_indexes, const int64_t *starts, const int64_t *paths, const int64_t *ends)
{
    if (!offsets || !contexts || !unit_item || !unit_var || !unit_ids || !starts || !paths || !ends || n_items < 1 ||
        n_units < 1 || B < 1 || L < 1) {
        set_error("%s: bad argument", fn);
        return C2V_EINVAL;
    }
    if (shuffle_variable_indexes && (!var_pos || !variable_indexes || n_vars < 0)) {
        set_error("%s: shuffle_variable_indexes needs var_pos and variable_indexes", fn);
        return C2V_EINVAL;
    }
    if (n_vars > BB_MAX_VARS) {
        set_error("%s: %d variable indexes (max %d)", fn, n_vars, BB_MAX_VARS);
        return C2V_EUNSUPPORTED;
    }
    return C2V_OK;
}

extern "C" int c2v_build_batch_vars(const int64_t *offsets, const int32_t *contexts, int64_t n_items,
                                    const int64_t *unit_item, const int64_t *unit_var, const int64_t *unit_label,
                                    int64_t n_units, const int64_t *unit_ids, int32_t B, int32_t L, uint64_t seed,
                                    int64_t question_token, const int32_t *var_pos, int64_t terminal_count,
                                    const int64_t *variable_indexes, int32_t n_vars, int32_t shuffle_variable_indexes,
                                    int64_t *starts, int64_t *paths, int64_t *ends, int64_t *label, void *stream)
{
    const int rc = vars_args_ok("c2v_build_batch_vars", offsets, contexts, n_items, unit_item, unit_var, n_units, unit_ids,
                                B, L, var_pos, variable_indexes, n_vars, shuffle_variable_indexes, starts, paths, ends);
    if (rc != C2V_OK) return rc;
    build_batch_vars_kernel<<<(unsigned)B, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const long long *>(offsets), contexts, n_items, reinterpret_cast<const long long *>(unit_item),
        reinterpret_cast<const long long *>(unit_var), reinterpret_cast<const long long *>(unit_label), n_units,
        reinterpret_cast<const long long *>(unit_ids), L, seed, question_token, var_pos, terminal_count,
        reinterpret_cast<const long long *>(variable_indexes), n_vars, shuffle_variable_indexes,
        reinterpret_cast<long long *>(starts), reinterpret_cast<long long *>(paths), reinterpret_cast<long long *>(ends),
        reinterpret_cast<long long *>(label), nullptr);
    C2V_LAUNCH_OK("build_batch_vars_kernel");
    return C2V_OK;
}

extern "C" int c2v_build_batch_vars_packed(const int64_t *offsets, const int32_t *contexts, int64_t n_items,
                                           const int64_t *unit_item, const int64_t *unit_var, const int64_t *unit_label,
                                           int64_t n_units, const int64_t *unit_ids, int32_t B, int32_t L, uint64_t seed,
                                           int64_t question_token, const int32_t *var_pos, int64_t terminal_count,
                                           const int64_t *variable_indexes, int32_t n_vars,
                                           int32_t shuffle_variable_indexes, const int64_t *bag_offsets, int64_t *starts,
                                           int64_t *paths, int64_t *ends, int64_t *label, void *stream)
{
    if (!bag_offsets) { set_error("c2v_build_batch_vars_packed: bad argument (bag_offsets is NULL)"); return C2V_EINVAL; }
    const int rc = vars_args_ok("c2v_build_batch_vars_packed", offsets, contexts, n_items, unit_item, unit_var, n_units,
                                unit_ids, B, L, var_pos, variable_indexes, n_vars, shuffle_variable_indexes, starts, paths,
                                ends);
    if (rc != C2V_OK) return rc;
    build_batch_vars_kernel<true><<<(unsigned)B, 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const long long *>(offsets), contexts, n_items, reinterpret_cast<const long long *>(unit_item),
        reinterpret_cast<const long long *>(unit_var), reinterpret_cast<const long long *>(unit_label), n_units,
        reinterpret_cast<const long long *>(unit_ids), L, seed, question_token, var_pos, terminal_count,
        reinterpret_cast<const long long *>(variable_indexes), n_vars, shuffle_variable_indexes,
        reinterpret_cast<long long *>(starts), reinterpret_cast<long long *>(paths), reinterpret_cast<long long *>(ends),
        reinterpret_cast<long long *>(label), reinterpret_cast<const long long *>(bag_offsets));
    C2V_LAUNCH_OK("build_batch_vars_kernel<packed>");
    return C2V_OK;
}

extern "C" int c2v_count_unit_contexts(const int64_t *offsets, const int32_t *contexts, int64_t n_items,
                                       const int64_t *unit_item, const int64_t *unit_var, int64_t n_units, int64_t *counts,
                                       void *stream)
{
    if (!offsets || !contexts || !unit_item || !unit_var || !counts || n_items < 1 || n_units < 1) {
        set_error("c2v_count_unit_contexts: bad argument (NULL pointer, n_items < 1 or n_units < 1)");
        return C2V_EINVAL;
    }
    count_unit_contexts_kernel<<<(unsigned)((n_units + 7) / 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<const long long *>(offsets), contexts, n_items, reinterpret_cast<const long long *>(unit_item),
        reinterpret_cast<const long long *>(unit_var), n_units, reinterpret_cast<long long *>(counts));
    C2V_LAUNCH_OK("count_unit_contexts_kernel");
    return C2V_OK;
}

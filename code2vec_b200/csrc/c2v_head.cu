// c2v_head.cu -- label head next to the encode path, CUDA-core versions:
//   generic strided fp32 GEMM (+bias)            model.py:83 and its backward
//   angular-margin head                          model.py:71-80
//   fused log_softmax + NLL + argmax (+dlogits)  main.py:251-264, main.py:285
#include "c2v_common.cuh"

namespace c2v {

// ------------------------------------------------------------------------------------
// C[m,n] (+)= sum_k A(m,k) B(k,n) + bias[n] ; 64x64 tile, 16-wide k step, 4x4 per thread.
// Strides are in elements so NN / NT / TN all map onto it.
// ------------------------------------------------------------------------------------
constexpr int GT = 64, GK = 16;

// gridDim.z > 1: split-K, each z-slice handles k_per_split of K and adds its partial tile with atomics
// (the launcher zero-fills C first unless it accumulates).
__global__ void __launch_bounds__(256)
sgemm_kernel(int M, int N, int K, const float *__restrict__ A, long long a_sm, long long a_sk,
             const float *__restrict__ B, long long b_sk, long long b_sn,
             const float *__restrict__ bias, float *__restrict__ C, long long c_sm, int accumulate,
             int k_per_split)
{
    __shared__ float As[GK][GT + 4];
    __shared__ float Bs[GK][GT + 4];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.y * GT, n0 = blockIdx.x * GT;
    float acc[4][4] = {};
    const int k_begin = blockIdx.z * k_per_split;
    const int k_end = (k_begin + k_per_split < K) ? k_begin + k_per_split : K;
    const bool split = gridDim.z > 1;
    K = k_end;
    for (int k0 = k_begin; k0 < k_end; k0 += GK) {
        for (int i = tid; i < GT * GK; i += 256) {
            // choose the faster-varying index along the contiguous dimension of each operand
            int am, ak, bk, bn;
            if (a_sk == 1) { ak = i % GK; am = i / GK; } else { am = i % GT; ak = i / GT; }
            if (b_sn == 1) { bn = i % GT; bk = i / GT; } else { bk = i % GK; bn = i / GK; }
            const int gm = m0 + am, gk = k0 + ak;
            As[ak][am] = (gm < M && gk < K) ? A[gm * a_sm + gk * a_sk] : 0.0f;
            const int gn = n0 + bn, gk2 = k0 + bk;
            Bs[bk][bn] = (gn < N && gk2 < K) ? B[gk2 * b_sk + gn * b_sn] : 0.0f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < GK; ++k) {
            const float4 av = *reinterpret_cast<const float4 *>(&As[k][ty * 4]);
            const float4 bv = *reinterpret_cast<const float4 *>(&Bs[k][tx * 4]);
            const float a4[4] = {av.x, av.y, av.z, av.w};
            const float b4[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a4[i], b4[j], acc[i][j]);
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int gm = m0 + ty * 4 + i;
        if (gm >= M) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int gn = n0 + tx * 4 + j;
            if (gn >= N) continue;
            float v = acc[i][j] + ((bias && blockIdx.z == 0) ? bias[gn] : 0.0f);
            float *dst = C + gm * c_sm + gn;
            if (split) atomicAdd(dst, v);
            else *dst = accumulate ? *dst + v : v;
        }
    }
}

int launch_sgemm(int M, int N, int K, const float *A, long long a_sm, long long a_sk, const float *B,
                 long long b_sk, long long b_sn, const float *bias, float *C, long long c_sm,
                 bool accumulate, cudaStream_t st)
{
    if (M <= 0 || N <= 0) return C2V_OK;
    const int gx = (N + GT - 1) / GT, gy = (M + GT - 1) / GT;
    // few output tiles but a long reduction (d_cv = d_out . W_out: 32 tiles, K = label_count): split K
    int splits = 1;
    if (gx * gy < 128 && K >= 1024) {
        splits = 592 / (gx * gy);
        if (splits > K / 256) splits = K / 256;
        if (splits < 1) splits = 1;
    }
    int k_per = (K + splits - 1) / splits;
    k_per = (k_per + GK - 1) / GK * GK;
    splits = (K + k_per - 1) / k_per;
    if (splits > 1 && !accumulate) {
        if (c_sm == N) C2V_CUDA_OK(cudaMemsetAsync(C, 0, (size_t)M * N * sizeof(float), st));
        else C2V_CUDA_OK(cudaMemset2DAsync(C, (size_t)c_sm * sizeof(float), 0, (size_t)N * sizeof(float), M, st));
    }
    dim3 grid(gx, gy, splits);
    sgemm_kernel<<<grid, 256, 0, st>>>(M, N, K, A, a_sm, a_sk, B, b_sk, b_sn, bias, C, c_sm,
                                       accumulate ? 1 : 0, k_per);
    C2V_LAUNCH_OK("sgemm_kernel");
    return C2V_OK;
}

// ------------------------------------------------------------------------------------
// angular-margin head (model.py:71-80): one warp per (bag, class) pair group.
// ------------------------------------------------------------------------------------
__global__ void row_inv_norm_kernel(const float *__restrict__ X, long long rows, int H,
                                    float *__restrict__ inv)
{
    const long long r = (long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
    if (r >= rows) return;
    const int lane = threadIdx.x & 31;
    float s = 0.0f;
    for (int c = lane; c < H; c += 32) { const float v = X[r * H + c]; s = fmaf(v, v, s); }
    s = warp_sum(s);
    if (lane == 0) inv[r] = 1.0f / fmaxf(sqrtf(s), 1e-12f);   // F.normalize eps
}

// inv[r] = 1 / max(|X[r]|, 1e-12) for the rows of X [rows, H]
int launch_row_inv_norm(const float *X, long long rows, int H, float *inv, cudaStream_t st)
{
    if (rows <= 0) return C2V_OK;
    row_inv_norm_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(X, rows, H, inv);
    C2V_LAUNCH_OK("row_inv_norm_kernel");
    return C2V_OK;
}

// d[r] -= inv[r]^2 (x[r] . d[r]) x[r]: the gradient through F.normalize, given d = the gradient w.r.t. the unnormalised
// dot's operand (one warp per row of [rows, H]).  Exact for the angular head: sum_c dcos cos = sum_c G dot = x_r . (G W)_r.
__global__ void __launch_bounds__(256)
angular_project_rows_kernel(float *__restrict__ d, const float *__restrict__ x, const float *__restrict__ inv, long long rows,
                            int H)
{
    const long long r = (long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
    if (r >= rows) return;
    const int lane = threadIdx.x & 31;
    const float *xr = x + r * H;
    float *dr = d + r * H;
    float s = 0.0f;
    for (int c = lane; c < H; c += 32) s = fmaf(xr[c], dr[c], s);
    s = warp_sum(s);
    const float f = -inv[r] * inv[r] * s;
    for (int c = lane; c < H; c += 32) dr[c] = fmaf(f, xr[c], dr[c]);
}

int launch_angular_project(float *d, const float *x, const float *inv, long long rows, int H, cudaStream_t st)
{
    if (rows <= 0) return C2V_OK;
    angular_project_rows_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(d, x, inv, rows, H);
    C2V_LAUNCH_OK("angular_project_rows_kernel");
    return C2V_OK;
}

__global__ void angular_epilogue_kernel(float *__restrict__ out, const float *__restrict__ inv_cv,
                                        const float *__restrict__ inv_w,
                                        const long long *__restrict__ label, int B, long long C,
                                        float cos_m, float sin_m, float inv_temp, float *__restrict__ cos_out)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * C) return;
    const int b = (int)(i / C);
    const long long c = i % C;
    const float cosv = out[i] * inv_cv[b] * inv_w[c];
    if (cos_out) cos_out[i] = cosv;                        // kept for the backward (training)
    const float sinv = sqrtf(1.0f - cosv * cosv);
    float phi = cosv * cos_m - sinv * sin_m;
    if (!(cosv > 0.0f)) phi = cosv;
    out[i] = (label[b] == c ? phi : cosv) * inv_temp;
}

int launch_angular(const c2v_dims *d, const c2v_params *p, const float *cv, const long long *label,
                   int B, float margin, float inverse_temp, float *out, float *scratch,
                   cudaStream_t st, float *cos_out)
{
    const int H = d->encode;
    const long long C = d->label_count;
    float *inv_cv = scratch, *inv_w = scratch + B;
    int rc = launch_row_inv_norm(cv, B, H, inv_cv, st);
    if (rc != C2V_OK) return rc;
    rc = launch_row_inv_norm(p->output_weight, C, H, inv_w, st);
    if (rc != C2V_OK) return rc;
    rc = launch_sgemm(B, (int)C, H, cv, H, 1, p->output_weight, 1, H, nullptr, out, C, false, st);
    if (rc != C2V_OK) return rc;
    const long long n = (long long)B * C;
    angular_epilogue_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
        out, inv_cv, inv_w, label, B, C, cosf(margin), sinf(margin), inverse_temp, cos_out);
    C2V_LAUNCH_OK("angular_epilogue_kernel");
    return C2V_OK;
}

// ------------------------------------------------------------------------------------
// backward of the angular-margin head (autograd of model.py:71-80):
//   out = s (onehot phi + (1 - onehot) cos),  phi = cos > 0 ? cos cos_m - sin sin_m : cos,  sin = sqrt(1 - cos^2),
//   cos[b,c] = dot[b,c] icv[b] iw[c],  dot = cv . W^T,  icv = 1 / max(|cv_b|, 1e-12),  iw likewise (F.normalize)
//   dcos = s d_out (target column with cos > 0: x (cos_m + sin_m cos / sin));   G = dcos icv iw  (= d loss / d dot)
//   d_cv = G . W   - icv_b^2 (sum_c dcos cos) cv_b ;   d_W = G^T . cv - iw_c^2 (sum_b dcos cos) W_c
// angular_dcos_kernel overwrites d_out with G and accumulates the two correction sums; the GEMMs are launch_sgemm.
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
angular_dcos_kernel(float *__restrict__ g, const float *__restrict__ cosv, const float *__restrict__ inv_cv,
                    const float *__restrict__ inv_w, const long long *__restrict__ label, int B, long long C,
                    float cos_m, float sin_m, float inv_temp, float *__restrict__ rowsum, float *__restrict__ colsum)
{
    const int b = blockIdx.y;
    const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    float pc = 0.0f;
    if (c < C) {
        const size_t i = (size_t)b * C + c;
        const float co = cosv[i];
        float dcos = g[i] * inv_temp;
        if (label[b] == c && co > 0.0f) dcos *= cos_m + sin_m * co / sqrtf(1.0f - co * co);
        g[i] = dcos * inv_cv[b] * inv_w[c];
        pc = dcos * co;
        if (pc != 0.0f) atomicAdd(colsum + c, pc);
    }
    pc = warp_sum(pc);
    if ((threadIdx.x & 31) == 0 && pc != 0.0f) atomicAdd(rowsum + b, pc);
}
__global__ void angular_fix_rows_kernel(float *__restrict__ d, const float *__restrict__ x, const float *__restrict__ inv,
                                        const float *__restrict__ sums, long long rows, int H)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows * H) return;
    const long long r = i / H;
    d[i] = fmaf(-inv[r] * inv[r] * sums[r], x[i], d[i]);
}

int launch_angular_backward(const c2v_dims *d, const c2v_params *p, const float *cv, const long long *label, int B,
                            float margin, float inverse_temp, const float *cosine, const float *inv_cv, const float *inv_w,
                            float *d_out_inplace, float *d_cv, float *d_w, float *sums, cudaStream_t st)
{
    const int H = d->encode;
    const long long C = d->label_count;
    float *rowsum = sums, *colsum = sums + B;
    C2V_CUDA_OK(cudaMemsetAsync(sums, 0, (size_t)(B + C) * sizeof(float), st));
    angular_dcos_kernel<<<dim3((unsigned)((C + 255) / 256), (unsigned)B), 256, 0, st>>>(
        d_out_inplace, cosine, inv_cv, inv_w, label, B, C, cosf(margin), sinf(margin), inverse_temp, rowsum, colsum);
    C2V_LAUNCH_OK("angular_dcos_kernel");
    int rc = C2V_OK;
    if (d_cv) {
        rc = launch_sgemm(B, H, (int)C, d_out_inplace, C, 1, p->output_weight, H, 1, nullptr, d_cv, H, false, st);
        if (rc != C2V_OK) return rc;
        const long long n = (long long)B * H;
        angular_fix_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_cv, cv, inv_cv, rowsum, B, H);
        C2V_LAUNCH_OK("angular_fix_rows_kernel");
    }
    if (d_w) {
        rc = launch_sgemm((int)C, H, B, d_out_inplace, 1, C, cv, H, 1, nullptr, d_w, H, false, st);
        if (rc != C2V_OK) return rc;
        const long long n = C * H;
        angular_fix_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(d_w, p->output_weight, inv_w, colsum, C, H);
        C2V_LAUNCH_OK("angular_fix_rows_kernel");
    }
    return rc;
}

// ------------------------------------------------------------------------------------
// log_softmax + mean NLL + argmax (+ d_outputs) in one pass over the logits per row.
// One CTA per bag; loss is accumulated with one atomicAdd per bag (pre-zeroed by the host).
// ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
loss_argmax_kernel(const float *__restrict__ out, const long long *__restrict__ label, int B,
                   long long C, float *__restrict__ loss, long long *__restrict__ argmax,
                   float *__restrict__ maxval, float *__restrict__ d_out)
{
    __shared__ float s_val[8];
    __shared__ long long s_idx[8];
    __shared__ float s_sum[8];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float *r = out + (size_t)b * C;
    float mx = -INFINITY; long long am = 0x7fffffffffffffffLL;
    for (long long c = tid; c < C; c += 256) {
        const float v = r[c];
        if (v > mx) { mx = v; am = c; }         // strided scan keeps the first max per thread
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, mx, o);
        const long long oi = __shfl_xor_sync(0xffffffffu, am, o);
        if (ov > mx || (ov == mx && oi < am)) { mx = ov; am = oi; }   // torch.max: first max wins
    }
    if (lane == 0) { s_val[warp] = mx; s_idx[warp] = am; }
    __syncthreads();
    mx = s_val[0]; am = s_idx[0];
    for (int w = 1; w < 8; ++w)
        if (s_val[w] > mx || (s_val[w] == mx && s_idx[w] < am)) { mx = s_val[w]; am = s_idx[w]; }
    if (!(loss && label) && !(d_out && label)) {          // arg-max only: no second pass over the logits
        if (tid == 0) { if (argmax) argmax[b] = am; if (maxval) maxval[b] = mx; }
        return;
    }
    float s = 0.0f;
    for (long long c = tid; c < C; c += 256) s += __expf(r[c] - mx);
    s = warp_sum(s);
    if (lane == 0) s_sum[warp] = s;
    __syncthreads();
    s = 0.0f;
    for (int w = 0; w < 8; ++w) s += s_sum[w];
    if (tid == 0) {
        if (argmax) argmax[b] = am;
        if (maxval) maxval[b] = mx;
        if (loss && label) atomicAdd(loss, (mx + logf(s) - r[label[b]]) / (float)B);
    }
    if (d_out && label) {
        const float inv = 1.0f / s, invB = 1.0f / (float)B;
        const long long lab = label[b];
        float *g = d_out + (size_t)b * C;
        for (long long c = tid; c < C; c += 256)
            g[c] = (__expf(r[c] - mx) * inv - (c == lab ? 1.0f : 0.0f)) * invB;
    }
}

int launch_loss_argmax(const float *out, const long long *label, int B, long long C, float *loss,
                       long long *argmax, float *maxval, float *d_out, cudaStream_t st)
{
    if (loss) C2V_CUDA_OK(cudaMemsetAsync(loss, 0, sizeof(float), st));
    loss_argmax_kernel<<<B, 256, 0, st>>>(out, label, B, C, loss, argmax, maxval, d_out);
    C2V_LAUNCH_OK("loss_argmax_kernel");
    return C2V_OK;
}

// column sums of d_out [B, C] -> d_bias [C]
__global__ void colsum_kernel(const float *__restrict__ X, int B, long long C, float *__restrict__ out)
{
    const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= C) return;
    float s = 0.0f;
    for (int b = 0; b < B; ++b) s += X[(size_t)b * C + c];
    out[c] = s;
}
int launch_colsum(const float *X, int B, long long C, float *out, cudaStream_t st)
{
    colsum_kernel<<<(unsigned)((C + 255) / 256), 256, 0, st>>>(X, B, C, out);
    C2V_LAUNCH_OK("colsum_kernel");
    return C2V_OK;
}

}  // namespace c2v

// c2v_session.cu -- host-buffer entry points: the call a reference-side user with CPU
// tensors makes (main.py:166-169 `.to(device)` x4, model.forward main.py:282, torch.max
// main.py:285, then results read back on the host).
//
// Three streams and kSlots staging slots: the int64 index upload of batch i+1 runs on the copy
// stream while batch i computes, and the results of batch i drain on the download stream
// while batch i+1 computes.  With two slots the rate is capped at half of one batch's upload + compute + download;
// four slots let it reach max(upload, compute).
#include <cstring>
#include <new>

#include "c2v_common.cuh"

using namespace c2v;

static const int kSlots = 4;

struct c2v_session {
    int device;
    c2v_dims dims;
    int max_B, L;
    cudaStream_t s_up, s_run, s_down;
    struct Slot {
        long long *d_idx;      // starts | paths | ends | label | bag offsets (packed calls)
        float *d_cv, *d_att, *d_out, *d_score;
        long long *d_pred;
        void *ws_enc, *ws_lab;
        size_t ws_enc_bytes, ws_lab_bytes;
        long long *h_status;   // pinned
        cudaEvent_t up_done, run_done, down_done;
        bool busy;
        bool prepped;          // workspaces hold valid weight images (C2V_FLAG_REUSE_PREP)
        int64_t ticket;
    } slot[kSlots];
    int64_t next_ticket;
};

static void destroy_slot(c2v_session::Slot &s)
{
    cudaFree(s.d_idx); cudaFree(s.d_cv); cudaFree(s.d_att); cudaFree(s.d_out); cudaFree(s.d_score);
    cudaFree(s.d_pred); cudaFree(s.ws_enc); cudaFree(s.ws_lab);
    if (s.h_status) cudaFreeHost(s.h_status);
    if (s.up_done) cudaEventDestroy(s.up_done);
    if (s.run_done) cudaEventDestroy(s.run_done);
    if (s.down_done) cudaEventDestroy(s.down_done);
}

extern "C" {

int c2v_session_create(int device, const c2v_dims *d, int32_t max_B, int32_t L, c2v_session **out)
{
    if (!d || !out || max_B < 1 || L < 1) { set_error("c2v_session_create: bad argument"); return C2V_EINVAL; }
    C2V_CUDA_OK(cudaSetDevice(device));
    c2v_session *s = new (std::nothrow) c2v_session;
    if (!s) { set_error("out of host memory"); return C2V_EINVAL; }
    memset(s, 0, sizeof(*s));
    s->device = device; s->dims = *d; s->max_B = max_B; s->L = L;
    C2V_CUDA_OK(cudaStreamCreateWithFlags(&s->s_up, cudaStreamNonBlocking));
    C2V_CUDA_OK(cudaStreamCreateWithFlags(&s->s_run, cudaStreamNonBlocking));
    C2V_CUDA_OK(cudaStreamCreateWithFlags(&s->s_down, cudaStreamNonBlocking));
    const size_t n = (size_t)max_B * L;
    for (int i = 0; i < kSlots; ++i) {
        c2v_session::Slot &q = s->slot[i];
        // one slot serves padded and packed calls in any order: the packed workspace keeps the status word and the weight
        // images where the padded one has them and appends its row -> bag map, so REUSE_PREP stays valid across layouts
        const size_t ws_pad = c2v_encode_workspace_bytes(d, max_B, L);
        const size_t ws_packed = c2v_encode_packed_workspace_bytes(d, max_B, (int64_t)n);
        q.ws_enc_bytes = ws_pad > ws_packed ? ws_pad : ws_packed;
        q.ws_lab_bytes = c2v_label_workspace_bytes(d, max_B);
        C2V_CUDA_OK(cudaMalloc(&q.d_idx, (3 * n + max_B + max_B + 1) * sizeof(long long)));
        C2V_CUDA_OK(cudaMalloc(&q.d_cv, (size_t)max_B * d->encode * sizeof(float)));
        C2V_CUDA_OK(cudaMalloc(&q.d_att, n * sizeof(float)));
        C2V_CUDA_OK(cudaMalloc(&q.d_out, (size_t)max_B * d->label_count * sizeof(float)));
        C2V_CUDA_OK(cudaMalloc(&q.d_score, (size_t)max_B * sizeof(float)));
        C2V_CUDA_OK(cudaMalloc(&q.d_pred, (size_t)max_B * sizeof(long long)));
        C2V_CUDA_OK(cudaMalloc(&q.ws_enc, q.ws_enc_bytes));
        C2V_CUDA_OK(cudaMalloc(&q.ws_lab, q.ws_lab_bytes));
        C2V_CUDA_OK(cudaMallocHost(&q.h_status, 256));
        C2V_CUDA_OK(cudaEventCreateWithFlags(&q.up_done, cudaEventDisableTiming));
        C2V_CUDA_OK(cudaEventCreateWithFlags(&q.run_done, cudaEventDisableTiming));
        C2V_CUDA_OK(cudaEventCreateWithFlags(&q.down_done, cudaEventDisableTiming));
        q.ticket = -1;
    }
    *out = s;
    return C2V_OK;
}

void c2v_session_destroy(c2v_session *s)
{
    if (!s) return;
    cudaSetDevice(s->device);
    cudaDeviceSynchronize();
    for (int i = 0; i < kSlots; ++i) destroy_slot(s->slot[i]);
    cudaStreamDestroy(s->s_up); cudaStreamDestroy(s->s_run); cudaStreamDestroy(s->s_down);
    delete s;
}

// Both layouts once the arguments are checked: [B, L] (offsets == NULL, n = B * L) or packed (n = N contexts, host
// offsets [B + 1] already validated).
static int forward_host_impl(c2v_session *s, const c2v_params *p, const int64_t *starts, const int64_t *paths,
                             const int64_t *ends, const int64_t *offsets, const int64_t *label, int32_t B, size_t n,
                             float *outputs, float *code_vector, float *attention, int64_t *pred_label, float *pred_score,
                             int32_t algo, int64_t *ticket)
{
    C2V_CUDA_OK(cudaSetDevice(s->device));
    const int64_t t = s->next_ticket;
    c2v_session::Slot &q = s->slot[t % kSlots];
    if (q.busy) {   // the slot's previous batch must have fully drained
        C2V_CUDA_OK(cudaEventSynchronize(q.down_done));
        q.busy = false;
    }
    long long *d_s = q.d_idx, *d_p = q.d_idx + n, *d_e = q.d_idx + 2 * n, *d_l = q.d_idx + 3 * n, *d_off = d_l + B;
    C2V_CUDA_OK(cudaMemcpyAsync(d_s, starts, n * 8, cudaMemcpyHostToDevice, s->s_up));
    C2V_CUDA_OK(cudaMemcpyAsync(d_p, paths, n * 8, cudaMemcpyHostToDevice, s->s_up));
    C2V_CUDA_OK(cudaMemcpyAsync(d_e, ends, n * 8, cudaMemcpyHostToDevice, s->s_up));
    if (label) C2V_CUDA_OK(cudaMemcpyAsync(d_l, label, (size_t)B * 8, cudaMemcpyHostToDevice, s->s_up));
    if (offsets) C2V_CUDA_OK(cudaMemcpyAsync(d_off, offsets, ((size_t)B + 1) * 8, cudaMemcpyHostToDevice, s->s_up));
    C2V_CUDA_OK(cudaEventRecord(q.up_done, s->s_up));
    C2V_CUDA_OK(cudaStreamWaitEvent(s->s_run, q.up_done, 0));

    // weight images are per slot: honour the caller's reuse promise only once this slot has them
    const int base_algo = algo & 0xff;
    const int reuse = ((algo & C2V_FLAG_REUSE_PREP) && q.prepped) ? C2V_FLAG_REUSE_PREP : 0;
    int rc = offsets
        ? c2v_encode_forward_packed(&s->dims, p, (const int64_t *)d_s, (const int64_t *)d_p, (const int64_t *)d_e,
                                    (const int64_t *)d_off, B, (int64_t)n, s->L, nullptr, q.d_cv, q.d_att, nullptr, q.ws_enc,
                                    q.ws_enc_bytes, base_algo | reuse, s->s_run)
        : c2v_encode_forward(&s->dims, p, (const int64_t *)d_s, (const int64_t *)d_p, (const int64_t *)d_e, B, s->L, nullptr,
                             q.d_cv, q.d_att, q.ws_enc, q.ws_enc_bytes, base_algo | reuse, s->s_run);
    if (rc != C2V_OK) return rc;
    const bool want_head = outputs || pred_label || pred_score;
    // the [B, C] logits are only materialised when the caller asked for them (or the fused arg-max cannot serve this shape):
    // the predict surface (code vector, attention, arg-max, score) never writes them
    float *logits_dst = (outputs || base_algo == C2V_ALGO_FFMA || !c2v_label_loss_supported(&s->dims, B)) ? q.d_out : nullptr;
    if (want_head) {
        if (!p->output_weight) { set_error("c2v_forward_host: output_weight is NULL"); return C2V_EINVAL; }
        rc = c2v_label_logits_argmax(&s->dims, p, q.d_cv, B, logits_dst, pred_label ? (int64_t *)q.d_pred : nullptr,
                                     pred_score ? q.d_score : nullptr, q.ws_lab, q.ws_lab_bytes,
                                     (base_algo == C2V_ALGO_FFMA ? C2V_ALGO_FFMA : C2V_ALGO_AUTO) | reuse, s->s_run);
        if (rc != C2V_OK) return rc;
        q.prepped = true;
    }
    C2V_CUDA_OK(cudaEventRecord(q.run_done, s->s_run));
    C2V_CUDA_OK(cudaStreamWaitEvent(s->s_down, q.run_done, 0));
    C2V_CUDA_OK(cudaMemcpyAsync(code_vector, q.d_cv, (size_t)B * s->dims.encode * 4, cudaMemcpyDeviceToHost, s->s_down));
    C2V_CUDA_OK(cudaMemcpyAsync(attention, q.d_att, n * 4, cudaMemcpyDeviceToHost, s->s_down));
    if (outputs)
        C2V_CUDA_OK(cudaMemcpyAsync(outputs, q.d_out, (size_t)B * s->dims.label_count * 4, cudaMemcpyDeviceToHost, s->s_down));
    if (pred_label) C2V_CUDA_OK(cudaMemcpyAsync(pred_label, q.d_pred, (size_t)B * 8, cudaMemcpyDeviceToHost, s->s_down));
    if (pred_score) C2V_CUDA_OK(cudaMemcpyAsync(pred_score, q.d_score, (size_t)B * 4, cudaMemcpyDeviceToHost, s->s_down));
    C2V_CUDA_OK(cudaMemcpyAsync(q.h_status, static_cast<const char *>(q.ws_enc) + 24, 8, cudaMemcpyDeviceToHost, s->s_down));   // published count
    C2V_CUDA_OK(cudaEventRecord(q.down_done, s->s_down));
    // (the next upload into this slot's d_idx happens kSlots batches later, after the host has
    //  waited on down_done above, so it cannot overtake this batch's kernels)
    q.busy = true;
    q.ticket = t;
    s->next_ticket = t + 1;
    *ticket = t;
    return C2V_OK;
}

int c2v_forward_host_async(c2v_session *s, const c2v_params *p, const int64_t *starts,
                           const int64_t *paths, const int64_t *ends, const int64_t *label,
                           int32_t B, float *outputs, float *code_vector, float *attention,
                           int64_t *pred_label, float *pred_score, int32_t algo, int64_t *ticket)
{
    if (!s || !p || !starts || !paths || !ends || !code_vector || !attention || !ticket) {
        set_error("c2v_forward_host: NULL argument");
        return C2V_EINVAL;
    }
    if (B < 1 || B > s->max_B) { set_error("c2v_forward_host: B=%d not in [1,%d]", B, s->max_B); return C2V_EINVAL; }
    return forward_host_impl(s, p, starts, paths, ends, nullptr, label, B, (size_t)B * s->L, outputs, code_vector, attention,
                             pred_label, pred_score, algo, ticket);
}

int c2v_forward_host_packed_async(c2v_session *s, const c2v_params *p, const int64_t *starts, const int64_t *paths,
                                  const int64_t *ends, const int64_t *offsets, const int64_t *label, int32_t B, int64_t N,
                                  float *outputs, float *code_vector, float *attention, int64_t *pred_label,
                                  float *pred_score, int32_t algo, int64_t *ticket)
{
    if (!s || !p || !starts || !paths || !ends || !offsets || !code_vector || !attention || !ticket) {
        set_error("c2v_forward_host_packed: NULL argument");
        return C2V_EINVAL;
    }
    if (B < 1 || B > s->max_B) { set_error("c2v_forward_host_packed: B=%d not in [1,%d]", B, s->max_B); return C2V_EINVAL; }
    // the offsets are host memory: check them here, before anything is copied or launched
    if (offsets[0] != 0) {
        set_error("c2v_forward_host_packed: offsets[0] = %lld, must be 0", (long long)offsets[0]);
        return C2V_EINVAL;
    }
    for (int32_t b = 0; b < B; ++b) {
        const int64_t len = offsets[b + 1] - offsets[b];
        if (len < 1 || len > s->L) {
            set_error("c2v_forward_host_packed: bag %d holds %lld contexts, must hold 1 .. %d", b, (long long)len, s->L);
            return C2V_EINVAL;
        }
    }
    if (offsets[B] != N) {
        set_error("c2v_forward_host_packed: offsets[B] = %lld != N = %lld", (long long)offsets[B], (long long)N);
        return C2V_EINVAL;
    }
    return forward_host_impl(s, p, starts, paths, ends, offsets, label, B, (size_t)N, outputs, code_vector, attention,
                             pred_label, pred_score, algo, ticket);
}

int c2v_session_wait(c2v_session *s, int64_t ticket)
{
    if (!s) { set_error("session is NULL"); return C2V_EINVAL; }
    c2v_session::Slot &q = s->slot[ticket % kSlots];
    if (q.ticket != ticket) { set_error("ticket %lld is not in flight", (long long)ticket); return C2V_EINVAL; }
    C2V_CUDA_OK(cudaEventSynchronize(q.down_done));
    q.busy = false;
    if (q.h_status[0] != 0) {
        set_error("index out of range in self (%lld indices)", q.h_status[0]);   // nn.Embedding's message
        return C2V_EINDEX;
    }
    return C2V_OK;
}

int c2v_forward_host(c2v_session *s, const c2v_params *p, const int64_t *starts, const int64_t *paths,
                     const int64_t *ends, const int64_t *label, int32_t B, float *outputs,
                     float *code_vector, float *attention, int64_t *pred_label, float *pred_score,
                     int32_t algo)
{
    int64_t t = 0;
    int rc = c2v_forward_host_async(s, p, starts, paths, ends, label, B, outputs, code_vector,
                                    attention, pred_label, pred_score, algo, &t);
    if (rc != C2V_OK) return rc;
    return c2v_session_wait(s, t);
}

int c2v_forward_host_packed(c2v_session *s, const c2v_params *p, const int64_t *starts, const int64_t *paths,
                            const int64_t *ends, const int64_t *offsets, const int64_t *label, int32_t B, int64_t N,
                            float *outputs, float *code_vector, float *attention, int64_t *pred_label, float *pred_score,
                            int32_t algo)
{
    int64_t t = 0;
    int rc = c2v_forward_host_packed_async(s, p, starts, paths, ends, offsets, label, B, N, outputs, code_vector, attention,
                                           pred_label, pred_score, algo, &t);
    if (rc != C2V_OK) return rc;
    return c2v_session_wait(s, t);
}

}  // extern "C"

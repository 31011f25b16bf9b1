// wb_dtw_kernel.cu -- see wb_dtw_kernel.cuh.  One CTA per (alignment head, token, request); written as block-synchronous phases (functions
// of (tid, nthreads) reading only what earlier phases wrote) like wb_vad.cu, so that the host can walk the same arithmetic (dtw_qk_emulated).
// The arithmetic of a (head, token) never depends on the other requests of the launch or on the K layout: results are batch-invariant.
#include <cmath>
#include <vector>
#include "wb_common.h"
#include "wb_dtw_kernel.cuh"

namespace wb {

#define DTW_HD __host__ __device__ __forceinline__
constexpr int DTW_THREADS = 256;
constexpr int DTW_MAX_CTX = 1536;

struct DtwScratch { float q16[64]; float s[DTW_MAX_CTX]; float red[DTW_THREADS]; float stat[2]; };

DTW_HD int dq_n_ctx(const DtwQkArgs & a, int r) { return a.req[4 * r + 3]; }
DTW_HD int dq_n_tok(const DtwQkArgs & a, int r) { return a.req[4 * r + 2]; }

DTW_HD void dq_load(int tid, int nt, DtwScratch & S, const DtwQkArgs & a, int e, int t, int r) {
    const float * q = a.q + ((size_t) a.head_cap[e] * a.cap_rows + a.req[4 * r] + t) * 64;
    for (int i = tid; i < 64; i += nt) S.q16[i] = __half2float(__float2half_rn(q[i]));
}
DTW_HD void dq_scores(int tid, int nt, DtwScratch & S, const DtwQkArgs & a, int e, int r) {
    const __half * K = a.k_cross + (size_t) a.req[4 * r + 1] * a.slot_stride + (size_t) a.head_layer[e] * a.layer_stride;
    size_t key_stride;
    if (a.k_head_major) { K += (size_t) a.head_index[e] * a.Tp * 64; key_stride = 64; }
    else                { K += (size_t) a.head_index[e] * 64;        key_stride = (size_t) a.d; }
    const int n_ctx = dq_n_ctx(a, r);
    float mx = -INFINITY;
    for (int j = tid; j < n_ctx; j += nt) {
        const __half * kr = K + (size_t) j * key_stride;
        float acc = 0.0f;
        for (int i = 0; i < 64; ++i) acc = fmaf(__half2float(kr[i]), S.q16[i], acc);
        const float v = acc * a.scale;
        S.s[j] = v; mx = fmaxf(mx, v);
    }
    S.red[tid] = mx;
}
DTW_HD void dq_max(int tid, int nt, DtwScratch & S) {
    if (tid == 0) { float m = -INFINITY; for (int i = 0; i < nt; ++i) m = fmaxf(m, S.red[i]); S.stat[0] = m; }
}
DTW_HD void dq_exp(int tid, int nt, DtwScratch & S, const DtwQkArgs & a, int r) {
    const float m = S.stat[0];
    const int n_ctx = dq_n_ctx(a, r);
    float sum = 0.0f;
    for (int j = tid; j < n_ctx; j += nt) { const float p = expf(S.s[j] - m); S.s[j] = p; sum += p; }
    S.red[tid] = sum;
}
DTW_HD void dq_sum(int tid, int nt, DtwScratch & S) {
    if (tid == 0) { double s = 0.0; for (int i = 0; i < nt; ++i) s += (double) S.red[i]; S.stat[1] = (float) (1.0 / s); }
}
DTW_HD void dq_store(int tid, int nt, DtwScratch & S, const DtwQkArgs & a, int e, int t, int r) {
    const float inv = S.stat[1];
    const int n_ctx = dq_n_ctx(a, r), n_tok = dq_n_tok(a, r);
    float * out = a.out + a.req_out[r];
    for (int j = tid; j < n_ctx; j += nt) out[((size_t) e * n_ctx + j) * n_tok + t] = S.s[j] * inv;
}

__global__ void __launch_bounds__(DTW_THREADS) k_dtw_qk(const DtwQkArgs a) {
    __shared__ DtwScratch S;
    const int e = blockIdx.x, t = blockIdx.y, r = blockIdx.z, tid = threadIdx.x, nt = blockDim.x;
    if (t >= dq_n_tok(a, r)) return;                              // requests have different token counts: the grid covers the longest
    dq_load(tid, nt, S, a, e, t, r); __syncthreads();
    dq_scores(tid, nt, S, a, e, r);  __syncthreads();
    dq_max(tid, nt, S);              __syncthreads();
    dq_exp(tid, nt, S, a, r);        __syncthreads();
    dq_sum(tid, nt, S);              __syncthreads();
    dq_store(tid, nt, S, a, e, t, r);
}

bool dtw_qk_launch(const DtwQkArgs & a, cudaStream_t st) {
    if (a.n_heads <= 0 || a.n_req <= 0 || a.max_tokens <= 0 || a.max_tokens > 65535 || a.n_req > 65535) {
        set_error("dtw: bad launch shape (heads %d, requests %d, tokens %d)", a.n_heads, a.n_req, a.max_tokens); return false;
    }
    k_dtw_qk<<<dim3((unsigned) a.n_heads, (unsigned) a.max_tokens, (unsigned) a.n_req), DTW_THREADS, 0, st>>>(a);
    count_launch();
    WB_CUDA_OK(cudaGetLastError());
    return true;
}

void dtw_qk_emulated(const DtwQkArgs & a) {
    DtwScratch * Sp = new DtwScratch(); DtwScratch & S = *Sp;
    const int nt = DTW_THREADS;
    for (int r = 0; r < a.n_req; ++r) for (int e = 0; e < a.n_heads; ++e) for (int t = 0; t < dq_n_tok(a, r); ++t) {
        for (int tid = 0; tid < nt; ++tid) dq_load(tid, nt, S, a, e, t, r);
        for (int tid = 0; tid < nt; ++tid) dq_scores(tid, nt, S, a, e, r);
        for (int tid = 0; tid < nt; ++tid) dq_max(tid, nt, S);
        for (int tid = 0; tid < nt; ++tid) dq_exp(tid, nt, S, a, r);
        for (int tid = 0; tid < nt; ++tid) dq_sum(tid, nt, S);
        for (int tid = 0; tid < nt; ++tid) dq_store(tid, nt, S, a, e, t, r);
    }
    delete Sp;
}

__global__ void __launch_bounds__(256) k_dtw_capture(const float * q, int d, const int * cap_row, int n_rows, uint32_t head_mask, int cap_head0,
                                                     float * cap, int cap_rows) {
    dtw_capture_rows(q, d, cap_row, n_rows, head_mask, cap_head0, cap, cap_rows, blockIdx.x * blockDim.x + threadIdx.x, gridDim.x * blockDim.x);
}

bool dtw_capture_launch(const float * q, int d, const int * cap_row, int n_rows, uint32_t head_mask, int cap_head0, float * cap, int cap_rows, cudaStream_t st) {
    const unsigned items = (unsigned) n_rows * (unsigned) __builtin_popcount(head_mask) * 16u;
    k_dtw_capture<<<(items + 255) / 256, 256, 0, st>>>(q, d, cap_row, n_rows, head_mask, cap_head0, cap, cap_rows);
    count_launch();
    WB_CUDA_OK(cudaGetLastError());
    return true;
}

// host walk of the phases for one request on slot 0: q [n_sel][n_tokens][d] f32 (whole rows of each captured layer), k [n_layers][...]
// f16 bits in the given layout, heads as (layer slot, layer, head) triples.  The query slices are repacked into the capture layout first.
static int dbg_dtw_qk(const float * q, const uint16_t * k, int Tp, int d, const int * triples, int n_heads, int n_tokens, int n_audio_ctx,
                      float scale, int k_head_major, float * out) {
    if (!q || !k || !triples || !out || n_audio_ctx > DTW_MAX_CTX) return -1;
    if (n_heads <= 0 || n_tokens <= 0 || n_audio_ctx <= 0) return 0;
    std::vector<int> hc((size_t) n_heads), ly((size_t) n_heads), hd((size_t) n_heads);
    std::vector<float> cap((size_t) n_heads * n_tokens * 64);
    for (int e = 0; e < n_heads; ++e) {
        hc[e] = e; ly[e] = triples[3 * e + 1]; hd[e] = triples[3 * e + 2];
        for (int t = 0; t < n_tokens; ++t) for (int i = 0; i < 64; ++i)
            cap[((size_t) e * n_tokens + t) * 64 + i] = q[((size_t) triples[3 * e] * n_tokens + t) * d + hd[e] * 64 + i];
    }
    const int req[4] = { 0, 0, n_tokens, n_audio_ctx };
    const int64_t req_out[1] = { 0 };
    DtwQkArgs a;
    a.q = cap.data(); a.cap_rows = n_tokens;
    a.k_cross = reinterpret_cast<const __half *>(k); a.slot_stride = 0; a.layer_stride = (int64_t) Tp * d; a.k_head_major = k_head_major; a.Tp = Tp;
    a.head_cap = hc.data(); a.head_layer = ly.data(); a.head_index = hd.data();
    a.req = req; a.req_out = req_out; a.n_heads = n_heads; a.n_req = 1; a.max_tokens = n_tokens; a.d = d; a.scale = scale; a.out = out;
    dtw_qk_emulated(a);
    return 0;
}

} // namespace wb

// host-only test hook: q [n_sel][n_tokens][d] f32, k [n_layers][Tp][d] f16 bits, heads as (layer slot, layer, head) triples
extern "C" __attribute__((visibility("default"))) int wb200_dbg_dtw_qk(const float * q, const uint16_t * k, int Tp, int d, const int * triples, int n_heads,
                                                                       int n_tokens, int n_audio_ctx, float scale, float * out) {
    return wb::dbg_dtw_qk(q, k, Tp, d, triples, n_heads, n_tokens, n_audio_ctx, scale, 0, out);
}
// host-only test hook: the same with the cross K in either layout; k_head_major = 1: k [n_layers][d/64][Tp][64] (the persistent decode
// kernel's cross K/V layout)
extern "C" __attribute__((visibility("default"))) int wb200_dbg_dtw_qk_layout(const float * q, const uint16_t * k, int Tp, int d, const int * triples,
                                                                              int n_heads, int n_tokens, int n_audio_ctx, float scale, int k_head_major,
                                                                              float * out) {
    return wb::dbg_dtw_qk(q, k, Tp, d, triples, n_heads, n_tokens, n_audio_ctx, scale, k_head_major != 0, out);
}

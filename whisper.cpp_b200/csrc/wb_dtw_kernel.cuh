// wb_dtw_kernel.cuh -- cross-attention WEIGHTS of the alignment heads for DTW token timestamps: softmax(f16(q) . K^T * 64^-1/4) over the
// audio positions, per (alignment head, text token).  This is what the reference's non-flash decoder graph keeps as aheads_cross_QKs
// (src/whisper.cpp:2722-2741: KQ = mul_mat(Kcross F16, Q -> F16), soft_max_ext(KQ, scale = KQscale)).
//
// Capture contract shared by both decoder paths: a decode row whose capture index c (packed row table, Engine::decode) is >= 0 leaves,
// for every alignment head, the 64 f32 values of that head from its layer's cross-Q output in q[capture head][c][64] -- the value the
// cross-attention consumes, before its f16 rounding.  The persistent kernel copies them at the start of its cross-attention phase, the
// kernel chain with k_dtw_capture right after its cross-Q GEMV; both call dtw_capture_rows.
#pragma once
#include <cstdint>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <vector>
#include "wb_common.h"

namespace wb {

struct DtwQkArgs {
    const float  * q;            // captured queries [n_capture_heads][cap_rows][64]  (before the 64^-1/4 scale)
    int cap_rows;
    const __half * k_cross;      // cross K of slot s, layer l at k_cross + s * slot_stride + l * layer_stride, already scaled by 64^-1/4
    int64_t slot_stride, layer_stride;
    int k_head_major;            // 0: a layer is token-major [Tp][d]; 1: head-major [d/64][Tp][64] (the persistent decode kernel's layout)
    int Tp;                      // keys per head in the head-major layout
    const int * head_cap;        // per alignment head: its capture head (index into q)
    const int * head_layer;      // per alignment head: text layer
    const int * head_index;      // per alignment head: head inside the layer
    const int * req;             // per request, 4 ints: capture index of its first token, cross-KV slot, tokens, audio positions
    const int64_t * req_out;     // per request: offset of its weights in out, [n_heads][n_audio_ctx][n_tokens] (tokens fastest: the reference's host copy)
    int n_heads, n_req, max_tokens, d;
    float scale;                 // 64^-1/4
    float * out;
};

bool dtw_qk_launch(const DtwQkArgs & a, cudaStream_t st);
// the same phases walked on the host (test hook; pointers are host pointers)
void dtw_qk_emulated(const DtwQkArgs & a);

// ---- the warping path of each request, computed from its weights on the device (dtw_path of wb_dtw.cpp, bit for bit)
// Per request: 5 ints (n_tokens, n_audio_ctx, n_heads, M = audio positions used, sot_len); N = n_tokens - sot_len - 1 path rows.
// Three launches cover every request of a batch: k_dtw_norm (mean and scale of each (head, position) column over the tokens),
// k_dtw_cost (7-wide median over time per head, mean over heads, negated: cost [N][M]) and k_dtw_sweep (one CTA per request: anti-diagonal
// sweep with 2-bit trace codes in shared memory, then the backtrace).  Every f32 operation the host does separately is an _rn intrinsic
// on the device (nvcc would contract a*b + c into an FMA) and a plain operator in the host walk; double sums keep the host's order.
// A request with N <= 0, M <= 7 or no heads gets an empty path, like dtw_path.
constexpr int DTW_REQ_INTS = 5;
struct DtwPathArgs {
    const float * w;             // weights: request r at w + off[4r], [n_heads][n_audio_ctx][n_tokens]
    const int * req;             // DTW_REQ_INTS per request
    const int64_t * off;         // per request, 4 offsets: weights (floats of w), column stats (float2 of stat), cost (floats), path (ints)
    float2 * stat;               // [n_heads][M] (mean, scale) per request
    float * cost;                // [N][M] per request
    int * path;                  // per request: tok_idx [N + M], time_idx [N + M], then the path length (1 int)
    int n_req;
};

// grow-only device buffers of a batch of path requests
class DtwPaths {
  public:
    // upload req / weight offsets (request r's weights at w + w_off[r], device memory) and launch the three kernels on st
    bool enqueue(const float * w, const std::vector<int> & req, const std::vector<int64_t> & w_off, cudaStream_t st);
    bool fetch(cudaStream_t st);      // queue the copy of every path to the host
    // after st has synchronised: the path of request r (tok_idx, time_idx in path order)
    void get(int r, std::vector<int32_t> & tok, std::vector<int32_t> & time) const;
  private:
    DevBuf<int> d_req, d_path; DevBuf<int64_t> d_off; DevBuf<float2> d_stat; DevBuf<float> d_cost;
    std::vector<int> h_req, h_path; std::vector<int64_t> h_off;
};

// chain path: copy the alignment-head slices of the rows of one pass from the cross-Q output q [n_rows][d]
bool dtw_capture_launch(const float * q, int d, const int * cap_row, int n_rows, uint32_t head_mask, int cap_head0, float * cap, int cap_rows, cudaStream_t st);

#ifdef __CUDACC__
// Rows t with cap_row[t] >= 0: for every head h set in head_mask (the alignment heads of this layer, in increasing order, capture heads
// cap_head0, cap_head0 + 1, ...) copy q[t][64h .. 64h + 63] to cap[capture head][cap_row[t]][0 .. 63].  Work item i = one float4;
// items i0, i0 + step, ...  q is read through L2: the persistent kernel wrote it in the same launch from other SMs.
__device__ __forceinline__ void dtw_capture_rows(const float * q, int d, const int * cap_row, int n_rows, uint32_t head_mask, int cap_head0,
                                                 float * cap, int cap_rows, unsigned i0, unsigned step) {
    const unsigned per_row = (unsigned) __popc(head_mask) * 16u, total = (unsigned) n_rows * per_row;
    for (unsigned i = i0; i < total; i += step) {
        const int t = (int) (i / per_row), r = (int) (i - (unsigned) t * per_row), k = r >> 4, c = r & 15;
        const int ci = __ldg(cap_row + t);
        if (ci < 0) continue;
        uint32_t m = head_mask;
        for (int s = 0; s < k; ++s) m &= m - 1;                  // drop the k lowest alignment heads of the layer
        const int h = __ffs((int) m) - 1;
        const float4 v = __ldcg(reinterpret_cast<const float4 *>(q + (size_t) t * d + h * 64) + c);
        reinterpret_cast<float4 *>(cap + ((size_t) (cap_head0 + k) * cap_rows + ci) * 64)[c] = v;
    }
}
#endif

} // namespace wb

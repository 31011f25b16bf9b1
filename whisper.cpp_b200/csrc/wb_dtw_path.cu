// wb_dtw_path.cu -- the warping path of DTW token timestamps on the device (DtwPaths, see wb_dtw_kernel.cuh).  Like k_dtw_qk, every stage
// is written as __host__ __device__ functions of one work item or of (tid, nthreads) between block barriers, so that the host can walk
// exactly the device's arithmetic (wb200_dbg_dtw_path).  A request's path never depends on the other requests of the launch.
// (A translation unit of its own: the sweep's dynamic shared memory would round up the static shared memory of k_dtw_qk.)
#include <algorithm>
#include <cmath>
#include <vector>
#include "wb_common.h"
#include "wb_dtw.h"
#include "wb_dtw_kernel.cuh"

namespace wb {

#define DTW_HD __host__ __device__ __forceinline__

constexpr int DTW_PATH_THREADS = 256;           // k_dtw_norm / k_dtw_cost: one column / one cell per thread
constexpr int DTW_SWEEP_THREADS = 512;          // k_dtw_sweep: one path row per thread (N + 1 <= 448 rows at n_text_ctx = 448)
constexpr int DTW_MEDFILT = 7;                  // median filter width of the reference (dtw_path's medfilt_width)
constexpr size_t DTW_SWEEP_SMEM_MAX = 232448;   // opt-in shared memory per block on sm_90

// f32 / f64 operations the host does one by one: _rn intrinsics on the device (no FMA contraction), plain operators in the host walk
DTW_HD float dp_add(float x, float y) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(x, y);
#else
    return x + y;
#endif
}
DTW_HD float dp_sub(float x, float y) {
#ifdef __CUDA_ARCH__
    return __fsub_rn(x, y);
#else
    return x - y;
#endif
}
DTW_HD float dp_mul(float x, float y) {
#ifdef __CUDA_ARCH__
    return __fmul_rn(x, y);
#else
    return x * y;
#endif
}
DTW_HD float dp_div(float x, float y) {
#ifdef __CUDA_ARCH__
    return __fdiv_rn(x, y);
#else
    return x / y;
#endif
}
DTW_HD float dp_sqrt(float x) {
#ifdef __CUDA_ARCH__
    return __fsqrt_rn(x);
#else
    return sqrtf(x);
#endif
}
DTW_HD double dp_ddiv(double x, double y) {
#ifdef __CUDA_ARCH__
    return __ddiv_rn(x, y);
#else
    return x / y;
#endif
}

struct DtwReq { int n_tok, n_ctx, n_heads, M, sot, N; };
DTW_HD DtwReq dp_req(const DtwPathArgs & a, int r) {
    const int * p = a.req + DTW_REQ_INTS * r;
    DtwReq q; q.n_tok = p[0]; q.n_ctx = p[1]; q.n_heads = p[2]; q.M = p[3]; q.sot = p[4]; q.N = p[0] - p[4] - 1;
    return q;
}
DTW_HD bool dp_empty(const DtwReq & q) { return q.N <= 0 || q.M <= DTW_MEDFILT || q.n_heads <= 0; }
DTW_HD int dp_words(const DtwReq & q) { return (q.M + 15) >> 4; }        // trace words per path row: 16 two-bit codes each

// 1. column c = (head, position j < M): mean over the tokens (double sum -> f32), centered sum of squares grouped like centered_sumsq
// (wb_dtw.cpp), scale 1 / sqrt(var + 1e-9)
DTW_HD void dp_norm_col(const DtwPathArgs & a, int r, int c) {
    const DtwReq q = dp_req(a, r);
    const int h = c / q.M, j = c - h * q.M, n = q.n_tok;
    const float * x = a.w + a.off[4 * r] + ((size_t) h * q.n_ctx + j) * n;
    double s = 0.0;
    for (int i = 0; i < n; ++i) s += (double) x[i];
    const float mean = dp_div((float) s, (float) n);
    double ss = 0.0; int i = 0;
    for (; i + 7 < n; i += 8) {
        float v[8];
        for (int k = 0; k < 8; ++k) { const float d = dp_sub(x[i + k], mean); v[k] = dp_mul(d, d); }
        const float a0 = dp_add(v[4], v[0]), a1 = dp_add(v[5], v[1]), a2 = dp_add(v[6], v[2]), a3 = dp_add(v[7], v[3]);
        ss += (double) dp_add(dp_add(a0, a2), dp_add(a1, a3));
    }
    for (; i < n; ++i) { const float d = dp_sub(x[i], mean); ss += (double) dp_mul(d, d); }
    const float var = (float) dp_ddiv(ss, (double) n);
    a.stat[a.off[4 * r + 1] + c] = make_float2(mean, dp_div(1.0f, dp_sqrt(dp_add(var, 1e-9f))));
}

DTW_HD void dp_cswap(float & x, float & y) { const float lo = y < x ? y : x, hi = y < x ? x : y; x = lo; y = hi; }
// the 4th smallest of 7 (what std::sort(v, v + 7)[3] returns): a 16-comparator sorting network
DTW_HD float dp_median7(float * v) {
    dp_cswap(v[0], v[6]); dp_cswap(v[2], v[3]); dp_cswap(v[4], v[5]);
    dp_cswap(v[0], v[2]); dp_cswap(v[1], v[4]); dp_cswap(v[3], v[6]);
    dp_cswap(v[0], v[1]); dp_cswap(v[2], v[5]); dp_cswap(v[3], v[4]);
    dp_cswap(v[1], v[2]); dp_cswap(v[4], v[6]);
    dp_cswap(v[2], v[3]); dp_cswap(v[4], v[5]);
    dp_cswap(v[1], v[2]); dp_cswap(v[3], v[4]); dp_cswap(v[5], v[6]);
    return v[3];
}

// 2. cell e = (token row i < N, position j < M), i fastest (neighbouring threads read neighbouring tokens): per head the median of the
// normalised weights at positions j - 3 .. j + 3 (reflected at both ends) of token sot + i; the double sum over heads in head order;
// cost = (f32 sum / heads) * -1
DTW_HD void dp_cost_cell(const DtwPathArgs & a, int r, int e) {
    const DtwReq q = dp_req(a, r);
    const int j = e / q.N, i = e - j * q.N, hw = DTW_MEDFILT / 2;
    const float * w = a.w + a.off[4 * r] + q.sot + i;
    const float2 * st = a.stat + a.off[4 * r + 1];
    double s = 0.0;
    for (int h = 0; h < q.n_heads; ++h) {
        float v[DTW_MEDFILT];
        for (int o = -hw; o <= hw; ++o) {
            int idx = j + o;
            if (idx < 0) idx = -idx; else if (idx >= q.M) idx = 2 * (q.M - 1) - idx;
            const float2 ms = st[(size_t) h * q.M + idx];
            v[o + hw] = dp_mul(dp_sub(w[((size_t) h * q.n_ctx + idx) * q.n_tok], ms.x), ms.y);
        }
        s += (double) dp_median7(v);
    }
    a.cost[a.off[4 * r + 2] + (size_t) i * q.M + j] = dp_mul(dp_div((float) s, (float) q.n_heads), -1.0f);
}

// 3. anti-diagonal sweep of one request.  Shared memory: D = three diagonals of N + 1 floats (row i at index i), T = N rows of
// dp_words(q) words of 2-bit trace codes for cells (i >= 1, j >= 1); row i is written only by the thread that owns it (i mod nt).
struct DtwShm { float * D; uint32_t * T; };
DTW_HD void dp_sweep_init(int tid, int nt, DtwShm S, const DtwReq & q) {
    const int nw = q.N * dp_words(q);
    for (int k = tid; k < nw; k += nt) S.T[k] = 0u;
    for (int i = tid; i <= q.N; i += nt) { S.D[i] = i == 0 ? 0.0f : INFINITY; S.D[q.N + 1 + i] = INFINITY; }   // diagonals 0 and 1
}
// diagonal d = i + j >= 2 into buffer d % 3 from d - 1 and d - 2: D[i][j] = cost + min(diagonal, up, left), strict comparisons pick
// diagonal, then up, else left (dtw_path)
DTW_HD void dp_sweep_diag(int tid, int nt, DtwShm S, const DtwPathArgs & a, int r, const DtwReq & q, int d) {
    const int ld = q.N + 1, W = dp_words(q);
    float * cur = S.D + (d % 3) * ld;
    const float * p1 = S.D + ((d + 2) % 3) * ld, * p2 = S.D + ((d + 1) % 3) * ld;
    const float * cost = a.cost + a.off[4 * r + 2];
    for (int i = tid; i <= q.N; i += nt) {
        const int j = d - i;
        if (j < 0 || j > q.M) continue;                           // outside the grid: never read
        if (i == 0 || j == 0) { cur[i] = INFINITY; continue; }
        const float c0 = p2[i - 1], c1 = p1[i - 1], c2 = p1[i];
        float c; uint32_t t;
        if (c0 < c1 && c0 < c2) { c = c0; t = 0u; } else if (c1 < c0 && c1 < c2) { c = c1; t = 1u; } else { c = c2; t = 2u; }
        cur[i] = dp_add(cost[(size_t) (i - 1) * q.M + (j - 1)], c);
        S.T[(size_t) (i - 1) * W + ((j - 1) >> 4)] |= t << (2 * ((j - 1) & 15));
    }
}
DTW_HD void dp_step(const uint32_t * T, int W, int & i, int & j) {
    const uint32_t t = i == 0 ? 2u : j == 0 ? 1u : (T[(size_t) (i - 1) * W + ((j - 1) >> 4)] >> (2 * ((j - 1) & 15))) & 3u;
    if (t == 0u) { --i; --j; } else if (t == 1u) --i; else --j;
}
// 4. backtrace from (N, M) by thread 0: count the steps, then write (i - 1, j - 1) of every cell left on the way, in path order
DTW_HD void dp_backtrace(int tid, DtwShm S, const DtwPathArgs & a, int r, const DtwReq & q) {
    if (tid != 0) return;
    const int W = dp_words(q), cap = q.N + q.M;
    int * tok = a.path + a.off[4 * r + 3], * tim = tok + cap;
    int n = 0;
    for (int i = q.N, j = q.M; i > 0 || j > 0; ++n) dp_step(S.T, W, i, j);
    for (int i = q.N, j = q.M, k = n; i > 0 || j > 0;) { --k; tok[k] = i - 1; tim[k] = j - 1; dp_step(S.T, W, i, j); }
    tok[2 * cap] = n;
}

__global__ void __launch_bounds__(DTW_PATH_THREADS) k_dtw_norm(const DtwPathArgs a) {
    const int r = blockIdx.y, c = blockIdx.x * blockDim.x + threadIdx.x;
    const DtwReq q = dp_req(a, r);
    if (!dp_empty(q) && c < q.n_heads * q.M) dp_norm_col(a, r, c);
}
__global__ void __launch_bounds__(DTW_PATH_THREADS) k_dtw_cost(const DtwPathArgs a) {
    const int r = blockIdx.y, e = blockIdx.x * blockDim.x + threadIdx.x;
    const DtwReq q = dp_req(a, r);
    if (!dp_empty(q) && e < q.N * q.M) dp_cost_cell(a, r, e);
}
__global__ void __launch_bounds__(DTW_SWEEP_THREADS) k_dtw_sweep(const DtwPathArgs a) {
    extern __shared__ float dp_smem[];
    const int r = blockIdx.x, tid = threadIdx.x, nt = blockDim.x;
    const DtwReq q = dp_req(a, r);
    if (dp_empty(q)) { if (tid == 0) a.path[a.off[4 * r + 3]] = 0; return; }
    const DtwShm S = { dp_smem, reinterpret_cast<uint32_t *>(dp_smem + 3 * (q.N + 1)) };
    dp_sweep_init(tid, nt, S, q); __syncthreads();
    for (int d = 2; d <= q.N + q.M; ++d) { dp_sweep_diag(tid, nt, S, a, r, q, d); __syncthreads(); }
    dp_backtrace(tid, S, a, r, q);
}

static size_t dp_sweep_smem(const DtwReq & q) { return dp_empty(q) ? 0 : ((size_t) 3 * (q.N + 1) + (size_t) q.N * dp_words(q)) * 4; }

// per request: weights offset (given), stat / cost / path offsets; totals and grid sizes.  The path of a request takes 2 * cap + 1 ints
// (cap = N + M, 0 for an empty path; the last int is the length).
static bool dp_layout(const std::vector<int> & req, const std::vector<int64_t> & w_off, std::vector<int64_t> & off, int64_t & n_stat,
                      int64_t & n_cost, int64_t & n_path, int & max_cols, int & max_cells, size_t & smem) {
    const int n_req = (int) w_off.size();
    if (n_req <= 0 || n_req > 65535 || req.size() != (size_t) DTW_REQ_INTS * n_req) { set_error("dtw path: bad batch of %d requests", n_req); return false; }
    off.assign((size_t) 4 * n_req, 0);
    n_stat = n_cost = n_path = 0; max_cols = max_cells = 0; smem = 0;
    DtwPathArgs a; a.req = req.data();
    for (int r = 0; r < n_req; ++r) {
        const DtwReq q = dp_req(a, r);
        if (q.n_tok <= 0 || q.n_ctx <= 0 || q.n_heads < 0 || q.M < 0 || q.sot < 0 || w_off[(size_t) r] < 0) {
            set_error("dtw path: bad request %d (tokens %d, audio positions %d, heads %d, M %d, sot_len %d)", r, q.n_tok, q.n_ctx, q.n_heads, q.M, q.sot);
            return false;
        }
        off[(size_t) 4 * r] = w_off[(size_t) r];
        off[(size_t) 4 * r + 1] = n_stat; off[(size_t) 4 * r + 2] = n_cost; off[(size_t) 4 * r + 3] = n_path;
        n_path += 1;
        if (dp_empty(q)) continue;
        if (q.M > q.n_ctx || (int64_t) q.n_heads * q.M > (1 << 30) || (int64_t) q.N * q.M > (1 << 30) || dp_sweep_smem(q) > DTW_SWEEP_SMEM_MAX) {
            set_error("dtw path: request %d too large (tokens %d, audio positions %d, heads %d, M %d)", r, q.n_tok, q.n_ctx, q.n_heads, q.M);
            return false;
        }
        n_stat += (int64_t) q.n_heads * q.M; n_cost += (int64_t) q.N * q.M; n_path += (int64_t) 2 * (q.N + q.M);
        max_cols = std::max(max_cols, q.n_heads * q.M); max_cells = std::max(max_cells, q.N * q.M); smem = std::max(smem, dp_sweep_smem(q));
    }
    return true;
}

bool DtwPaths::enqueue(const float * w, const std::vector<int> & req, const std::vector<int64_t> & w_off, cudaStream_t st) {
    int64_t n_stat, n_cost, n_path; int max_cols, max_cells; size_t smem;
    if (!dp_layout(req, w_off, h_off, n_stat, n_cost, n_path, max_cols, max_cells, smem)) return false;
    h_req = req;
    const int n_req = (int) w_off.size();
    if (h_req.size() > d_req.n && !d_req.alloc(h_req.size())) return false;
    if (h_off.size() > d_off.n && !d_off.alloc(h_off.size())) return false;
    if ((size_t) n_stat > d_stat.n && !d_stat.alloc((size_t) n_stat)) return false;
    if ((size_t) n_cost > d_cost.n && !d_cost.alloc((size_t) n_cost)) return false;
    if ((size_t) n_path > d_path.n && !d_path.alloc((size_t) n_path)) return false;
    WB_CUDA_OK(cudaMemcpyAsync(d_req.p, h_req.data(), h_req.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    WB_CUDA_OK(cudaMemcpyAsync(d_off.p, h_off.data(), h_off.size() * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    count_h2d(h_req.size() * sizeof(int) + h_off.size() * sizeof(int64_t));
    DtwPathArgs a;
    a.w = w; a.req = d_req.p; a.off = d_off.p; a.stat = d_stat.p; a.cost = d_cost.p; a.path = d_path.p;
    a.n_req = n_req;
    if (max_cells > 0) {
        k_dtw_norm<<<dim3((unsigned) (max_cols + DTW_PATH_THREADS - 1) / DTW_PATH_THREADS, (unsigned) n_req), DTW_PATH_THREADS, 0, st>>>(a);
        k_dtw_cost<<<dim3((unsigned) (max_cells + DTW_PATH_THREADS - 1) / DTW_PATH_THREADS, (unsigned) n_req), DTW_PATH_THREADS, 0, st>>>(a);
        count_launch(2);
        WB_CUDA_OK(cudaGetLastError());
    }
    WB_CUDA_OK(ensure_dyn_smem((const void *) k_dtw_sweep, smem));
    k_dtw_sweep<<<(unsigned) n_req, DTW_SWEEP_THREADS, smem, st>>>(a);
    count_launch();
    WB_CUDA_OK(cudaGetLastError());
    h_path.resize((size_t) n_path);
    return true;
}

bool DtwPaths::fetch(cudaStream_t st) {
    WB_CUDA_OK(cudaMemcpyAsync(h_path.data(), d_path.p, h_path.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
    count_d2h(h_path.size() * sizeof(int));
    return true;
}

static void dp_get(const int * req, const int * path, int64_t off, std::vector<int32_t> & tok, std::vector<int32_t> & time) {
    DtwPathArgs a; a.req = req;
    const DtwReq q = dp_req(a, 0);
    const int cap = dp_empty(q) ? 0 : q.N + q.M, n = path[off + 2 * cap];
    tok.assign(path + off, path + off + n); time.assign(path + off + cap, path + off + cap + n);
}

void DtwPaths::get(int r, std::vector<int32_t> & tok, std::vector<int32_t> & time) const {
    dp_get(h_req.data() + DTW_REQ_INTS * r, h_path.data(), h_off[(size_t) 4 * r + 3], tok, time);
}

// host walk of the three kernels, request by request, phase by phase (pointers are host pointers)
static void dtw_path_emulated(const DtwPathArgs & a) {
    for (int r = 0; r < a.n_req; ++r) {
        const DtwReq q = dp_req(a, r);
        if (dp_empty(q)) { a.path[a.off[4 * r + 3]] = 0; continue; }
        for (int c = 0; c < q.n_heads * q.M; ++c) dp_norm_col(a, r, c);
        for (int e = 0; e < q.N * q.M; ++e) dp_cost_cell(a, r, e);
        std::vector<uint32_t> shm(dp_sweep_smem(q) / 4);
        const DtwShm S = { reinterpret_cast<float *>(shm.data()), shm.data() + 3 * (q.N + 1) };
        const int nt = DTW_SWEEP_THREADS;
        for (int tid = 0; tid < nt; ++tid) dp_sweep_init(tid, nt, S, q);
        for (int d = 2; d <= q.N + q.M; ++d) for (int tid = 0; tid < nt; ++tid) dp_sweep_diag(tid, nt, S, a, r, q, d);
        for (int tid = 0; tid < nt; ++tid) dp_backtrace(tid, S, a, r, q);
    }
}

// test hook (host): one request's path from dtw_path (device_walk = 0) or from the host walk of the device phases (1)
static int dbg_dtw_path(const float * qk, int n_tokens, int n_audio_ctx, int n_heads, int M, int sot_len, int device_walk, int * tok, int * time, int cap) {
    if (!qk || !tok || !time) { set_error("dtw path: null argument"); return -1; }
    std::vector<int32_t> ti, tj;
    if (device_walk) {
        const std::vector<int> req = { n_tokens, n_audio_ctx, n_heads, M, sot_len };
        const std::vector<int64_t> w_off = { 0 };
        std::vector<int64_t> off; int64_t n_stat, n_cost, n_path; int max_cols, max_cells; size_t smem;
        if (!dp_layout(req, w_off, off, n_stat, n_cost, n_path, max_cols, max_cells, smem)) return -1;
        std::vector<float2> stat((size_t) n_stat); std::vector<float> cost((size_t) n_cost); std::vector<int> path((size_t) n_path);
        DtwPathArgs a;
        a.w = qk; a.req = req.data(); a.off = off.data(); a.stat = stat.data(); a.cost = cost.data(); a.path = path.data();
        a.n_req = 1;
        dtw_path_emulated(a);
        dp_get(req.data(), path.data(), off[3], ti, tj);
    } else {
        dtw_path(qk, n_tokens, n_audio_ctx, n_heads, M, sot_len, DTW_MEDFILT, ti, tj);
    }
    if ((int) ti.size() > cap) { set_error("dtw path: %zu steps, room for %d", ti.size(), cap); return -1; }
    std::copy(ti.begin(), ti.end(), tok); std::copy(tj.begin(), tj.end(), time);
    return (int) ti.size();
}

// test hook (GPU): several requests uploaded together, the three kernels launched once for all of them, every path returned.
// w: all weights (host), request r at w + w_off[r]; req: DTW_REQ_INTS per request; request r's path is written at tok / time +
// out_off[r] (room for N + M steps), its length to len[r]
static int dbg_dtw_path_device(int device, const float * w, int64_t n_w, const int64_t * w_off, const int * req, int n_req,
                               int * tok, int * time, const int64_t * out_off, int * len) {
    if (!w || !w_off || !req || !tok || !time || !out_off || !len || n_req <= 0 || n_w <= 0) { set_error("dtw path: bad arguments"); return -1; }
    WB_CUDA_OKV(cudaSetDevice(device), -1);
    DevBuf<float> dw;
    if (!dw.alloc((size_t) n_w)) return -1;
    WB_CUDA_OKV(cudaMemcpy(dw.p, w, (size_t) n_w * sizeof(float), cudaMemcpyHostToDevice), -1);
    cudaStream_t st;
    WB_CUDA_OKV(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking), -1);
    int rc = 0;
    {
        DtwPaths P;
        const bool ok = P.enqueue(dw.p, std::vector<int>(req, req + (size_t) DTW_REQ_INTS * n_req), std::vector<int64_t>(w_off, w_off + n_req), st) &&
                        P.fetch(st);
        const cudaError_t e = cudaStreamSynchronize(st);
        if (!ok) rc = -1;
        else if (e != cudaSuccess) { set_error("dtw path: %s", cudaGetErrorString(e)); rc = -1; }
        else for (int r = 0; r < n_req; ++r) {
            std::vector<int32_t> ti, tj;
            P.get(r, ti, tj);
            std::copy(ti.begin(), ti.end(), tok + out_off[r]); std::copy(tj.begin(), tj.end(), time + out_off[r]);
            len[r] = (int) ti.size();
        }
    }
    cudaStreamDestroy(st);
    return rc;
}

} // namespace wb

// host-only test hook: the warping path of weights [n_heads][n_audio_ctx][n_tokens] over M audio positions, from dtw_path (device_walk
// = 0) or from the host walk of k_dtw_norm / k_dtw_cost / k_dtw_sweep (1).  Returns the path length, -1 on error (wb200_last_error)
extern "C" __attribute__((visibility("default"))) int wb200_dbg_dtw_path(const float * qk, int n_tokens, int n_audio_ctx, int n_heads, int M,
                                                                         int sot_len, int device_walk, int * tok, int * time, int cap) {
    return wb::dbg_dtw_path(qk, n_tokens, n_audio_ctx, n_heads, M, sot_len, device_walk, tok, time, cap);
}
// GPU test hook: the paths of n_req requests (5 ints each: n_tokens, n_audio_ctx, n_heads, M, sot_len) from one launch of each kernel
extern "C" __attribute__((visibility("default"))) int wb200_dbg_dtw_path_device(int device, const float * w, int64_t n_w, const int64_t * w_off,
                                                                                const int * req, int n_req, int * tok, int * time,
                                                                                const int64_t * out_off, int * len) {
    return wb::dbg_dtw_path_device(device, w, n_w, w_off, req, n_req, tok, time, out_off, len);
}

// wb_common.h -- error reporting, launch accounting and small RAII helpers shared by the engine sources.
#pragma once
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

namespace wb {

// thread-local last-error text (exposed through wb200_last_error)
void set_error(const char * fmt, ...) __attribute__((format(printf, 1, 2)));
const char * last_error();

// every kernel launch issued by this library bumps this counter (bench.py reports it as gpu_launches)
void     count_launch(uint64_t n = 1);
// cudaFuncAttributeMaxDynamicSharedMemorySize is per device: remember (device, kernel) -> bytes so that a process that opens
// contexts on several GPUs configures every kernel on each of them (thread-safe; a no-op once the size is covered)
cudaError_t ensure_dyn_smem(const void * kernel, size_t bytes);
uint64_t launch_count();

// ---- optional per-kernel-class timing (CUDA events on the launching stream); off by default.  bench.py uses it for
// the roofline entry: algorithmic bytes / flops are supplied by the launcher, durations come from event pairs.
enum ProfClass { PC_GEMM = 0, PC_GEMV = 1, PC_ATTN = 2, PC_OTHER = 3, PC_COUNT = 4 };
void prof_enable(bool on);
bool prof_enabled();
struct ProfScope {
    int idx = -1; cudaStream_t st;
    ProfScope(int cls, cudaStream_t stream, double bytes, double flops);
    ~ProfScope();
};
// sums since the last prof_enable(true); synchronises the device.  arrays of PC_COUNT
void prof_collect(double * ms, uint64_t * launches, double * bytes, double * flops);

// coarse engine counters (wb200_counters): [0] decode passes [1] decode rows [2] decode GPU ms (events around each pass)
// [3] decode host ms (wall time inside Engine::decode) [4] encode calls [5] encode windows [6] encode GPU ms [7] graph replays
// [8] k_dtw_qk GPU ms [9] DTW passes [10] host DTW ms (dtw_assign) [11] device DTW path GPU ms (k_dtw_norm, k_dtw_cost, k_dtw_sweep)
// [12] run-ahead decode rows launched (Group::run) [13] run-ahead rows accepted, i.e. whose results a member's real request took
void   counter_add(int idx, double v);
double counter_get(int idx);

// host<->device traffic issued by the library (bytes), for bench.py's e2e accounting
void     count_h2d(uint64_t n);
void     count_d2h(uint64_t n);
uint64_t h2d_bytes();
uint64_t d2h_bytes();

// NVTX range around the engine's coarse steps (mel, encode, decode pass, VAD) for `ncu --nvtx` / Nsight filtering; active only with
// WB200_NVTX=1 (header-only NVTX3, no link dependency; a no-op without a profiler attached)
struct NvtxRange { bool on; explicit NvtxRange(const char * name); ~NvtxRange(); NvtxRange(const NvtxRange &) = delete; NvtxRange & operator=(const NvtxRange &) = delete; };

// logging through the whisper_log_set callback (default: stderr)
enum LogLevel { LOG_DEBUG = 1, LOG_INFO = 2, LOG_WARN = 3, LOG_ERROR = 4 };
void logf(int level, const char * fmt, ...) __attribute__((format(printf, 2, 3)));

#define WB_CUDA_OK(expr) \
    do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) { ::wb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e_)); return false; } } while (0)
#define WB_CUDA_OKV(expr, rv) \
    do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) { ::wb::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(e_)); return rv; } } while (0)

template <typename T> struct DevBuf {
    T * p = nullptr; size_t n = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete; DevBuf & operator=(const DevBuf &) = delete;
    ~DevBuf() { release(); }
    bool alloc(size_t count, bool zero = false) {
        release();
        if (count == 0) return true;
        if (cudaMalloc(&p, count * sizeof(T)) != cudaSuccess) { p = nullptr; set_error("cudaMalloc(%zu bytes) failed", count * sizeof(T)); return false; }
        n = count;
        if (zero && cudaMemset(p, 0, count * sizeof(T)) != cudaSuccess) { set_error("cudaMemset failed"); return false; }
        return true;
    }
    void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
    size_t bytes() const { return n * sizeof(T); }
};

} // namespace wb

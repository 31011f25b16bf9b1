// wb_fattn.cu -- fused encoder self-attention on wgmma (replaces ggml_flash_attn_ext in whisper_build_graph_encoder,
// src/whisper.cpp:2142-2167; CPU semantics ggml/src/ggml-cpu/ops.cpp:8479-8715).
//
//   out[q, h*64 + :] = softmax_k( scale * Q_h[q,:] . K_h[k,:] ) @ V_h[k,:]     over k = 0 .. 1535
//
// The 36 padded keys (rows 1500..1535) are all-zero and NOT masked in the reference (SURVEY.md fact 4): here K rows beyond
// n_ctx are zero-filled by TMA and the V^T buffer keeps zeros in those columns, so they take part in max and sum exactly
// like in the reference.
//
// One CTA = 128 queries of one head, three warpgroups: warpgroup 0 is the TMA producer (one thread), warpgroups 1 and 2 own 64 queries
// each.  Two passes over the 24 key blocks of 64:
//   pass 1  S_j = Q K_j^T (4 x wgmma m64n64k16, both operands in smem, S in registers)  -> row maxima only
//   pass 2  S_j again, p = exp2((s - m) * scale*log2e) with the FINAL maximum m, rounded to f16 in registers, which are the A operand of
//           O += P_j V_j (4 x wgmma m64n64k16, A from registers, V^T from smem) accumulated in registers, l += sum p
// Knowing m before any exponent is taken removes the online-softmax rescaling of O; the price is recomputing QK^T once: +1/3 tensor work
// on 14% of the encoder flops.
#include "wb_gemm.cuh"
#include "wb_ptx.cuh"
#include "wb_common.h"
#include "wb_kernels.cuh"

namespace wb {

static constexpr int FA_THREADS = 384;
static constexpr int FA_KSTAGES = 3, FA_VSTAGES = 2;
static constexpr int FA_KB = 64;                   // keys per block
static constexpr int FA_Q_BYTES = 128 * 128, FA_K_BYTES = FA_KB * 128, FA_V_BYTES = 64 * FA_KB * 2;
static constexpr int FA_SMEM = FA_Q_BYTES + FA_KSTAGES * FA_K_BYTES + FA_VSTAGES * FA_V_BYTES + 1024 + 256;

struct FattnParams { int T, n_kb; float scale_log2e; __half * out; int64_t ldo, out_win; };

__device__ __forceinline__ float ex2f(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ uint32_t pack_half2(float a, float b) { const __half2 h = __floats2half2_rn(a, b); return *reinterpret_cast<const uint32_t *>(&h); }

__global__ void __launch_bounds__(FA_THREADS, 1)
fattn_enc_kernel(const FattnParams p, const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t * smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t * sQ = smem;
    uint8_t * sK = sQ + FA_Q_BYTES;
    uint8_t * sV = sK + FA_KSTAGES * FA_K_BYTES;
    uint64_t * bars = reinterpret_cast<uint64_t *>(sV + FA_VSTAGES * FA_V_BYTES);
    uint64_t * k_full = bars,       * k_empty = bars + 3;
    uint64_t * v_full = bars + 6,   * v_empty = bars + 8;
    uint64_t * q_full = bars + 10;

    const int wg = threadIdx.x >> 7, lane = threadIdx.x & 31;
    const int q0 = blockIdx.x * 128, h = blockIdx.y, w = blockIdx.z;
    const int n_kb = p.n_kb;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
        for (int i = 0; i < FA_KSTAGES; ++i) { mbar_init(&k_full[i], 1); mbar_init(&k_empty[i], 8); }    // released by the 8 MMA warps
        for (int i = 0; i < FA_VSTAGES; ++i) { mbar_init(&v_full[i], 1); mbar_init(&v_empty[i], 8); }
        mbar_init(q_full, 1);
        mbar_fence_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ---------------------------------------------------------------- TMA producer
        if (threadIdx.x == 0) {
            mbar_arrive_expect_tx(q_full, FA_Q_BYTES);
            tma_load_4d(sQ, &tmQ, q_full, 0, q0, h, w);
            int ks = 0; uint32_t kph = 0; int vs = 0; uint32_t vph = 0;
            for (int pass = 0; pass < 2; ++pass) {
                for (int j = 0; j < n_kb; ++j) {
                    mbar_wait(&k_empty[ks], kph ^ 1);
                    mbar_arrive_expect_tx(&k_full[ks], FA_K_BYTES);
                    tma_load_4d(sK + ks * FA_K_BYTES, &tmK, &k_full[ks], 0, j * FA_KB, h, w);
                    if (++ks == FA_KSTAGES) { ks = 0; kph ^= 1; }
                    if (pass == 1) {
                        mbar_wait(&v_empty[vs], vph ^ 1);
                        mbar_arrive_expect_tx(&v_full[vs], FA_V_BYTES);
                        tma_load_4d(sV + vs * FA_V_BYTES, &tmV, &v_full[vs], j * FA_KB, 0, h, w);
                        if (++vs == FA_VSTAGES) { vs = 0; vph ^= 1; }
                    }
                }
            }
        }
        return;
    }

    // -------------------------------------------------------------------- MMA + softmax warpgroups
    // thread t holds query rows r0 = 16*(t/32) + (t%32)/4 and r0 + 8 of its warpgroup's 64, key / output columns 8*j + 2*(t%4) (+1)
    const int cw = wg - 1, t = threadIdx.x & 127;
    const int r0 = cw * 64 + 16 * (t >> 5) + ((t & 31) >> 2);
    const uint64_t qdesc = wgmma_desc_sw128(smem_u32(sQ + cw * 64 * 128));
    int ks = 0; uint32_t kph = 0;
    float S[32];
    auto scores = [&]() {                                  // S = Q K_j^T of the next K stage; the stage is released afterwards
        mbar_wait(&k_full[ks], kph);
        wgmma_fence();
        const uint64_t kdesc = wgmma_desc_sw128(smem_u32(sK + ks * FA_K_BYTES));
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_f16_ss<64>(S, qdesc + 2*k, kdesc + 2*k, k ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(S);
        __syncwarp();
        if (lane == 0) mbar_arrive(&k_empty[ks]);
        if (++ks == FA_KSTAGES) { ks = 0; kph ^= 1; }
    };
    mbar_wait(q_full, 0);
    // pass 1: row maxima of the raw scores
    float m[2] = { -INFINITY, -INFINITY };
    for (int j = 0; j < n_kb; ++j) {
        scores();
#pragma unroll
        for (int i = 0; i < 32; ++i) m[(i >> 1) & 1] = fmaxf(m[(i >> 1) & 1], S[i]);
    }
    float mc[2], l[2] = { 0.0f, 0.0f };
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 1));
        m[r] = fmaxf(m[r], __shfl_xor_sync(0xffffffffu, m[r], 2));
        mc[r] = m[r] * p.scale_log2e;
    }
    // pass 2: probabilities with the final maximum, O += P V
    float O[32];
    int vs = 0; uint32_t vph = 0;
    for (int j = 0; j < n_kb; ++j) {
        scores();
        uint32_t a[4][4];
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
            const int r = (i >> 1) & 1;
            const float p0 = ex2f(fmaf(S[i],     p.scale_log2e, -mc[r]));
            const float p1 = ex2f(fmaf(S[i + 1], p.scale_log2e, -mc[r]));
            const uint32_t hp = pack_half2(p0, p1);
            // the tensor core consumes the ROUNDED probabilities: accumulate the same values into the denominator
            const float2 pr = __half22float2(*reinterpret_cast<const __half2 *>(&hp));
            l[r] += pr.x + pr.y;
            a[i >> 3][(i & 7) >> 1] = hp;                  // keys 16*s .. 16*s + 15 = S[8s .. 8s + 7]: the A fragment of k-step s
        }
        mbar_wait(&v_full[vs], vph);
        wgmma_fence();
        const uint64_t vdesc = wgmma_desc_sw128(smem_u32(sV + vs * FA_V_BYTES));
#pragma unroll
        for (int s = 0; s < 4; ++s) wgmma_f16_rs_n64(O, a[s], vdesc + 2*s, (j | s) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(O);
        __syncwarp();
        if (lane == 0) mbar_arrive(&v_empty[vs]);
        if (++vs == FA_VSTAGES) { vs = 0; vph ^= 1; }
    }
    // epilogue: O / l -> f16 -> global
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
        l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
        const int qg = q0 + r0 + 8 * r;
        if (qg >= p.T) continue;
        const float inv = 1.0f / l[r];
        __half * orow = p.out + (int64_t) w * p.out_win + (int64_t) qg * p.ldo + h * 64 + 2 * (t & 3);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
            *reinterpret_cast<uint32_t *>(orow + 8 * jj) = pack_half2(O[4 * jj + 2 * r] * inv, O[4 * jj + 2 * r + 1] * inv);
    }
}

// Q, K: f16 [n_win][T][ld_qk] with head h at columns h*64 (K at +k_off); Vt: f16 [n_win][H*64][Tp]; out: f16 [n_win*T][ldo]
bool fattn_encoder(const __half * qk, int ld_qk, int k_off, const __half * vt, int T, int Tp, int H, int n_win, float scale,
                   __half * out, int ldo, cudaStream_t st) {
    CUtensorMap tmQ, tmK, tmV;
    if (!make_tmap_f16(&tmQ, qk,         64, T, H, n_win, ld_qk, 64, (uint64_t) T * ld_qk, 128)) return false;
    if (!make_tmap_f16(&tmK, qk + k_off, 64, T, H, n_win, ld_qk, 64, (uint64_t) T * ld_qk, FA_KB)) return false;
    if (!make_tmap_f16(&tmV, vt, Tp, 64, H, n_win, Tp, (uint64_t) 64 * Tp, (uint64_t) H * 64 * Tp, 64)) return false;
    WB_CUDA_OK(ensure_dyn_smem(reinterpret_cast<const void *>(fattn_enc_kernel), FA_SMEM));
    FattnParams p; p.T = T; p.n_kb = Tp / FA_KB; p.scale_log2e = scale * 1.4426950408889634f; p.out = out; p.ldo = ldo; p.out_win = (int64_t) T * ldo;
    ProfScope prof(PC_ATTN, st, 0.0, (double) n_win * H * (3.0 * 2 * T * (double) Tp * 64));   // QK twice + PV
    fattn_enc_kernel<<<dim3((T + 127) / 128, H, n_win), FA_THREADS, FA_SMEM, st>>>(p, tmQ, tmK, tmV);
    count_launch();
    return cudaGetLastError() == cudaSuccess;
}

} // namespace wb

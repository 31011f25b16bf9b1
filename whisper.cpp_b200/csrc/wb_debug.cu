// wb_debug.cu -- wb200_dbg_* entry points: drive single kernels from host buffers so the parity tests can pin
// each one against the oracle in isolation.  Not used by the product path.
#include <cstring>
#include <vector>
#include "wb_common.h"
#include "wb_decode_mk.cuh"
#include "wb_gemm.cuh"
#include "wb_kernels.cuh"

using namespace wb;

extern "C" {

// C[n][m] (f32, token-major) = sum_k W[m][k] * X[n][k] ; W given in FILE layout (f16 rows or ggml quant blocks),
// X given as f32 and rounded to f16 on the way in (as the engine does).  flags bit0: apply gelu; bit1: m-major output;
// bit2: the persistent kernel (quantised weights expanded to f16 once, both operands through TMA); bit3: the activation tile fetched
// as two half-height TMA boxes, bit4 = f16 output, bit5 = in-place f32 residual (out holds x on entry), bit6 (with bit4, M a multiple of
// 64) = head-major f16 output [M / 64][N][64] (the cross K/V layout), handed back in the token-major [N][M] view.
__attribute__((visibility("default")))
int wb200_dbg_gemm(int wtype, int M, int N, int K, const void * w_file, const float * x, const float * bias,
                   float * out, int BN, int flags) {
    cudaStream_t st = 0;
    DevBuf<uint8_t> wraw; DevBuf<__half> xh; DevBuf<float> xf, dout, dbias;
    const size_t wbytes = (size_t) ((double) M * K * wt_bpw(wtype) + 0.5);
    if (!wraw.alloc(wbytes) || !xf.alloc((size_t) N * K) || !xh.alloc((size_t) N * K) || !dout.alloc((size_t) M * N)) return -1;
    WB_CUDA_OKV(cudaMemcpy(wraw.p, w_file, wbytes, cudaMemcpyHostToDevice), -2);
    WB_CUDA_OKV(cudaMemcpy(xf.p, x, (size_t) N * K * 4, cudaMemcpyHostToDevice), -2);
    if (bias) { if (!dbias.alloc(M)) return -1; WB_CUDA_OKV(cudaMemcpy(dbias.p, bias, (size_t) M * 4, cudaMemcpyHostToDevice), -2); }
    f32_to_f16(xf.p, xh.p, (int64_t) N * K, st);

    GemmDesc g;
    g.M = M; g.N = N; g.K = K; g.BN = BN;
    DevBuf<uint8_t> planar;
    if (wtype == WT_F16) {
        g.A.type = WT_F16; g.A.base = wraw.p;
        if (!make_tmap_f16(&g.tmA, wraw.p, K, M, 1, 1, K, 0, 0, 128)) return -3;
    } else if (wt_is_block32(wtype)) {
        if (!planar.alloc(wbytes + 64)) return -1;
        if (!repack_block32(wtype, wraw.p, planar.p, M, K, &g.A, st)) return -4;
    } else if (wt_is_kquant(wtype)) {
        g.A.type = wtype; g.A.N = M; g.A.K = K; g.A.base = wraw.p;
    } else { set_error("wb200_dbg_gemm: unsupported wtype %d", wtype); return -5; }
    if (!make_tmap_f16(&g.tmB, xh.p, K, N, 1, 1, K, 0, 0, (flags & 8) ? BN / 2 : BN)) return -3;
    if (flags & 8) g.half_box_b = 1;
    DevBuf<__half> a16;
    if (flags & 4) {
        g.v2 = 1;
        if (wtype != WT_F16) {
            if (!a16.alloc((size_t) M * K)) return -1;
            g.a16 = a16.p;
            if (!make_tmap_f16(&g.tmA, a16.p, K, M, 1, 1, K, 0, 0, 128)) return -3;
        }
    }
    g.ep.bias_m = bias ? dbias.p : nullptr;
    g.ep.act = (flags & 1) ? 1 : 0;
    g.ep.out = dout.p; g.ep.out_f16 = 0;
    g.ep.out_mmajor = (flags & 2) ? 1 : 0;
    g.ep.ldo = (flags & 2) ? N : M;
    DevBuf<__half> dout16;
    if (flags & 16) {                                            // f16 output (token-major), widened to f32 for the caller
        if (!dout16.alloc((size_t) M * N)) return -1;
        g.ep.out = dout16.p; g.ep.out_f16 = 1;
        if (flags & 64) {
            if (M % 64 || (flags & 2)) { set_error("wb200_dbg_gemm: head-major output needs M %% 64 == 0 and token-major flags"); return -5; }
            g.ep.hm_rows = N;
        }
    }
    if (flags & 32) {                                            // in-place f32 residual: `out` holds x on entry, x + W a on return
        WB_CUDA_OKV(cudaMemcpy(dout.p, out, (size_t) M * N * 4, cudaMemcpyHostToDevice), -2);
        g.ep.res = dout.p; g.ep.ldr = M;
    }
    cudaError_t e = gemm_launch(g, st);
    if (e != cudaSuccess) { set_error("gemm_launch: %s", cudaGetErrorString(e)); return -6; }
    e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error("gemm sync: %s", cudaGetErrorString(e)); return -7; }
    if (flags & 16) {
        std::vector<__half> h((size_t) M * N);
        WB_CUDA_OKV(cudaMemcpy(h.data(), dout16.p, (size_t) M * N * 2, cudaMemcpyDeviceToHost), -2);
        if (flags & 64) {
            for (int m = 0; m < M; ++m) for (int n = 0; n < N; ++n) out[(size_t) n * M + m] = __half2float(h[((size_t) (m / 64) * N + n) * 64 + (m % 64)]);
        } else
        for (size_t i = 0; i < h.size(); ++i) out[i] = __half2float(h[i]);
        return 0;
    }
    WB_CUDA_OKV(cudaMemcpy(out, dout.p, (size_t) M * N * 4, cudaMemcpyDeviceToHost), -2);
    return 0;
}



// encoder self-attention kernel alone: q, k, v f32 [n_win][T][H*64] (rounded to f16 on the way in), out f32 [n_win][T][H*64]; keys T..Tp-1 are
// the all-zero padding rows that take part in the softmax (SURVEY.md fact 4)
__attribute__((visibility("default")))
int wb200_dbg_fattn(const float * q, const float * k, const float * v, int T, int Tp, int H, int n_win, float scale, float * out) {
    cudaStream_t st = 0;
    const int d = H * 64;
    std::vector<__half> hqk((size_t) n_win * T * 2 * d), hvt((size_t) n_win * d * Tp, __float2half(0.0f));
    for (int w = 0; w < n_win; ++w)
        for (int t = 0; t < T; ++t)
            for (int e = 0; e < d; ++e) {
                const size_t i = ((size_t) w * T + t) * d + e;
                hqk[((size_t) w * T + t) * 2 * d + e]     = __float2half_rn(q[i]);
                hqk[((size_t) w * T + t) * 2 * d + d + e] = __float2half_rn(k[i]);
                hvt[((size_t) w * d + e) * Tp + t]        = __float2half_rn(v[i]);
            }
    DevBuf<__half> dqk, dvt, dout;
    if (!dqk.alloc(hqk.size()) || !dvt.alloc(hvt.size()) || !dout.alloc((size_t) n_win * T * d)) return -1;
    WB_CUDA_OKV(cudaMemcpy(dqk.p, hqk.data(), hqk.size() * 2, cudaMemcpyHostToDevice), -2);
    WB_CUDA_OKV(cudaMemcpy(dvt.p, hvt.data(), hvt.size() * 2, cudaMemcpyHostToDevice), -2);
    if (!fattn_encoder(dqk.p, 2 * d, d, dvt.p, T, Tp, H, n_win, scale, dout.p, d, st)) return -3;
    WB_CUDA_OKV(cudaStreamSynchronize(st), -4);
    std::vector<__half> ho((size_t) n_win * T * d);
    WB_CUDA_OKV(cudaMemcpy(ho.data(), dout.p, ho.size() * 2, cudaMemcpyDeviceToHost), -2);
    for (size_t i = 0; i < ho.size(); ++i) out[i] = __half2float(ho[i]);
    return 0;
}

// log-mel of a PCM buffer; mel_out [n_mel][n_len]; returns n_len (<0 on error)
__attribute__((visibility("default")))
int wb200_dbg_mel(const float * pcm, int n_samples, const float * filters, int n_mel, float * mel_out, int64_t cap) {
    const int n_len = (n_samples + 480000) / 160;
    if ((int64_t) n_mel * n_len > cap) return -1;
    DevBuf<float> dp, df, dm, dg;
    if (!dp.alloc(n_samples > 0 ? n_samples : 1) || !df.alloc((size_t) n_mel * 201) || !dm.alloc((size_t) n_mel * n_len) || !dg.alloc(4)) return -2;
    WB_CUDA_OKV(cudaMemcpy(dp.p, pcm, (size_t) n_samples * 4, cudaMemcpyHostToDevice), -3);
    WB_CUDA_OKV(cudaMemcpy(df.p, filters, (size_t) n_mel * 201 * 4, cudaMemcpyHostToDevice), -3);
    mel_spectrogram(dp.p, n_samples, df.p, n_mel, dm.p, n_len, dg.p, 0);
    WB_CUDA_OKV(cudaDeviceSynchronize(), -4);
    WB_CUDA_OKV(cudaMemcpy(mel_out, dm.p, (size_t) n_mel * n_len * 4, cudaMemcpyDeviceToHost), -3);
    return n_len;
}

__attribute__((visibility("default")))
int wb200_dbg_layernorm(const float * x, const float * w, const float * b, float eps, int rows, int d, float * out32, uint16_t * out16) {
    DevBuf<float> dx, dw, db, do32; DevBuf<__half> do16;
    if (!dx.alloc((size_t) rows * d) || !dw.alloc(d) || !db.alloc(d) || !do32.alloc((size_t) rows * d) || !do16.alloc((size_t) rows * d)) return -1;
    cudaMemcpy(dx.p, x, (size_t) rows * d * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(dw.p, w, (size_t) d * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(db.p, b, (size_t) d * 4, cudaMemcpyHostToDevice);
    layernorm(dx.p, dw.p, db.p, eps, rows, d, do16.p, do32.p, 0);
    WB_CUDA_OKV(cudaDeviceSynchronize(), -4);
    cudaMemcpy(out32, do32.p, (size_t) rows * d * 4, cudaMemcpyDeviceToHost);
    cudaMemcpy(out16, do16.p, (size_t) rows * d * 2, cudaMemcpyDeviceToHost);
    return 0;
}

// y[t][n] via the decode GEMV; weights in FILE layout.  flags bit0 gelu, bit1 fused LayerNorm (ln_w, ln_b given), bit2 = v2 (mma) kernel
__attribute__((visibility("default")))
int wb200_dbg_gemv(int wtype, int N, int K, int n_tok, const void * w_file, const float * x, const float * bias,
                   const float * scale, const float * res, const float * ln_w, const float * ln_b, float * out, int flags) {
    cudaStream_t st = 0;
    const size_t wbytes = (size_t) ((double) N * K * wt_bpw(wtype) + 0.5);
    DevBuf<uint8_t> wraw, planar; DevBuf<float> dx, dbias, dscale, dres, dlw, dlb, dout;
    if (!wraw.alloc(wbytes) || !dx.alloc((size_t) n_tok * K) || !dout.alloc((size_t) n_tok * N)) return -1;
    cudaMemcpy(wraw.p, w_file, wbytes, cudaMemcpyHostToDevice);
    cudaMemcpy(dx.p, x, (size_t) n_tok * K * 4, cudaMemcpyHostToDevice);
    GemvArgs a;
    if (wtype == WT_F16 || wt_is_kquant(wtype)) { a.W.type = wtype; a.W.N = N; a.W.K = K; a.W.base = wraw.p; }
    else if (wt_is_block32(wtype)) { if (!planar.alloc(wbytes + 64)) return -1; if (!repack_block32(wtype, wraw.p, planar.p, N, K, &a.W, st)) return -4; }
    else return -5;
    if (bias)  { dbias.alloc(N);  cudaMemcpy(dbias.p, bias, (size_t) N * 4, cudaMemcpyHostToDevice); a.bias = dbias.p; }
    if (scale) { dscale.alloc(N); cudaMemcpy(dscale.p, scale, (size_t) N * 4, cudaMemcpyHostToDevice); a.scale = dscale.p; }
    if (res)   { dres.alloc((size_t) n_tok * N); cudaMemcpy(dres.p, res, (size_t) n_tok * N * 4, cudaMemcpyHostToDevice); a.res = dres.p; }
    if (flags & 2) { dlw.alloc(K); dlb.alloc(K); cudaMemcpy(dlw.p, ln_w, (size_t) K * 4, cudaMemcpyHostToDevice); cudaMemcpy(dlb.p, ln_b, (size_t) K * 4, cudaMemcpyHostToDevice); a.ln_w = dlw.p; a.ln_b = dlb.p; }
    a.x = dx.p; a.n_tok = n_tok; a.act = (flags & 1) ? 1 : 0; a.out = dout.p;
    DevBuf<uint8_t> scratch;
    if (flags & 4) { if (!scratch.alloc(8 * act_tok_stride(a.W.type, K))) return -1; gemv2(a, scratch.p, st); }
    else gemv(a, st);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { set_error("gemv: %s", cudaGetErrorString(e)); return -7; }
    cudaMemcpy(out, dout.p, (size_t) n_tok * N * 4, cudaMemcpyDeviceToHost);
    return 0;
}

// decode attention kernels.  kc/vc given as f16 bit patterns [n_cells][d]
__attribute__((visibility("default")))
int wb200_dbg_attn_self(const float * q, const uint16_t * kc, const uint16_t * vc, const int * idx, int ld_idx, const int * n_kv,
                        int n_tok, int n_head, int n_cells, float * out) {
    const int d = n_head * 64;
    DevBuf<float> dq, dout; DevBuf<__half> dk, dv; DevBuf<int> di, dn;
    dq.alloc((size_t) n_tok * d); dout.alloc((size_t) n_tok * d); dk.alloc((size_t) n_cells * d); dv.alloc((size_t) n_cells * d);
    di.alloc((size_t) n_tok * ld_idx); dn.alloc(n_tok);
    cudaMemcpy(dq.p, q, (size_t) n_tok * d * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(dk.p, kc, (size_t) n_cells * d * 2, cudaMemcpyHostToDevice);
    cudaMemcpy(dv.p, vc, (size_t) n_cells * d * 2, cudaMemcpyHostToDevice);
    cudaMemcpy(di.p, idx, (size_t) n_tok * ld_idx * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(dn.p, n_kv, (size_t) n_tok * 4, cudaMemcpyHostToDevice);
    attn_self_decode(dq.p, d, dk.p, dv.p, di.p, ld_idx, dn.p, n_tok, n_head, d, dout.p, d, 0);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { set_error("attn_self: %s", cudaGetErrorString(e)); return -7; }
    cudaMemcpy(out, dout.p, (size_t) n_tok * d * 4, cudaMemcpyDeviceToHost);
    return 0;
}
__attribute__((visibility("default")))
int wb200_dbg_attn_cross(const float * q, const uint16_t * kc, const uint16_t * vc, int n_keys, int n_tok, int n_head, float scale, float * out) {
    const int d = n_head * 64;
    DevBuf<float> dq, dout, dpart; DevBuf<__half> dk, dv; DevBuf<int> dslot, dcnt;
    dq.alloc((size_t) n_tok * d); dout.alloc((size_t) n_tok * d); dk.alloc((size_t) n_tok * n_keys * d); dv.alloc((size_t) n_tok * n_keys * d);
    dpart.alloc((size_t) n_tok * n_head * 32 * 66); dslot.alloc(n_tok); dcnt.alloc((size_t) n_tok * n_head, true);
    std::vector<int> slots(n_tok); for (int i = 0; i < n_tok; ++i) slots[i] = i;
    cudaMemcpy(dslot.p, slots.data(), (size_t) n_tok * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(dq.p, q, (size_t) n_tok * d * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(dk.p, kc, (size_t) n_tok * n_keys * d * 2, cudaMemcpyHostToDevice);
    cudaMemcpy(dv.p, vc, (size_t) n_tok * n_keys * d * 2, cudaMemcpyHostToDevice);
    for (int rep = 0; rep < 2; ++rep)   // twice: the second run checks that the arrival counters were reset
        attn_cross_decode(dq.p, d, dk.p, dv.p, dslot.p, (int64_t) n_keys * d, n_keys, n_tok, n_head, d, scale, dpart.p, dcnt.p, dout.p, d, 0);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { set_error("attn_cross: %s", cudaGetErrorString(e)); return -7; }
    cudaMemcpy(out, dout.p, (size_t) n_tok * d * 4, cudaMemcpyDeviceToHost);
    return 0;
}

// W [N][K] in FILE layout -> tile-major records on the device (the decoder's layout) -> every element read back through the token-embedding
// reader: out f32 [N][K]
__attribute__((visibility("default")))
int wb200_dbg_tm_dequant(int wtype, int N, int K, const void * w_file, float * out) {
    if (wt_tm_rec_bytes(wtype) == 0 || K % wt_tm_rec_k(wtype) || K % 32) { set_error("wb200_dbg_tm_dequant: no tile-major layout for type %d, K=%d", wtype, K); return -5; }
    DevBuf<uint8_t> wraw, tm; DevBuf<float> dout;
    const size_t wbytes = (size_t) ((double) N * K * wt_bpw(wtype) + 0.5);
    if (!wraw.alloc(wbytes) || !tm.alloc(wt_tm_bytes(wtype, N, K), true) || !dout.alloc((size_t) N * K)) return -1;
    WB_CUDA_OKV(cudaMemcpy(wraw.p, w_file, wbytes, cudaMemcpyHostToDevice), -2);
    QMat W; W.type = wtype; W.N = N; W.K = K; W.base = tm.p; W.layout = 1;
    if (!repack_tile_major(wtype, wraw.p, W, 0, N, 0)) return -4;
    dequant_rows_f32(W, dout.p, 0);
    WB_CUDA_OKV(cudaMemcpy(out, dout.p, (size_t) N * K * 4, cudaMemcpyDeviceToHost), -2);
    return 0;
}

// W [N][K] in FILE layout -> planar 32-blocks (K-quants: the verbatim super-blocks) on the device (the encoder's and the kernel chain's
// layout) -> every element read back through the token-embedding reader: out f32 [N][K]
__attribute__((visibility("default")))
int wb200_dbg_planar_dequant(int wtype, int N, int K, const void * w_file, float * out) {
    if (!(wt_is_block32(wtype) || wt_is_kquant(wtype)) || K % wt_tm_rec_k(wtype)) { set_error("wb200_dbg_planar_dequant: no planar layout for type %d, K=%d", wtype, K); return -5; }
    DevBuf<uint8_t> wraw, planar; DevBuf<float> dout;
    const size_t wbytes = (size_t) ((double) N * K * wt_bpw(wtype) + 0.5);
    if (!wraw.alloc(wbytes) || !planar.alloc(wbytes + 64) || !dout.alloc((size_t) N * K)) return -1;
    WB_CUDA_OKV(cudaMemcpy(wraw.p, w_file, wbytes, cudaMemcpyHostToDevice), -2);
    QMat W;
    if (wt_is_kquant(wtype)) { W.type = wtype; W.N = N; W.K = K; W.base = wraw.p; }
    else if (!repack_block32(wtype, wraw.p, planar.p, N, K, &W, 0)) return -4;
    dequant_rows_f32(W, dout.p, 0);
    WB_CUDA_OKV(cudaMemcpy(out, dout.p, (size_t) N * K * 4, cudaMemcpyDeviceToHost), -2);
    return 0;
}

// One phase of the persistent decode kernel (mk_probe_launch) from host buffers.  Row buffers have the pass's 64 rows; the phase works on
// rows [row0, row0 + n_tok) with n_cta CTAs.  `out` is copied to the device before the launch and back after it, so a sentinel fill shows
// every write.  Per phase (wb_decode_mk.cuh MkProbePhase; actq(K) = the decode kernel's quantised rows of length K, wb_decode_mk.cu):
//   LNQ:   in = f32 [64][K], bias / scale = LayerNorm b / w [K]            -> out = actq(K)
//   Q8K:   in = f32 [64][lds]                                              -> out = actq(K)
//   GEMV:  w_file [N][K], in = actq(K), bias / scale [N], res [64][N], act -> out = f32 [64][N]; with kv_d > 0 outputs [kv_d, 3 kv_d) are
//          appended as f16 to kc / vc [n_cells][kv_d] (in / out) at cell[64]
//   GEMV_PAIR (FC1): w_file [N][K], in = actq(K), bias [N]; always GELU   -> out = actq(N)
//   LOGITS_WARP: w_file [N][K], in = actq(K)                               -> out = f32 [64][N]
//   ATTN_SELF:  in = f32 qkv rows [64][3d], kc / vc [n_cells][d], nkv [64], idx [64][ld_idx] -> out = actq(d) (K-quants: f32 [64][d])
//   ATTN_CROSS: in = f32 q rows [64][d], xk / xv head-major [n_slots][n_head][kv_rows][64], slot [64] -> out = actq(d) (K-quants: f32 [64][3d],
//          columns 0 .. d-1 written); N = encoder positions (MkArgs::n_audio_ctx, 0: n_keys): keys N .. n_keys - 1 count as zero rows;
//          kv_rows = rows per head of the buffer (MkArgs::kv_rows, 0: n_keys), the engine's is its largest padded context
struct Wb200MkPhaseIo {
    int wtype, phase, n_cta, row0, n_tok;
    int N, K, lds, act, kv_d;
    const void * w_file;
    const void * in; int64_t in_bytes;
    const float * bias, * scale, * res;
    void * out; int64_t out_bytes;
    const int * cell;
    uint16_t * kc, * vc; int n_cells;
    int d, n_head, ld_idx;
    const int * nkv, * idx;
    const uint16_t * xk, * xv; int n_keys, n_slots;
    const int * slot;
    float kq_scale, eps;
    int kv_rows;
};

__attribute__((visibility("default")))
int wb200_dbg_mk_phase(const Wb200MkPhaseIo * io) {
    constexpr int R = 64;
    const Wb200MkPhaseIo & s = *io;
    const bool kq = wt_is_kquant(s.wtype);
    MkArgs a = {};
    MkProbe p = {};
    p.phase = s.phase; p.row0 = s.row0; p.n_tok = s.n_tok; p.act = s.act; p.kv_d = s.kv_d; p.lds = s.lds; p.K = s.K;
    a.d = s.d; a.n_head = s.n_head; a.n_tok = s.row0 + s.n_tok; a.n_keys = s.n_keys; a.ld_idx = s.ld_idx;
    a.kq_scale = s.kq_scale; a.eps = s.eps; a.prefetch = 4;     // cross K/V streamed with the evict-first hint, as the engine launches it
    DevBuf<uint8_t> wraw, tm, din, dout; DevBuf<float> dbias, dscale, dres, dqkv, dq2;
    DevBuf<int> dcell, dnkv, didx, dslot; DevBuf<__half> dkc, dvc, dxk, dxv; DevBuf<MkLayer> dL; DevBuf<QMat> dW;
    if (!din.alloc(s.in_bytes) || !dout.alloc(s.out_bytes)) return -1;
    WB_CUDA_OKV(cudaMemcpy(din.p, s.in, s.in_bytes, cudaMemcpyHostToDevice), -2);
    WB_CUDA_OKV(cudaMemcpy(dout.p, s.out, s.out_bytes, cudaMemcpyHostToDevice), -2);
    auto up_f = [&](DevBuf<float> & b, const float * h, size_t n) { if (!h) return true; if (!b.alloc(n)) return false; return cudaMemcpy(b.p, h, n * 4, cudaMemcpyHostToDevice) == cudaSuccess; };
    auto up_i = [&](DevBuf<int> & b, const int * h, size_t n) { if (!h) return true; if (!b.alloc(n)) return false; return cudaMemcpy(b.p, h, n * 4, cudaMemcpyHostToDevice) == cudaSuccess; };
    auto up_h = [&](DevBuf<__half> & b, const uint16_t * h, size_t n) { if (!h) return true; if (!b.alloc(n)) return false; return cudaMemcpy(b.p, h, n * 2, cudaMemcpyHostToDevice) == cudaSuccess; };
    const bool gemv = s.phase == MKP_GEMV || s.phase == MKP_GEMV_PAIR || s.phase == MKP_LOGITS_WARP;
    if (gemv) {
        if (wt_tm_rec_bytes(s.wtype) == 0 || s.K % wt_tm_rec_k(s.wtype) || s.K % 32) { set_error("wb200_dbg_mk_phase: no tile-major layout for type %d, K=%d", s.wtype, s.K); return -5; }
        const size_t wbytes = (size_t) ((double) s.N * s.K * wt_bpw(s.wtype) + 0.5);
        if (!wraw.alloc(wbytes) || !tm.alloc(wt_tm_bytes(s.wtype, s.N, s.K), true)) return -1;
        WB_CUDA_OKV(cudaMemcpy(wraw.p, s.w_file, wbytes, cudaMemcpyHostToDevice), -2);
        p.W.type = s.wtype; p.W.N = s.N; p.W.K = s.K; p.W.base = tm.p; p.W.layout = 1;
        if (!repack_tile_major(s.wtype, wraw.p, p.W, 0, s.N, 0)) return -4;
        if (!dW.alloc(1)) return -1;
        WB_CUDA_OKV(cudaMemcpy(dW.p, &p.W, sizeof(QMat), cudaMemcpyHostToDevice), -2);
        p.Wg = dW.p;
        p.x = din.p;
        if (!up_f(dbias, s.bias, s.N) || !up_f(dscale, s.scale, s.N) || !up_f(dres, s.res, (size_t) R * s.N) || !up_i(dcell, s.cell, R)) return -1;
        p.bias = dbias.p; p.scale = dscale.p; p.res = dres.p; a.cell = dcell.p;
        if (s.phase == MKP_GEMV_PAIR) p.dst = dout.p; else p.out = reinterpret_cast<float *>(dout.p);
        if (s.kv_d > 0) {
            if (!s.cell || !up_h(dkc, s.kc, (size_t) s.n_cells * s.kv_d) || !up_h(dvc, s.vc, (size_t) s.n_cells * s.kv_d)) return -1;
            p.kc = dkc.p; p.vc = dvc.p;
        }
    } else if (s.phase == MKP_LNQ || s.phase == MKP_Q8K) {
        p.src = reinterpret_cast<const float *>(din.p); p.dst = dout.p;
        if (s.phase == MKP_LNQ && (!up_f(dscale, s.scale, s.K) || !up_f(dbias, s.bias, s.K))) return -1;
        p.scale = dscale.p; p.bias = dbias.p;
    } else if (s.phase == MKP_ATTN_SELF || s.phase == MKP_ATTN_CROSS) {
        MkLayer L = {};
        const bool self = s.phase == MKP_ATTN_SELF;
        if (!dqkv.alloc((size_t) R * 3 * s.d) || !dq2.alloc((size_t) R * s.d)) return -1;
        float * const q_in = self ? dqkv.p : dq2.p;
        WB_CUDA_OKV(cudaMemcpy(q_in, din.p, s.in_bytes, cudaMemcpyDeviceToDevice), -2);
        if (kq) { if (self) a.q2 = reinterpret_cast<float *>(dout.p); else a.qkv = reinterpret_cast<float *>(dout.p); }
        else a.actq = dout.p;
        if (!a.qkv) a.qkv = dqkv.p;
        if (!a.q2) a.q2 = dq2.p;
        if (self) {
            if (!up_h(dkc, s.kc, (size_t) s.n_cells * s.d) || !up_h(dvc, s.vc, (size_t) s.n_cells * s.d) || !up_i(dnkv, s.nkv, R) || !up_i(didx, s.idx, (size_t) R * s.ld_idx)) return -1;
            L.kc = dkc.p; L.vc = dvc.p; a.nkv = dnkv.p; a.idx = didx.p;
        } else {
            const int rows = s.kv_rows > 0 ? s.kv_rows : s.n_keys;
            const size_t n = (size_t) s.n_slots * rows * s.d;
            if (s.n_keys % 128) { set_error("wb200_dbg_mk_phase: n_keys %d is not a multiple of 128", s.n_keys); return -5; }
            if (s.N < 0 || s.N > s.n_keys) { set_error("wb200_dbg_mk_phase: %d encoder positions for %d keys", s.N, s.n_keys); return -5; }
            if (rows < s.n_keys) { set_error("wb200_dbg_mk_phase: %d rows per head for %d keys", rows, s.n_keys); return -5; }
            a.n_audio_ctx = s.N > 0 ? s.N : s.n_keys; a.kv_rows = rows;
            if (!up_h(dxk, s.xk, n) || !up_h(dxv, s.xv, n) || !up_i(dslot, s.slot, R)) return -1;
            L.xk = dxk.p; L.xv = dxv.p; a.slot = dslot.p; a.slot_stride = (int64_t) rows * s.d;
        }
        if (!dL.alloc(1)) return -1;
        WB_CUDA_OKV(cudaMemcpy(dL.p, &L, sizeof(L), cudaMemcpyHostToDevice), -2);
        p.L = dL.p;
    }
    if (!mk_probe_launch(a, p, s.wtype, s.n_cta, 0)) return -6;
    const cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { set_error("decode kernel probe: %s", cudaGetErrorString(e)); return -7; }
    WB_CUDA_OKV(cudaMemcpy(s.out, dout.p, s.out_bytes, cudaMemcpyDeviceToHost), -2);
    if (s.kc && s.phase == MKP_GEMV && s.kv_d > 0) {
        WB_CUDA_OKV(cudaMemcpy(s.kc, dkc.p, (size_t) s.n_cells * s.kv_d * 2, cudaMemcpyDeviceToHost), -2);
        WB_CUDA_OKV(cudaMemcpy(s.vc, dvc.p, (size_t) s.n_cells * s.kv_d * 2, cudaMemcpyDeviceToHost), -2);
    }
    return 0;
}

} // extern "C"

// wb_engine.cu -- see wb_engine.h.  Graph structure follows whisper_build_graph_conv / _encoder / _cross / _decoder
// (src/whisper.cpp:1982-2042, 2044-2275, 2278-2354, 2466-2844); every `ggml_mul_mat (+add/scale/gelu/cpy)` group of the
// reference is one wgmma GEMM launch (encode) or one fused GEMV launch (decode step) here.
#include <algorithm>
#include <cmath>
#include <chrono>
#include <cstring>
#include "wb_engine.h"
#include "wb_dtw_kernel.cuh"
#include "wb_kernels.cuh"

namespace wb {

static inline int pad256(int n) { return (n + 255) / 256 * 256; }

struct EncLayerPlan { GemmDesc qk, v, s, pv, o, fc1, fc2; };
struct EncPlan {
    int n_ctx = 0, n_win = 0;
    GemmDesc conv1, conv2, conv2_tap, cross;
    std::vector<EncLayerPlan> layers;
};

void Engine::drop_graphs() {
    for (auto & kv : graphs) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
    graphs.clear();
}

Engine::~Engine() {
    if (m) cudaSetDevice(m->device);
    if (st) cudaStreamSynchronize(st);                            // a run-ahead pass may still be queued
    mk_trace_dump();
    drop_graphs();
    delete plan;
    for (PassSlot & s : pslot) {
        if (s.hints) cudaFreeHost(s.hints);
        if (s.hsamp) cudaFreeHost(s.hsamp);
        if (s.ev0) cudaEventDestroy(s.ev0);
        if (s.ev1) cudaEventDestroy(s.ev1);
    }
    if (hlogits) cudaFreeHost(hlogits);
    if (hdraws) cudaFreeHost(hdraws);
    for (auto & e : ev) if (e) cudaEventDestroy(e);
    if (st) cudaStreamDestroy(st);
}

bool Engine::init(const Model * model, int cap_windows) {
    m = model; cap_win = std::max(1, cap_windows);
    WB_CUDA_OK(cudaSetDevice(m->device));
    WB_CUDA_OK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    for (auto & e : ev) WB_CUDA_OK(cudaEventCreate(&e));
    for (PassSlot & s : pslot) { WB_CUDA_OK(cudaEventCreate(&s.ev0)); WB_CUDA_OK(cudaEventCreate(&s.ev1)); }
    const HParams & hp = m->hp;
    const int d = hp.n_audio_state, H = hp.n_audio_head, T = hp.n_audio_ctx, Tp = pad256(T), M = hp.n_mels, Lt = hp.n_text_layer, V = hp.n_vocab;
    const size_t B = cap_win;
    Tp_max = Tp;
    debug_taps = getenv("WB200_DEBUG_TAPS") != nullptr;
    use_graphs = getenv("WB200_NO_GRAPHS") == nullptr;
    fused_attn = getenv("WB200_UNFUSED_ATTN") == nullptr;
    gemm_v2 = getenv("WB200_GEMM_V1") == nullptr;
    if (gemm_v2 && m->wtype != WT_F16 && m->wtype != WT_F32 && !m->cross_kv.f16) {
        const size_t dd = (size_t) hp.n_audio_state * hp.n_audio_state;
        if (!wf16.alloc(std::max<size_t>(4 * dd, (size_t) 2 * hp.n_text_layer * dd))) return false;
    }
    gemv_v2 = getenv("WB200_GEMV_V1") == nullptr;
    (void) B; (void) H; (void) M; (void) Tp;
    if (!alloc_encoder_ws() || !kv_cross.alloc((size_t) cap_win * 2 * Lt * Tp * d, true)) return false;
    slot_ctx.assign((size_t) cap_win, 0);
    {
        cudaDeviceProp prop; WB_CUDA_OK(cudaGetDeviceProperties(&prop, m->device));
        n_sm = prop.multiProcessorCount;
        use_mk = m->dec_tm;
        max_rows = use_mk ? mk_max_rows() : 8;                   // the layout decides: tile-major decoder weights <=> persistent kernel
        if (use_mk && (!mk_supported(m->wtype == WT_F32 ? WT_F16 : m->wtype) || mk_smem_bytes(m->wtype == WT_F32 ? WT_F16 : m->wtype, hp.n_text_state) > 227 * 1024 || !prop.cooperativeLaunch)) {
            set_error("decode: the persistent kernel cannot run on this device/model; set WB200_MEGAKERNEL=0"); return false;
        }
        if (const char * pf = getenv("WB200_MK_PREFETCH")) mk_prefetch = atoi(pf);
        // slower than the first generation where it was measured (DESIGN.md section 4), kept for the A/B
        if (use_mk && !mk_bar.alloc(mk_bar_words(n_sm), true)) return false;
        // WB200_MK_PARTS=1..4: partitions of a pass of 32 rows or more (1 = every CTA on one barrier); WB200_MK_TURNS: partitions that may
        // stream cross K/V at the same time.  Defaults: what measured fastest at 64 rows (DESIGN.md section 4)
        if (const char * np = getenv("WB200_MK_PARTS")) mk_parts = std::min(std::max(atoi(np), 1), MK_MAX_PARTS);
        if (const char * ts = getenv("WB200_MK_TURNS")) mk_turns = std::min(std::max(atoi(ts), 1), MK_MAX_PARTS);
        sm_ghz = prop.clockRate * 1e-6;
        if (const char * tp = getenv("WB200_MK_TRACE")) { if (use_mk && *tp) { mk_trace_path = tp; if (!mk_trace.alloc(4096, true)) return false; } }
    }
    // decoder workspaces (max_rows rows per pass)
    const size_t R = max_rows;
    if (!dx.alloc(R * d) || !dqkv.alloc(R * 3 * d) || !dattn.alloc(R * d) || !dq2.alloc(R * d) || !dh.alloc(R * 4 * d) ||
        !dlogits.alloc(R * V) || !xpart.alloc(R * H * 32 * 66) || !xcnt.alloc(R * H, true)) return false;
    if (use_mk && !dhq.alloc(R * 4 * d * 2 + R * 4 * d / 8 + 256)) return false;
    if (!act_scratch.alloc(8 * act_tok_stride(m->wtype == WT_F32 ? WT_F16 : m->wtype, 4 * d) + 256)) return false;
    if (!set_cells(pad256(hp.n_text_ctx))) return false;
    WB_CUDA_OK(cudaMallocHost(&hlogits, (size_t) max_rows * V * sizeof(float)));
    for (PassSlot & s : pslot) WB_CUDA_OK(cudaMallocHost(&s.hsamp, (size_t) max_rows * SAMP_MAX_DRAWS * sizeof(SampOut)));
    WB_CUDA_OK(cudaMallocHost(&hdraws, (size_t) max_rows * SAMP_MAX_DRAWS * sizeof(double)));
    if (!dsamp.alloc((size_t) PASS_SLOTS * max_rows * SAMP_MAX_DRAWS) || !ddraws.alloc((size_t) max_rows * SAMP_MAX_DRAWS) || !samp_mask.alloc((size_t) (V + 31) / 32, true)) return false;
    return true;
}

// encoder workspaces for cap_win windows per batched pass (transient contents)
bool Engine::alloc_encoder_ws() {
    const HParams & hp = m->hp;
    const int d = hp.n_audio_state, H = hp.n_audio_head, T = hp.n_audio_ctx, Tp = pad256(T), M = hp.n_mels;
    const size_t B = cap_win;
    if (!mel_win.alloc(B * (2*T + 2) * M, true) || !h1.alloc(B * (2*T + 2) * d, true) || !x.alloc(B * T * d) || !xn.alloc(B * T * d) ||
        !qk.alloc(B * T * 2 * d) || !vt.alloc(B * d * Tp, true) || (!fused_attn && (!S.alloc(B * H * T * Tp) || !P.alloc(B * H * T * Tp))) ||
        !attn.alloc(B * T * d) || !hfc.alloc(B * T * 4 * d) || !enc16.alloc(B * T * d)) return false;
    if (debug_taps && (!enc32.alloc(B * T * d) || !conv32.alloc(B * T * d))) return false;
    delete plan; plan = nullptr;                                  // tensor maps point into the old buffers
    return true;
}

bool Engine::resize(int new_cap, int new_cps) {
    const HParams & hp = m->hp;
    WB_CUDA_OK(cudaSetDevice(m->device));
    WB_CUDA_OK(cudaStreamSynchronize(st));
    const int Lt = hp.n_text_layer, d = hp.n_text_state, Tp = Tp_max;
    const int old_cap = cap_win, old_cps = cps, keep = std::min(old_cap, new_cap);
    drop_graphs();
    if (new_cap != old_cap) {
        cap_win = new_cap;
        if (!alloc_encoder_ws()) return false;
        const size_t slot_e = (size_t) 2 * Lt * Tp * d;
        DevBuf<__half> nx;
        if (!nx.alloc((size_t) new_cap * slot_e, true)) return false;
        if (kv_cross.p) WB_CUDA_OK(cudaMemcpy(nx.p, kv_cross.p, (size_t) keep * slot_e * sizeof(__half), cudaMemcpyDeviceToDevice));
        std::swap(nx.p, kv_cross.p); std::swap(nx.n, kv_cross.n);
        slot_ctx.resize((size_t) new_cap, 0);                     // the context length of each surviving slot's cross K/V goes with it
    }
    if (new_cap != old_cap || new_cps != old_cps || !kv_k.p) {
        const size_t e = (size_t) Lt * new_cap * new_cps * d;
        DevBuf<__half> nk, nv;
        if (!nk.alloc(e, true) || !nv.alloc(e, true)) return false;
        if (kv_k.p && old_cps > 0) {
            const size_t w = (size_t) std::min(old_cps, new_cps) * d * sizeof(__half);
            for (int s = 0; s < keep; ++s) {                       // [layer][slot][cell][d]: one 2-D copy per slot, a row per layer
                WB_CUDA_OK(cudaMemcpy2D(nk.p + (size_t) s * new_cps * d, (size_t) new_cap * new_cps * d * sizeof(__half),
                                        kv_k.p + (size_t) s * old_cps * d, (size_t) old_cap * old_cps * d * sizeof(__half), w, Lt, cudaMemcpyDeviceToDevice));
                WB_CUDA_OK(cudaMemcpy2D(nv.p + (size_t) s * new_cps * d, (size_t) new_cap * new_cps * d * sizeof(__half),
                                        kv_v.p + (size_t) s * old_cps * d, (size_t) old_cap * old_cps * d * sizeof(__half), w, Lt, cudaMemcpyDeviceToDevice));
            }
        }
        std::swap(nk.p, kv_k.p); std::swap(nk.n, kv_k.n); std::swap(nv.p, kv_v.p); std::swap(nv.n, kv_v.n);
        cps = new_cps; n_cells = new_cap * new_cps;
    }
    WB_CUDA_OK(cudaDeviceSynchronize());
    if (use_mk && !mk_build_table()) return false;
    return true;
}

bool Engine::set_cells(int n) {
    const HParams & hp = m->hp;
    WB_CUDA_OK(cudaSetDevice(m->device));
    WB_CUDA_OK(cudaStreamSynchronize(st));                        // queued passes read the buffers and row tables replaced here
    drop_graphs();
    n_cells = n; cps = n / std::max(1, cap_win);
    const size_t e = (size_t) hp.n_text_layer * n * hp.n_text_state;
    if (!kv_k.alloc(e, true) || !kv_v.alloc(e, true)) return false;
    ld_idx = pad256(hp.n_text_ctx);          // a query attends to at most n_text_ctx positions
    const size_t nints = (size_t) max_rows * (8 + ld_idx);
    if (!dints.alloc(nints)) return false;
    for (PassSlot & s : pslot) {
        if (s.hints) cudaFreeHost(s.hints);
        s.hints = nullptr;
        WB_CUDA_OK(cudaMallocHost(&s.hints, nints * sizeof(int)));
    }
    if (use_mk && !mk_build_table()) return false;
    return true;
}

void Engine::mk_trace_collect(int n_layer, bool logits) {
    const int ns = 1 + 24 * n_layer + (logits ? 3 : 0);
    std::vector<long long> h(ns);
    if (cudaMemcpy(h.data(), mk_trace.p, ns * sizeof(long long), cudaMemcpyDeviceToHost) != cudaSuccess) return;
    if (mk_trace_sum.empty()) mk_trace_sum.assign(28, 0.0);
    for (int l = 0; l < n_layer; ++l)
        for (int k = 0; k < 24; ++k) mk_trace_sum[k] += (double) (h[1 + 24 * l + k] - h[24 * l + k]) / n_layer;
    if (logits) { mk_trace_sum[24] += (double) (h[ns - 3] - h[ns - 4]); mk_trace_sum[25] += (double) (h[ns - 2] - h[ns - 3]); mk_trace_sum[26] += (double) (h[ns - 1] - h[ns - 2]); }
    mk_trace_sum[27] += (double) (h[ns - 1] - h[0]);
    {   // sub-phase stamps of the six GEMV phases of layer 1 (MK_FINE)
        std::vector<long long> f(48);
        if (cudaMemcpy(f.data(), mk_trace.p + 2048, 48 * sizeof(long long), cudaMemcpyDeviceToHost) == cudaSuccess) {
            if (mk_fine.empty()) mk_fine.assign(30, 0.0);
            for (int g = 0; g < 6; ++g) for (int k = 0; k < 5; ++k) mk_fine[5 * g + k] += (double) (f[8 * g + k + 1] - f[8 * g + k]);
        }
    }
    {   // SM clocks the CTA that releases partition 0 waited for the partition's turn to stream cross K/V (the kernel accumulates)
        long long w = 0;
        if (cudaMemcpy(&w, mk_trace.p + 2100, sizeof(w), cudaMemcpyDeviceToHost) == cudaSuccess) mk_turn_clk += (double) w / n_layer;
        cudaMemset(mk_trace.p + 2100, 0, sizeof(long long));
    }
    ++mk_trace_n;
}
void Engine::mk_trace_dump() {
    if (mk_trace_path.empty() || !mk_trace_n) return;
    FILE * f = fopen(mk_trace_path.c_str(), "a");
    if (!f) return;
    static const char * ph[12] = { "1 ln->q8", "2 qkv", "3 self-attn", "4 o-proj", "5 ln->q8", "6 cross-q", "7 cross-attn", "8 cross-o", "9 ln->q8", "10 fc1+gelu", "10b h->q8", "11 fc2" };
    const double us = 1e-3 / sm_ghz / (double) mk_trace_n;
    fprintf(f, "# persistent decode kernel, CTA 0, average over %llu passes with logits (us; SM clock %.3f GHz)\n", (unsigned long long) mk_trace_n, sm_ghz);
    fprintf(f, "%-16s %10s %10s\n", "phase (per layer)", "work", "barrier");
    double tot = 0.0;
    for (int p = 0; p < 12; ++p) {
        fprintf(f, "%-16s %10.2f %10.2f\n", ph[p], mk_trace_sum[2*p] * us, mk_trace_sum[2*p + 1] * us);
        tot += (mk_trace_sum[2*p] + mk_trace_sum[2*p + 1]) * us;
    }
    if (!mk_fine.empty()) {
        static const char * gn[6] = { "qkv", "o", "cross-q", "cross-o", "fc1", "fc2" };
        fprintf(f, "GEMV sub-phases, layer 1 (us): stage rows | k-loop of the first iteration | partials->smem + sync | epilogue + sync | remaining iterations\n");
        for (int g = 0; g < 6; ++g) fprintf(f, "  %-8s %7.2f %7.2f %7.2f %7.2f %7.2f\n", gn[g], mk_fine[5*g] * us, mk_fine[5*g+1] * us, mk_fine[5*g+2] * us, mk_fine[5*g+3] * us, mk_fine[5*g+4] * us);
    }
    fprintf(f, "partitions %d, turns %d: wait of partition 0 for its turn to stream cross K/V %.2f us per layer (inside the barrier of 6 cross-q)\n", mk_parts, mk_turns, mk_turn_clk * us);
    fprintf(f, "layer total %.2f us; final ln %.2f + barrier %.2f us, logits %.2f us; whole pass %.1f us\n", tot, mk_trace_sum[24] * us, mk_trace_sum[25] * us, mk_trace_sum[26] * us, mk_trace_sum[27] * us);
    fclose(f);
}

// per-layer descriptor table of the persistent decode kernel (weights of the model + the KV buffers of this engine)
bool Engine::mk_build_table() {
    const HParams & hp = m->hp;
    const int Lt = hp.n_text_layer, d = hp.n_text_state, Tp = Tp_max;
    std::vector<MkLayer> tab(Lt);
    for (int l = 0; l < Lt; ++l) {
        const DecLayerW & L = m->dec[l];
        MkLayer & t = tab[l];
        t.qkv = L.qkv; t.o = L.o; t.cq = L.cq; t.co = L.co; t.fc1 = L.fc1; t.fc2 = L.fc2;
        t.ln0_w = L.ln0.w; t.ln0_b = L.ln0.b; t.lnc_w = L.lnc.w; t.lnc_b = L.lnc.b; t.lnm_w = L.lnm.w; t.lnm_b = L.lnm.b;
        t.qkv_bias = L.qkv_bias; t.qkv_scale = L.qkv_scale; t.o_bias = L.o_bias; t.cq_bias = L.cq_bias; t.co_bias = L.co_bias;
        t.fc1_bias = L.fc1_bias; t.fc2_bias = L.fc2_bias;
        t.kc = kv_k.p + (size_t) l * n_cells * d; t.vc = kv_v.p + (size_t) l * n_cells * d;
        t.xk = kv_cross.p + (size_t) l * Tp * d;  t.xv = kv_cross.p + (size_t) (Lt + l) * Tp * d;
        t.cap_mask = dtw_layer_mask.empty() ? 0u : dtw_layer_mask[l]; t.cap_head0 = dtw_layer_head0.empty() ? 0 : dtw_layer_head0[l];
    }
    if (!mk_layers.alloc(Lt)) return false;
    WB_CUDA_OK(cudaMemcpy(mk_layers.p, tab.data(), Lt * sizeof(MkLayer), cudaMemcpyHostToDevice));
    return true;
}

// ---------------------------------------------------------------------------------------------------- audio front-end
FrontEnd::~FrontEnd() {
    if (m) cudaSetDevice(m->device);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (st) cudaStreamDestroy(st);
}
bool FrontEnd::init(const Model * model) {
    m = model;
    WB_CUDA_OK(cudaSetDevice(m->device));
    WB_CUDA_OK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    WB_CUDA_OK(cudaEventCreate(&ev0)); WB_CUDA_OK(cudaEventCreate(&ev1));
    return gmax.alloc(4);
}
bool FrontEnd::pcm_upload(const float * samples, int n_samples) {
    WB_CUDA_OK(cudaSetDevice(m->device));
    if ((size_t) n_samples > pcm.n && !pcm.alloc(std::max(n_samples, 1))) return false;
    if (n_samples > 0) { WB_CUDA_OK(cudaMemcpyAsync(pcm.p, samples, (size_t) n_samples * 4, cudaMemcpyHostToDevice, st)); count_h2d((uint64_t) n_samples * 4); }
    WB_CUDA_OK(cudaStreamSynchronize(st));
    pcm_resident = n_samples;
    return true;
}
bool FrontEnd::pcm_to_mel(const float * samples, int n_samples, bool samples_on_device) {
    NvtxRange nvtx("wb200.mel");
    WB_CUDA_OK(cudaSetDevice(m->device));
    if (!samples && n_samples > 0 && pcm_resident != n_samples) { set_error("pcm_to_mel: no host samples and no resident PCM of %d samples", n_samples); return false; }
    n_mel = m->n_filt_mel;
    n_len = (n_samples + 480000) / 160;                       // whisper.cpp:3202-3218
    n_len_org = 1 + (n_samples + 200 - 400) / 160;            // whisper.cpp:3220
    if (samples && !samples_on_device) pcm_resident = 0;
    if (!samples_on_device && (size_t) std::max(n_samples, 1) > pcm.n && !pcm.alloc(std::max(n_samples, 1))) return false;
    if ((size_t) n_mel * n_len > mel.n && !mel.alloc((size_t) n_mel * n_len)) return false;
    WB_CUDA_OK(cudaEventRecord(ev0, st));
    const float * src = pcm.p;
    if (samples_on_device && samples) src = samples;
    else if (n_samples > 0 && samples) { WB_CUDA_OK(cudaMemcpyAsync(pcm.p, samples, (size_t) n_samples * 4, cudaMemcpyHostToDevice, st)); count_h2d((uint64_t) n_samples * 4); }
    mel_spectrogram(src, n_samples, m->filters, n_mel, mel.p, n_len, gmax.p, st);
    WB_CUDA_OK(cudaEventRecord(ev1, st));
    WB_CUDA_OK(cudaStreamSynchronize(st));
    cudaEventElapsedTime(&last_mel_ms, ev0, ev1);
    return true;
}
bool FrontEnd::set_mel(const float * data, int n_len_, int n_mel_) {
    WB_CUDA_OK(cudaSetDevice(m->device));
    n_len = n_len_; n_len_org = n_len_; n_mel = n_mel_;
    if ((size_t) std::max(1, n_mel * n_len) > mel.n && !mel.alloc((size_t) std::max(1, n_mel * n_len))) return false;
    if (data) WB_CUDA_OK(cudaMemcpyAsync(mel.p, data, (size_t) n_mel * n_len * 4, cudaMemcpyHostToDevice, st));
    else      WB_CUDA_OK(cudaMemsetAsync(mel.p, 0, (size_t) n_mel * n_len * 4, st));   // whisper-bench passes NULL, 0 (bench.cpp:69)
    WB_CUDA_OK(cudaStreamSynchronize(st));
    return true;
}

// ---------------------------------------------------------------------------------------------------- encoder plan
static bool build_plan(Engine & E, int n_ctx, int n_win) {
    const Model & m = *E.m; const HParams & hp = m.hp;
    const int d = hp.n_audio_state, H = hp.n_audio_head, T = n_ctx, Tp = pad256(T), M = hp.n_mels, Lt = hp.n_text_layer, La = hp.n_audio_layer;
    const int NT = n_win * T;
    delete E.plan; E.plan = new EncPlan(); EncPlan & P = *E.plan;
    P.n_ctx = n_ctx; P.n_win = n_win;
    const int64_t win_rows = 2 * hp.n_audio_ctx + 2;            // allocation stride of mel_win / h1 (full-size windows)
    QMat f16A; f16A.type = WT_F16;

    { // conv1: [d x 2T] = sum_tap W1[tap] (d x M) * melT[t + tap] (whisper.cpp:2012-2015; ggml_conv_1d = im2col(F16) + mul_mat)
        GemmDesc & g = P.conv1; g.M = d; g.N = 2*T; g.K = M; g.taps = 3; g.BN = 256; g.nb0 = n_win; g.A = f16A; g.A.base = m.conv1_w;
        g.a_zsel[0] = 3; g.a_zsel[1] = 0; g.b_zsel[0] = 3; g.b_zsel[1] = 1;
        if (!make_tmap_f16(&g.tmA, m.conv1_w, M, d, 3, 1, M, (uint64_t) d * M, 0, 128)) return false;
        if (!make_tmap_f16(&g.tmB, E.mel_win.p, M, 2*T, 3, n_win, M, M, win_rows * M, 256)) return false;
        g.ep.bias_m = m.conv1_b; g.ep.act = 1; g.ep.out = E.h1.p; g.ep.out_f16 = 1; g.ep.ldo = d; g.ep.n_row_off = 1; g.ep.out_b0 = win_rows * d;
    }
    { // conv2 (stride 2) + GELU + positional embedding (whisper.cpp:2017-2020, 2094-2095)
        GemmDesc & g = P.conv2; g.M = d; g.N = T; g.K = d; g.taps = 3; g.BN = 256; g.nb0 = n_win; g.A = f16A; g.A.base = m.conv2_w;
        g.a_zsel[0] = 3; g.a_zsel[1] = 0; g.b_zsel[0] = 3; g.b_zsel[1] = 1;
        if (!make_tmap_f16(&g.tmA, m.conv2_w, d, d, 3, 1, d, (uint64_t) d * d, 0, 128)) return false;
        if (!make_tmap_f16(&g.tmB, E.h1.p, d, T, 3, n_win, 2*d, d, win_rows * d, 256)) return false;
        g.ep.bias_m = m.conv2_b; g.ep.act = 1; g.ep.res = m.e_pe; g.ep.ldr = d; g.ep.out = E.x.p; g.ep.ldo = d; g.ep.out_b0 = (int64_t) T * d;
        P.conv2_tap = g; P.conv2_tap.ep.res = nullptr; P.conv2_tap.ep.out = E.conv32.p;
    }
    // activation-side tile: 256 tokens per CTA, or 128 when a d x NT GEMM would otherwise leave SMs idle (one window: 10 x 6 = 60 CTAs)
    const int bn = (((NT + 255) / 256) * ((d + 127) / 128) < E.n_sm) ? 128 : 256;
    CUtensorMap tm_xn, tm_xn_win, tm_attn, tm_hfc, tm_q, tm_k, tm_p, tm_vt, tm_enc;
    if (!make_tmap_f16(&tm_xn, E.xn.p, d, NT, 1, 1, d, 0, 0, bn)) return false;
    if (!make_tmap_f16(&tm_xn_win, E.xn.p, d, T, n_win, 1, d, (uint64_t) T * d, 0, bn)) return false;
    if (!make_tmap_f16(&tm_attn, E.attn.p, d, NT, 1, 1, d, 0, 0, bn)) return false;
    if (!make_tmap_f16(&tm_hfc, E.hfc.p, 4*d, NT, 1, 1, 4*d, 0, 0, bn)) return false;
    if (!make_tmap_f16(&tm_q, E.qk.p,     64, T, H, n_win, 2*d, 64, (uint64_t) T * 2 * d, 256)) return false;
    if (!make_tmap_f16(&tm_k, E.qk.p + d, 64, T, H, n_win, 2*d, 64, (uint64_t) T * 2 * d, 128)) return false;
    if (!E.fused_attn && !make_tmap_f16(&tm_p, E.P.p, Tp, T, H, n_win, Tp, (uint64_t) T * Tp, (uint64_t) H * T * Tp, 128)) return false;
    if (!make_tmap_f16(&tm_vt, E.vt.p, Tp, 64, H, n_win, Tp, (uint64_t) 64 * Tp, (uint64_t) d * Tp, 64)) return false;
    if (!make_tmap_f16(&tm_enc, E.enc16.p, d, T, n_win, 1, d, (uint64_t) T * d, 0, bn)) return false;

    P.layers.resize(La);
    for (int l = 0; l < La; ++l) {
        const EncLayerW & L = m.enc[l]; EncLayerPlan & lp = P.layers[l];
        { GemmDesc & g = lp.qk; g.M = 2*d; g.N = NT; g.K = d; g.BN = bn; g.A = L.qk; g.tmB = tm_xn;        // whisper.cpp:2119-2130
          if (L.qk.type == WT_F16 && !make_tmap_f16(&g.tmA, L.qk.base, d, 2*d, 1, 1, d, 0, 0, 128)) return false;
          g.ep.bias_m = L.qk_bias; g.ep.out = E.qk.p; g.ep.out_f16 = 1; g.ep.ldo = 2*d; }
        { GemmDesc & g = lp.v; g.M = d; g.N = T; g.K = d; g.BN = bn; g.nb0 = n_win; g.A = L.v; g.tmB = tm_xn_win; g.b_zsel[0] = 1; g.b_zsel[1] = 0;  // 2134-2138
          if (L.v.type == WT_F16 && !make_tmap_f16(&g.tmA, L.v.base, d, d, 1, 1, d, 0, 0, 128)) return false;
          g.ep.bias_m = L.v_bias; g.ep.out = E.vt.p; g.ep.out_f16 = 1; g.ep.out_mmajor = 1; g.ep.ldo = Tp; g.ep.out_b0 = (int64_t) d * Tp; }
        { GemmDesc & g = lp.s; g.M = Tp; g.N = T; g.K = 64; g.BN = 256; g.nb0 = H; g.nb1 = n_win; g.A = f16A; g.A.base = E.qk.p + d;     // K.Q^T, 1536 padded keys
          g.tmA = tm_k; g.tmB = tm_q; g.a_zsel[0] = 1; g.a_zsel[1] = 2;
          g.ep.alpha = 1.0f / sqrtf(64.0f); g.ep.out = E.S.p; g.ep.ldo = Tp; g.ep.out_b0 = (int64_t) T * Tp; g.ep.out_b1 = (int64_t) H * T * Tp; }
        { GemmDesc & g = lp.pv; g.M = T; g.N = 64; g.K = Tp; g.BN = 64; g.nb0 = H; g.nb1 = n_win; g.A = f16A; g.A.base = E.P.p;
          g.tmA = tm_p; g.tmB = tm_vt; g.a_zsel[0] = 1; g.a_zsel[1] = 2;
          g.ep.out = E.attn.p; g.ep.out_f16 = 1; g.ep.out_mmajor = 1; g.ep.ldo = d; g.ep.out_b0 = 64; g.ep.out_b1 = (int64_t) T * d; }
        { GemmDesc & g = lp.o; g.M = d; g.N = NT; g.K = d; g.BN = bn; g.A = L.o; g.tmB = tm_attn;           // 2200-2208
          if (L.o.type == WT_F16 && !make_tmap_f16(&g.tmA, L.o.base, d, d, 1, 1, d, 0, 0, 128)) return false;
          g.ep.bias_m = L.o_bias; g.ep.res = E.x.p; g.ep.ldr = d; g.ep.out = E.x.p; g.ep.ldo = d; }
        { GemmDesc & g = lp.fc1; g.M = 4*d; g.N = NT; g.K = d; g.BN = bn; g.A = L.fc1; g.tmB = tm_xn;       // 2225-2232
          if (L.fc1.type == WT_F16 && !make_tmap_f16(&g.tmA, L.fc1.base, d, 4*d, 1, 1, d, 0, 0, 128)) return false;
          g.ep.bias_m = L.fc1_bias; g.ep.act = 1; g.ep.out = E.hfc.p; g.ep.out_f16 = 1; g.ep.ldo = 4*d; }
        { GemmDesc & g = lp.fc2; g.M = d; g.N = NT; g.K = 4*d; g.BN = bn; g.A = L.fc2; g.tmB = tm_hfc;      // 2235-2242
          if (L.fc2.type == WT_F16 && !make_tmap_f16(&g.tmA, L.fc2.base, 4*d, d, 1, 1, 4*d, 0, 0, 128)) return false;
          g.ep.bias_m = L.fc2_bias; g.ep.res = E.x.p; g.ep.ldr = d; g.ep.out = E.x.p; g.ep.ldo = d; }
    }
    { // cross K/V of every text layer in one launch (whisper.cpp:2306-2347)
        GemmDesc & g = P.cross; g.M = d; g.N = T; g.K = d; g.BN = bn; g.nb0 = 2 * Lt; g.nb1 = n_win; g.A = m.cross_kv; g.a_rows_per_b0 = d;
        g.tmB = tm_enc; g.b_zsel[0] = 2; g.b_zsel[1] = 0;
        if (m.cross_kv.type == WT_F16) {
            if (!make_tmap_f16(&g.tmA, m.cross_kv.base, d, (uint64_t) 2 * Lt * d, 1, 1, d, 0, 0, 128)) return false;
        }
        g.ep.bias_m = m.cross_bias; g.ep.scale_m = m.cross_scale; g.ep.out = E.kv_cross.p; g.ep.out_f16 = 1; g.ep.ldo = d;
        g.ep.out_b0 = (int64_t) E.Tp_max * d; g.ep.out_b1 = (int64_t) 2 * Lt * E.Tp_max * d;
        if (E.use_mk && mk_cross_head_major()) g.ep.hm_rows = E.Tp_max;                  // the persistent decode kernel streams K/V head by head (wb_decode_mk.cu)
    }
    if (E.gemm_v2) {
        // second-generation kernel: quantised weights are expanded to f16 once per launch into E.wf16 (every launch of the stream reuses the
        // same scratch: the previous GEMM has finished reading it when the next expansion starts) and reach the tensor cores through TMA
        auto to_v2 = [&](GemmDesc & g, int64_t rows) -> bool {
            g.v2 = 1;
            if (g.A.type == WT_F16) return true;
            if (g.A.f16) {                                        // expanded once at load (wb_model.cu)
                g.a16 = const_cast<__half *>(g.A.f16); g.a16_keep = 1;
                return make_tmap_f16(&g.tmA, g.A.f16, g.K, rows, 1, 1, g.K, 0, 0, 128);
            }
            if (!E.wf16.p) { g.v2 = 0; return true; }
            g.a16 = E.wf16.p;
            return make_tmap_f16(&g.tmA, E.wf16.p, g.K, rows, 1, 1, g.K, 0, 0, 128);
        };
        if (!to_v2(P.conv1, 0) || !to_v2(P.conv2, 0) || !to_v2(P.conv2_tap, 0)) return false;
        for (auto & lp : P.layers) {
            if (!to_v2(lp.qk, 2*d) || !to_v2(lp.v, d) || !to_v2(lp.o, d) || !to_v2(lp.fc1, 4*d) || !to_v2(lp.fc2, d)) return false;
        }
        if (!to_v2(P.cross, (int64_t) 2 * Lt * d)) return false;
    }
    return true;
}

#define WB_GEMM(desc) do { cudaError_t e_ = gemm_launch(desc, st); if (e_ != cudaSuccess) { set_error("%s:%d gemm_launch: %s", __FILE__, __LINE__, cudaGetErrorString(e_)); return false; } } while (0)

bool Engine::encode(const EncSrc * srcs, int n_win, int n_ctx) {
    NvtxRange nvtx("wb200.encode");
    const HParams & hp = m->hp;
    WB_CUDA_OK(cudaSetDevice(m->device));
    if (n_win < 1 || n_win > cap_win) { set_error("encode: n_win=%d exceeds the state's capacity %d", n_win, cap_win); return false; }
    if (n_ctx <= 0 || n_ctx > hp.n_audio_ctx) { set_error("encode: bad n_ctx %d", n_ctx); return false; }
    if (!plan || plan->n_ctx != n_ctx || plan->n_win != n_win) {
        if (plan && plan->n_ctx != n_ctx) {   // different padding: make sure the encoder's padded key rows are zero again
            WB_CUDA_OK(cudaMemsetAsync(vt.p, 0, vt.bytes(), st));
            WB_CUDA_OK(cudaMemsetAsync(h1.p, 0, h1.bytes(), st));
        }
        if (!build_plan(*this, n_ctx, n_win)) return false;
    }
    const int d = hp.n_audio_state, H = hp.n_audio_head, T = n_ctx, Tp = pad256(T), M = hp.n_mels;
    const int NT = n_win * T;
    const int64_t win_rows = 2 * hp.n_audio_ctx + 2;
    EncPlan & PL = *plan;

    WB_CUDA_OK(cudaEventRecord(ev[1], st));
    bool identity_slots = true;
    for (int w = 0; w < n_win; ++w) {
        if (srcs[w].n_mel != M) { set_error("encode: mel has %d bands, model expects %d", srcs[w].n_mel, M); return false; }
        if (srcs[w].slot < 0 || srcs[w].slot >= cap_win) { set_error("encode: bad slot %d", srcs[w].slot); return false; }
        identity_slots &= (srcs[w].slot == w);
        mel_window_f16(srcs[w].mel, srcs[w].n_len, M, srcs[w].seek, 2*T, mel_win.p + (size_t) w * win_rows * M, st);
    }
    WB_GEMM(PL.conv1);
    if (debug_taps) WB_GEMM(PL.conv2_tap);
    WB_GEMM(PL.conv2);
    WB_CUDA_OK(cudaEventRecord(ev[2], st));
    for (size_t l = 0; l < PL.layers.size(); ++l) {
        const EncLayerW & L = m->enc[l]; EncLayerPlan & lp = PL.layers[l];
        layernorm(x.p, L.ln0.w, L.ln0.b, hp.eps, NT, d, xn.p, nullptr, st);
        WB_GEMM(lp.qk);
        WB_GEMM(lp.v);
        if (fused_attn) {
            if (!fattn_encoder(qk.p, 2*d, d, vt.p, T, Tp, H, n_win, 1.0f / sqrtf(64.0f), attn.p, d, st)) { set_error("fattn_encoder launch failed"); return false; }
        } else {
            WB_GEMM(lp.s);
            softmax_rows_f16(S.p, P.p, (int64_t) n_win * H * T, Tp, st);
            WB_GEMM(lp.pv);
        }
        WB_GEMM(lp.o);
        layernorm(x.p, L.ln1.w, L.ln1.b, hp.eps, NT, d, xn.p, nullptr, st);
        WB_GEMM(lp.fc1);
        WB_GEMM(lp.fc2);
    }
    layernorm(x.p, m->e_ln.w, m->e_ln.b, hp.eps, NT, d, enc16.p, debug_taps ? enc32.p : nullptr, st);
    WB_CUDA_OK(cudaEventRecord(ev[3], st));
    if (T < hp.n_audio_ctx) {
        // The cross GEMM writes rows [0, T) of each head (head-major) or block (token-major); rows [T, Tp_max) of the slots written here
        // may hold an earlier, longer encode and must read as zero keys: both decoders attend to the padding up to pad256(T).  Rows from
        // n_audio_ctx on are never written, so a full-context encode has nothing to clear.  Other slots keep their cross K/V untouched.
        const int dt = hp.n_text_state, Lt = hp.n_text_layer;
        const bool hm = use_mk && mk_cross_head_major();
        const size_t row = hm ? 64 : (size_t) dt, blocks = hm ? (size_t) 2 * Lt * (dt / 64) : (size_t) 2 * Lt;
        for (int w = 0; w < n_win; ++w) {
            __half * base = kv_cross.p + (size_t) srcs[w].slot * 2 * Lt * Tp_max * dt;
            WB_CUDA_OK(cudaMemset2DAsync(base + (size_t) T * row, (size_t) Tp_max * row * sizeof(__half), 0, (size_t) (Tp_max - T) * row * sizeof(__half), blocks, st));
        }
    }
    if (identity_slots) {
        WB_GEMM(PL.cross);
    } else {                          // windows land in arbitrary cross-KV slots: one launch per window
        for (int w = 0; w < n_win; ++w) {
            GemmDesc g = PL.cross;
            g.nb1 = 1; g.b1_in_off = w; g.a16_keep = (w > 0) || g.A.f16 != nullptr;
            g.ep.out = kv_cross.p + (size_t) srcs[w].slot * 2 * hp.n_text_layer * Tp_max * d;
            WB_GEMM(g);
        }
    }
    WB_CUDA_OK(cudaEventRecord(ev[4], st));
    WB_CUDA_OK(cudaStreamSynchronize(st));
    cudaEventElapsedTime(&last_ms[1], ev[1], ev[2]);
    cudaEventElapsedTime(&last_ms[2], ev[2], ev[3]);
    cudaEventElapsedTime(&last_ms[3], ev[3], ev[4]);
    counter_add(4, 1); counter_add(5, n_win); counter_add(6, last_ms[1] + last_ms[2] + last_ms[3]);
    enc_n_ctx = n_ctx; enc_n_win = n_win;
    for (int w = 0; w < n_win; ++w) slot_ctx[(size_t) srcs[w].slot] = n_ctx;
    return true;
}

// ---------------------------------------------------------------------------------------------------- decoder
bool Engine::set_samp_mask(uint64_t key, const std::vector<uint32_t> & bits) {
    if (key == samp_mask_key) return true;
    WB_CUDA_OK(cudaSetDevice(m->device));
    if (bits.size() != samp_mask.n) { set_error("set_samp_mask: size mismatch"); return false; }
    WB_CUDA_OK(cudaStreamSynchronize(st));
    WB_CUDA_OK(cudaMemcpy(samp_mask.p, bits.data(), bits.size() * 4, cudaMemcpyHostToDevice));
    samp_mask_key = key;
    return true;
}

bool Engine::decode_pass_enqueue(int n, bool any_logits, int n_keys, int n_audio_ctx, const SampCfg * samp, bool tok_indirect) {
    const HParams & hp = m->hp;
    const int d = hp.n_text_state, H = hp.n_text_head, Lt = hp.n_text_layer, V = hp.n_vocab;
    const int Tp = Tp_max;                                         // kv_cross layout stride
    const float kq_scale = powf(64.0f, -0.25f);                    // whisper.cpp:2514
    const int R = max_rows;
    const size_t nint = (size_t) 8 * R + (size_t) n * ld_idx;          // packed: tok | pos | cell | slot | n_kv | rowinfo[2] | capture index | idx rows
    WB_CUDA_OK(cudaMemcpyAsync(dints.p, hints, nint * sizeof(int), cudaMemcpyHostToDevice, st));
    const int * d_tok = dints.p, * d_pos = dints.p + R, * d_cell = dints.p + 2 * R, * d_slot = dints.p + 3 * R, * d_nkv = dints.p + 4 * R, * d_row = dints.p + 5 * R;
    const int * d_cap = dints.p + 7 * R, * d_idx = dints.p + 8 * R;

    auto chain_gemv = [&](const GemvArgs & a) { if (gemv_v2) gemv2(a, act_scratch.p, st); else gemv(a, st); };
    if (tok_indirect) tok_resolve(dints.p, dsamp.p, n, st);
    dec_embed(m->d_te, m->d_pe, d_tok, d_pos, n, d, dx.p, st);
    if (use_mk) {
        MkArgs a;
        a.layers = mk_layers.p; a.n_layer = Lt; a.d = d; a.n_head = H; a.n_tok = n; a.n_keys = n_keys; a.ld_idx = ld_idx; a.n_vocab = V;
        a.n_audio_ctx = n_audio_ctx;                                    // n_keys is this rounded up to 256
        a.kv_rows = Tp;                                                 // the cross GEMM lays each head out over Tp_max rows
        a.want_logits = any_logits ? 1 : 0;
        a.tok = d_tok; a.pos = d_pos; a.cell = d_cell; a.slot = d_slot; a.nkv = d_nkv; a.idx = d_idx;
        a.slot_stride = (int64_t) 2 * Lt * Tp * d; a.kq_scale = kq_scale; a.eps = hp.eps;
        a.te = m->d_te; a.pe = m->d_pe; a.lnf_w = m->d_ln.w; a.lnf_b = m->d_ln.b;
        a.x = dx.p; a.qkv = dqkv.p; a.q2 = dq2.p; a.logits = dlogits.p;
        a.actq = reinterpret_cast<uint8_t *>(dattn.p); a.h = dh.p; a.hq = dhq.p;
        a.xpart = xpart.p; a.xcnt = xcnt.p;
        if (pass_capture) { a.cap = dtw_q.p; a.cap_row = d_cap; a.cap_rows = dtw_cap_rows; }
        a.bar = mk_bar.p; a.bar_base = mk_bar_total; a.err = reinterpret_cast<int *>(mk_bar.p + 8); a.prefetch = mk_prefetch; a.trace = mk_trace.p;
        // A pass of 32 rows or more is cut into partitions unless a row attends to a self-KV cell that a row of ANOTHER 16-row group appends
        // in this pass (several tokens of one sequence: prompt and DTW passes): those stay on one barrier.
        if (n >= 32 && mk_parts > 1) {
            if (cell_group.size() < (size_t) n_cells) cell_group.assign(n_cells, 0);
            ++cell_stamp;
            if ((cell_stamp & 0xffffff) == 0) { std::fill(cell_group.begin(), cell_group.end(), 0u); cell_stamp = 1; }
            const int * h_cell = hints + 2 * R, * h_nkv = hints + 4 * R, * h_idx = hints + 8 * R;
            for (int t = 0; t < n; ++t) cell_group[h_cell[t]] = (cell_stamp << 8) | (uint32_t) (t >> 4);
            bool shared = false;
            for (int t = 0; t < n && !shared; ++t) {
                const int * row = h_idx + (size_t) t * ld_idx;
                for (int k = 0; k < h_nkv[t]; ++k) {
                    const uint32_t cgv = cell_group[row[k]];
                    if ((cgv >> 8) == cell_stamp && (int) (cgv & 0xff) != (t >> 4)) { shared = true; break; }
                }
            }
            if (!shared) a.n_part = std::min(mk_parts, (n + 15) / 16);
        }
        a.turn_slots = mk_turns;
        std::copy(mk_bar_part, mk_bar_part + MK_MAX_PARTS, a.part_base);
        // algorithmic bytes of one pass: every decoder weight once, the cross K/V of each row, the self K/V each row attends to
        double wbytes = 0.0, flops = 0.0;
        for (int l = 0; l < Lt; ++l) {
            const DecLayerW & L = m->dec[l];
            for (const QMat * W : { &L.qkv, &L.o, &L.cq, &L.co, &L.fc1, &L.fc2 }) { wbytes += (double) W->N * W->K * wt_bpw(W->type); flops += 2.0 * W->N * W->K * n; }
        }
        if (any_logits) { wbytes += (double) m->d_te.N * m->d_te.K * wt_bpw(m->d_te.type); flops += 2.0 * m->d_te.N * m->d_te.K * n; }
        double kvbytes = 0.0;
        for (int j = 0; j < n; ++j) kvbytes += (double) Lt * 2.0 * d * 2.0 * ((double) n_keys + hints[4 * R + j]);
        flops += kvbytes;                                           // 2 flops per KV element (f16 = 2 bytes): same number
        ProfScope prof(PC_GEMV, st, wbytes + kvbytes, flops);
        if (!mk_launch(a, m->wtype == WT_F32 ? WT_F16 : m->wtype, n_sm, st)) return false;
        for (int p = 0; p < a.n_part; ++p)
            mk_bar_part[p] += (unsigned long long) mk_partition(p, a.n_part, n_sm, n).nc * mk_layer_barriers(m->wtype == WT_F32 ? WT_F16 : m->wtype) * Lt;
        if (any_logits) mk_bar_total += (unsigned long long) n_sm;
    } else
    for (int l = 0; l < Lt; ++l) {
        const DecLayerW & L = m->dec[l];
        __half * kc = kv_k.p + (size_t) l * n_cells * d;
        __half * vc = kv_v.p + (size_t) l * n_cells * d;
        { GemvArgs a; a.W = L.qkv; a.x = dx.p; a.n_tok = n; a.ln_w = L.ln0.w; a.ln_b = L.ln0.b; a.eps = hp.eps;      // whisper.cpp:2536-2599
          a.bias = L.qkv_bias; a.scale = L.qkv_scale; a.out = dqkv.p; a.k_cache = kc; a.v_cache = vc; a.cells = d_cell; a.kv_d = d;
          chain_gemv(a); }
        attn_self_decode(dqkv.p, 3*d, kc, vc, d_idx, ld_idx, d_nkv, n, H, d, dattn.p, d, st);                            // 2603-2625
        { GemvArgs a; a.W = L.o; a.x = dattn.p; a.n_tok = n; a.bias = L.o_bias; a.res = dx.p; a.out = dx.p; chain_gemv(a); }    // 2647-2659
        { GemvArgs a; a.W = L.cq; a.x = dx.p; a.n_tok = n; a.ln_w = L.lnc.w; a.ln_b = L.lnc.b; a.eps = hp.eps;        // 2661-2681
          a.bias = L.cq_bias; a.out = dq2.p; chain_gemv(a); }
        if (pass_capture && dtw_layer_mask[l] != 0u &&               // DTW rows: keep the alignment-head queries of this layer
            !dtw_capture_launch(dq2.p, d, d_cap, n, dtw_layer_mask[l], dtw_layer_head0[l], dtw_q.p, dtw_cap_rows, st)) return false;
        attn_cross_decode(dq2.p, d, kv_cross.p + (size_t) l * Tp * d, kv_cross.p + (size_t) (Lt + l) * Tp * d, d_slot,
                          (int64_t) 2 * Lt * Tp * d, n_keys, n, H, d, kq_scale, xpart.p, xcnt.p, dattn.p, d, st);       // 2688-2705
        { GemvArgs a; a.W = L.co; a.x = dattn.p; a.n_tok = n; a.bias = L.co_bias; a.res = dx.p; a.out = dx.p; chain_gemv(a); }  // 2754-2766
        { GemvArgs a; a.W = L.fc1; a.x = dx.p; a.n_tok = n; a.ln_w = L.lnm.w; a.ln_b = L.lnm.b; a.eps = hp.eps;       // 2770-2794
          a.bias = L.fc1_bias; a.act = 1; a.out = dh.p; chain_gemv(a); }
        { GemvArgs a; a.W = L.fc2; a.x = dh.p; a.n_tok = n; a.bias = L.fc2_bias; a.res = dx.p; a.out = dx.p; chain_gemv(a); }   // 2797-2806
    }
    if (any_logits) {
        GemvArgs a; a.W = m->d_te; a.x = dx.p; a.n_tok = n; a.ln_w = m->d_ln.w; a.ln_b = m->d_ln.b; a.eps = hp.eps; a.out = dlogits.p;   // 2811-2827
        if (!use_mk) chain_gemv(a);      // the persistent kernel already wrote dlogits
        if (samp) {
            SampCfg c = *samp; c.mask = samp_mask.p;
            if (draw_stride > 1) WB_CUDA_OK(cudaMemcpyAsync(ddraws.p, hdraws, (size_t) n * draw_stride * sizeof(double), cudaMemcpyHostToDevice, st));
            greedy_sample(dlogits.p, V, n, d_row, c, dsamp_of(cur_slot), st, draw_stride > 1 ? ddraws.p : nullptr, draw_stride);
            WB_CUDA_OK(cudaMemcpyAsync(hsamp, dsamp_of(cur_slot), (size_t) n * draw_stride * sizeof(SampOut), cudaMemcpyDeviceToHost, st));
        } else {
            WB_CUDA_OK(cudaMemcpyAsync(hlogits, dlogits.p, (size_t) n * V * 4, cudaMemcpyDeviceToHost, st));
        }
    }
    return true;
}

bool Engine::pass_enqueue(const DecToken * rows, int n, const int * cells, const int * kv_idx, int ld, const int * n_kv, const SampCfg * samp,
                          const int * rowinfo, const double * draws, int stride, const int * cap_idx, const int * tok_src, int * slot_out) {
    const HParams & hp = m->hp;
    WB_CUDA_OK(cudaSetDevice(m->device));
    const int V = hp.n_vocab, R = max_rows;
    if (n < 1 || n > R) { set_error("decode: %d rows in one pass (1..%d)", n, R); return false; }
    int slot = 0;
    while (slot < PASS_SLOTS && pslot[slot].busy) ++slot;
    if (slot == PASS_SLOTS) { set_error("decode: every pass slot is in flight"); return false; }
    PassSlot & ps = pslot[slot];
    cur_slot = slot; hints = ps.hints; hsamp = ps.hsamp;
    int * h_tok = hints, * h_pos = hints + R, * h_cell = hints + 2 * R, * h_slot = hints + 3 * R, * h_nkv = hints + 4 * R, * h_row = hints + 5 * R;
    int * h_cap = hints + 7 * R, * h_idx = hints + 8 * R;
    bool any_logits = false, indirect = false;
    pass_capture = false;
    for (int j = 0; j < n; ++j) {
        const DecToken & t = rows[j];
        const int src = tok_src ? tok_src[j] : -1;
        if (src >= PASS_SLOTS * R * SAMP_MAX_DRAWS || (src < 0 && (t.token < 0 || t.token >= V)) || t.pos < 0 || t.pos >= hp.n_text_ctx || t.slot < 0 || t.slot >= cap_win) {
            set_error("decode: bad token/pos/slot (%d, %d, %d)", src >= 0 ? src : t.token, t.pos, t.slot); return false;
        }
        if (n_kv[j] > ld_idx || n_kv[j] > ld) { set_error("decode: %d attended cells exceed the index row (%d)", n_kv[j], ld_idx); return false; }
        h_tok[j] = src >= 0 ? -1 - src : t.token; h_pos[j] = t.pos; h_cell[j] = cells[j]; h_slot[j] = t.slot; h_nkv[j] = n_kv[j];
        h_row[2*j] = (samp && rowinfo) ? rowinfo[2*j] : 0; h_row[2*j + 1] = (samp && rowinfo) ? rowinfo[2*j + 1] : 0;
        memcpy(h_idx + (size_t) j * ld_idx, kv_idx + (size_t) j * ld, (size_t) n_kv[j] * sizeof(int));
        h_cap[j] = cap_idx ? cap_idx[j] : -1;
        if (h_cap[j] >= dtw_cap_rows) { set_error("decode: capture index %d exceeds the capture buffer (%d rows)", h_cap[j], dtw_cap_rows); return false; }
        pass_capture |= h_cap[j] >= 0;
        any_logits |= t.want_logits;
        indirect |= src >= 0;
    }
    const int n_ctx = slot_n_ctx(rows[0].slot), n_keys = pad256(n_ctx);   // encoder positions of the pass's cross K/V
    for (int j = 1; j < n; ++j)
        if (slot_n_ctx(rows[j].slot) != n_ctx) {
            set_error("decode: one pass over slots encoded at %d and %d positions", n_ctx, slot_n_ctx(rows[j].slot)); return false;
        }
    draw_stride = (samp && draws && stride > 1) ? std::min(stride, (int) SAMP_MAX_DRAWS) : 1;
    if (draw_stride > 1) {
        for (int j = 0; j < n; ++j) memcpy(hdraws + (size_t) j * draw_stride, draws + (size_t) j * stride, (size_t) draw_stride * sizeof(double));
        for (int j = 0; j < n; ++j) if (((h_row[2*j] >> 8) & 0x7f) > draw_stride) { set_error("decode: a row asks for more draws than the pass carries"); return false; }
        count_h2d((size_t) n * draw_stride * sizeof(double));
    } else {
        for (int j = 0; j < n; ++j) h_row[2*j] &= 0xff;           // no uniforms supplied: greedy picks only
    }
    if (indirect && !(use_mk && samp && any_logits)) { set_error("decode: token indirection needs the persistent kernel and the on-device sampler"); return false; }
    count_h2d(((size_t) 8 * R + (size_t) n * ld_idx) * sizeof(int));
    if (any_logits) count_d2h(samp ? (uint64_t) n * draw_stride * sizeof(SampOut) : (uint64_t) n * V * 4);

    // One pass = 8 kernels per text layer.  After the second use of a shape the chain is replayed as a CUDA graph
    // (all per-step values live in `dints`, so kernel arguments never change between steps).
    uint64_t key = (uint64_t) (n | (any_logits ? 128 : 0) | (samp ? 256 : 0)) | ((uint64_t) n_keys << 10) | ((uint64_t) draw_stride << 24);
    if (samp) key |= (uint64_t) ((uint32_t) (samp->token_eot * 31 + samp->token_beg * 17 + samp->token_nosp * 13 + samp->space_id * 7 + samp->max_initial_tid * 3 + samp->no_timestamps * 2 + samp->suppress_blank)) << 32;
    // a graph holds the pinned buffers of the slot it was captured in: only slot 0 replays them (the chain never has two passes in flight)
    StepGraph * sg = (use_graphs && !use_mk && !prof_enabled() && !pass_capture && slot == 0) ? &graphs[key] : nullptr;
    WB_CUDA_OK(cudaEventRecord(ps.ev0, st));
    if (sg && sg->exec) {
        WB_CUDA_OK(cudaGraphLaunch(sg->exec, st));
        count_launch(sg->launches);
        counter_add(7, 1);
    } else if (sg && sg->seen >= 1) {
        const uint64_t l0 = launch_count();
        cudaGraph_t g = nullptr;
        WB_CUDA_OK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        const bool ok = decode_pass_enqueue(n, any_logits, n_keys, n_ctx, samp);
        const cudaError_t ce = cudaStreamEndCapture(st, &g);
        if (!ok || ce != cudaSuccess) { if (g) cudaGraphDestroy(g); set_error("decode: graph capture failed: %s", cudaGetErrorString(ce)); return false; }
        sg->launches = launch_count() - l0;
        const cudaError_t ie = cudaGraphInstantiate(&sg->exec, g, 0);
        cudaGraphDestroy(g);
        if (ie != cudaSuccess) { sg->exec = nullptr; set_error("decode: cudaGraphInstantiate: %s", cudaGetErrorString(ie)); return false; }
        WB_CUDA_OK(cudaGraphLaunch(sg->exec, st));
    } else {
        if (sg) sg->seen++;
        if (!decode_pass_enqueue(n, any_logits, n_keys, n_ctx, samp, indirect)) return false;
    }
    WB_CUDA_OK(cudaEventRecord(ps.ev1, st));
    ps.busy = true; ps.n = n; ps.draw_stride = draw_stride; ps.any_logits = any_logits;
    *slot_out = slot;
    return true;
}

bool Engine::pass_wait(int slot) {
    PassSlot & ps = pslot[slot];
    if (!ps.busy) return true;
    WB_CUDA_OK(cudaSetDevice(m->device));
    ps.busy = false;
    WB_CUDA_OK(cudaEventSynchronize(ps.ev1));
    { float ms = 0.0f; cudaEventElapsedTime(&ms, ps.ev0, ps.ev1); counter_add(0, 1); counter_add(1, ps.n); counter_add(2, ms); }
    if (use_mk && mk_trace.p && ps.any_logits) mk_trace_collect(m->hp.n_text_layer, true);
    return true;
}

bool Engine::decode(const DecToken * rows, int n_rows, const int * cells, const int * kv_idx, int ld, const int * n_kv, float * const * logits_out,
                    const SampCfg * samp, const int * rowinfo, SampOut * samp_out, const double * draws, int stride, const int * cap_idx) {
    NvtxRange nvtx("wb200.decode");
    const int V = m->hp.n_vocab;
    const int64_t t_host0 = std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
    for (int r0 = 0; r0 < n_rows; r0 += max_rows) {
        const int n = std::min(max_rows, n_rows - r0);
        int slot = 0;
        if (!pass_enqueue(rows + r0, n, cells + r0, kv_idx + (size_t) r0 * ld, ld, n_kv + r0, samp, rowinfo ? rowinfo + 2 * r0 : nullptr,
                          draws ? draws + (size_t) r0 * stride : nullptr, stride, cap_idx ? cap_idx + r0 : nullptr, nullptr, &slot) ||
            !pass_wait(slot)) return false;
        const PassSlot & ps = pslot[slot];
        if (ps.any_logits && samp && samp_out) {
            for (int j = 0; j < n; ++j) if (rows[r0 + j].want_logits)
                for (int q = 0; q < ps.draw_stride; ++q) samp_out[(size_t) (r0 + j) * stride + q] = ps.hsamp[(size_t) j * ps.draw_stride + q];
        } else if (ps.any_logits && logits_out) {
            for (int j = 0; j < n; ++j) if (rows[r0 + j].want_logits && logits_out[r0 + j])
                memcpy(logits_out[r0 + j], hlogits + (size_t) j * V, (size_t) V * 4);
        }
    }
    counter_add(3, 1e-3 * (std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now().time_since_epoch()).count() - t_host0));
    return true;
}

} // namespace wb

namespace wb {
// ---------------------------------------------------------------------------------------------------- DTW capture
bool Engine::dtw_set_heads(const std::vector<std::pair<int, int>> & heads) {
    const HParams & hp = m->hp;
    const int Lt = hp.n_text_layer, H = hp.n_text_head;
    if (heads.empty()) return true;
    if (H > 32) { set_error("dtw: %d heads per layer, the capture takes at most 32", H); return false; }
    dtw_layer_mask.assign((size_t) Lt, 0u);
    for (const auto & lh : heads) {
        if (lh.first < 0 || lh.first >= Lt || lh.second < 0 || lh.second >= H) { set_error("dtw: alignment head (%d, %d) out of range", lh.first, lh.second); return false; }
        dtw_layer_mask[(size_t) lh.first] |= 1u << lh.second;
    }
    dtw_layer_head0.assign((size_t) Lt, 0);
    for (int l = 1; l < Lt; ++l) dtw_layer_head0[(size_t) l] = dtw_layer_head0[(size_t) l - 1] + __builtin_popcount(dtw_layer_mask[(size_t) l - 1]);
    dtw_n_heads = (int) heads.size();
    std::vector<int> tab((size_t) 3 * dtw_n_heads);                   // per alignment head: capture head | layer | head
    for (int e = 0; e < dtw_n_heads; ++e) {
        const int l = heads[(size_t) e].first, h = heads[(size_t) e].second;
        tab[(size_t) e] = dtw_layer_head0[(size_t) l] + __builtin_popcount(dtw_layer_mask[(size_t) l] & ((1u << h) - 1u));
        tab[(size_t) dtw_n_heads + e] = l; tab[(size_t) 2 * dtw_n_heads + e] = h;
    }
    WB_CUDA_OK(cudaSetDevice(m->device));
    if (!dtw_heads_dev.alloc(tab.size())) return false;
    WB_CUDA_OK(cudaMemcpy(dtw_heads_dev.p, tab.data(), tab.size() * sizeof(int), cudaMemcpyHostToDevice));
    return !use_mk || mk_build_table();
}

bool Engine::dtw_reserve(int n_rows) {
    if (n_rows <= dtw_cap_rows) return true;
    const int n_cap = dtw_layer_head0.empty() ? 0 : dtw_layer_head0.back() + __builtin_popcount(dtw_layer_mask.back());
    if (n_cap == 0) { set_error("dtw: the engine has no alignment heads"); return false; }
    WB_CUDA_OK(cudaSetDevice(m->device));
    WB_CUDA_OK(cudaStreamSynchronize(st));
    if (!dtw_q.alloc((size_t) n_cap * n_rows * 64)) return false;
    dtw_cap_rows = n_rows;
    return true;
}

bool Engine::dtw_weights(const std::vector<int> & req, const std::vector<int> & path, std::vector<std::vector<float> *> & out,
                         std::vector<std::vector<int32_t> *> & tok, std::vector<std::vector<int32_t> *> & time) {
    const HParams & hp = m->hp;
    const int n_req = (int) req.size() / 4, d = hp.n_text_state, Lt = hp.n_text_layer;
    WB_CUDA_OK(cudaSetDevice(m->device));
    std::vector<int64_t> off((size_t) n_req + 1, 0);
    int max_tokens = 0;
    for (int r = 0; r < n_req; ++r) {
        off[(size_t) r + 1] = off[(size_t) r] + (int64_t) dtw_n_heads * req[4 * r + 3] * req[4 * r + 2];
        max_tokens = std::max(max_tokens, req[4 * r + 2]);
    }
    if ((size_t) off.back() > dtw_out.n && !dtw_out.alloc((size_t) off.back())) return false;
    if (req.size() > dtw_req_dev.n && !dtw_req_dev.alloc(req.size())) return false;
    if ((size_t) n_req > dtw_req_out.n && !dtw_req_out.alloc((size_t) n_req)) return false;
    WB_CUDA_OK(cudaMemcpyAsync(dtw_req_dev.p, req.data(), req.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    WB_CUDA_OK(cudaMemcpyAsync(dtw_req_out.p, off.data(), (size_t) n_req * sizeof(int64_t), cudaMemcpyHostToDevice, st));
    DtwQkArgs a;
    a.q = dtw_q.p; a.cap_rows = dtw_cap_rows;
    a.k_cross = kv_cross.p; a.slot_stride = (int64_t) 2 * Lt * Tp_max * d; a.layer_stride = (int64_t) Tp_max * d;   // K part of each slot: [Lt][Tp][d]
    a.k_head_major = (use_mk && mk_cross_head_major()) ? 1 : 0; a.Tp = Tp_max;
    a.head_cap = dtw_heads_dev.p; a.head_layer = dtw_heads_dev.p + dtw_n_heads; a.head_index = dtw_heads_dev.p + 2 * dtw_n_heads;
    a.req = dtw_req_dev.p; a.req_out = dtw_req_out.p;
    a.n_heads = dtw_n_heads; a.n_req = n_req; a.max_tokens = max_tokens; a.d = d; a.scale = powf(64.0f, -0.25f); a.out = dtw_out.p;
    for (int r = 0; r < n_req; ++r)
        if (req[4 * r + 3] <= 0 || req[4 * r + 3] > std::min(Tp_max, 1536) ||   // 1536: the score row of k_dtw_qk in shared memory
             req[4 * r] < 0 || req[4 * r] + req[4 * r + 2] > dtw_cap_rows) { set_error("dtw: bad request %d", r); return false; }
    WB_CUDA_OK(cudaEventRecord(ev[5], st));
    if (!dtw_qk_launch(a, st)) return false;
    WB_CUDA_OK(cudaEventRecord(ev[6], st));
    std::vector<int> preq((size_t) DTW_REQ_INTS * n_req);
    for (int r = 0; r < n_req; ++r) {
        int * p = preq.data() + (size_t) DTW_REQ_INTS * r;
        p[0] = req[4 * r + 2]; p[1] = req[4 * r + 3]; p[2] = dtw_n_heads; p[3] = path[2 * r]; p[4] = path[2 * r + 1];
    }
    if (!dtw_paths.enqueue(dtw_out.p, preq, std::vector<int64_t>(off.begin(), off.end() - 1), st)) return false;
    WB_CUDA_OK(cudaEventRecord(ev[7], st));
    if (!dtw_paths.fetch(st)) return false;
    for (int r = 0; r < n_req; ++r) {
        std::vector<float> & o = *out[(size_t) r];
        o.resize((size_t) (off[(size_t) r + 1] - off[(size_t) r]));
        WB_CUDA_OK(cudaMemcpyAsync(o.data(), dtw_out.p + off[(size_t) r], o.size() * sizeof(float), cudaMemcpyDeviceToHost, st));
    }
    WB_CUDA_OK(cudaStreamSynchronize(st));
    count_d2h((uint64_t) off.back() * sizeof(float));
    for (int r = 0; r < n_req; ++r) dtw_paths.get(r, *tok[(size_t) r], *time[(size_t) r]);
    { float ms = 0.0f; cudaEventElapsedTime(&ms, ev[5], ev[6]); counter_add(8, ms); counter_add(9, n_req); }
    { float ms = 0.0f; cudaEventElapsedTime(&ms, ev[6], ev[7]); counter_add(11, ms); }
    return true;
}
} // namespace wb

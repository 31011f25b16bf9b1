// wb_model.cu -- legacy-ggml model file -> HBM (see wb_model.h for the layout decisions).
// Follows whisper_model_load (src/whisper.cpp:1485-1962) record by record; tensor names from src/whisper-arch.h:42-109.
#include <chrono>
#include "wb_dequant_host.h"
#include <cmath>
#include <cstring>
#include <functional>
#include "../../include/whisper_b200.h"
#include <cstdlib>
#include "wb_model.h"
#include "wb_gemm.cuh"
#include "wb_kernels.cuh"

namespace wb {

Model::~Model() {
    if (!allocs.empty()) cudaSetDevice(device);
    for (void * p : allocs) cudaFree(p);
}

// language codes in id order (src/whisper.cpp:278-381); used for the [_LANG_xx] names of synthesised vocab entries
extern const char * const g_lang_codes[100];

namespace {

struct Reader {
    whisper_model_loader * l;
    bool ok = true;
    template <typename T> bool rd(T & v) { return rdn(&v, sizeof(T)); }
    bool rdn(void * dst, size_t n) {
        if (n == 0) return true;
        size_t got = l->read(l->context, dst, n);
        if (got != n) ok = false;
        return got == n;
    }
};

void * dalloc(Model & m, size_t bytes, bool zero = true) {
    void * p = nullptr;
    if (bytes == 0) bytes = 16;
    if (cudaMalloc(&p, bytes) != cudaSuccess) { set_error("model: cudaMalloc(%zu) failed", bytes); return nullptr; }
    if (zero) cudaMemset(p, 0, bytes);
    m.allocs.push_back(p);
    m.bytes_weights += bytes;
    return p;
}

// allocate an [N][K] matrix of type t in its HBM layout
bool alloc_qmat(Model & m, int t, int N, int K, QMat & q, bool tile_major = false) {
    q.type = t; q.N = N; q.K = K;
    if (tile_major && wt_tm_rec_bytes(t) > 0 && K % 32 == 0 && K % wt_tm_rec_k(t) == 0) {
        const size_t bytes = wt_tm_bytes(t, N, K);
        q.base = dalloc(m, bytes);
        if (!q.base) return false;
        q.layout = 1;
        return cudaMemset(const_cast<void *>(q.base), 0, bytes) == cudaSuccess;
    }
    if (t == WT_F16) {
        q.base = dalloc(m, (size_t) N * K * 2);
        return q.base != nullptr;
    }
    if (wt_is_block32(t)) {
        if (K % 32) { set_error("model: K=%d not a multiple of 32 for block-quantised weights", K); return false; }
        const size_t nblk = (size_t) N * (K / 32);
        q.qs = (const uint8_t *) dalloc(m, nblk * wt_qs_bytes(t));
        q.d  = (const __half *)  dalloc(m, nblk * 2);
        if (wt_has_qh(t)) { q.qh = (const uint32_t *) dalloc(m, nblk * 4); if (!q.qh) return false; }
        if (wt_has_min(t)) { q.m = (const __half *) dalloc(m, nblk * 2); if (!q.m) return false; }
        return q.qs && q.d;
    }
    if (wt_is_kquant(t)) {
        if (K % 256) { set_error("model: K=%d not a multiple of 256 for K-quants", K); return false; }
        q.base = dalloc(m, (size_t) N * (K / 256) * wt_kq_block_bytes(t));
        return q.base != nullptr;
    }
    set_error("model: unsupported weight type %d (supported: F32->F16, F16, Q4_0, Q4_1, Q5_0, Q5_1, Q8_0, Q3_K, Q4_K, Q5_K)", t);
    return false;
}

struct Dest {
    enum Kind { VEC_F32, MAT, CONV } kind = VEC_F32;
    float * vec = nullptr; int64_t n = 0;           // VEC_F32: n floats
    QMat * mat = nullptr; int row_off = 0, rows = 0, cols = 0;   // MAT
    __half * conv = nullptr; int oc = 0, ic = 0;    // CONV
    bool seen = false;
};

__global__ void k_conv_reorder(const __half * __restrict__ src, __half * __restrict__ dst, int oc, int ic) {
    // src[oc][ic][3] -> dst[3][oc][ic]
    const int64_t n = (int64_t) oc * ic * 3;
    int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int k = (int) (i % 3); const int64_t r = i / 3; const int c = (int) (r % ic); const int o = (int) (r / ic);
    dst[((int64_t) k * oc + o) * ic + c] = src[i];
}
__global__ void k_fill(float * p, float v, int64_t n) {
    int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}

} // namespace

bool model_load(whisper_model_loader * loader, Model & m, Vocab & vocab, int device) {
    const auto t0 = std::chrono::steady_clock::now();
    m.device = device;
    if (device >= 0) WB_CUDA_OK(cudaSetDevice(device));          // device < 0: header + vocabulary only, nothing touches CUDA (host-side test hooks)
    Reader R{loader};

    uint32_t magic = 0;
    R.rd(magic);
    if (!R.ok || magic != 0x67676d6c) { set_error("invalid model data (bad magic)"); return false; }

    HParams & hp = m.hp;
    R.rd(hp.n_vocab); R.rd(hp.n_audio_ctx); R.rd(hp.n_audio_state); R.rd(hp.n_audio_head); R.rd(hp.n_audio_layer);
    R.rd(hp.n_text_ctx); R.rd(hp.n_text_state); R.rd(hp.n_text_head); R.rd(hp.n_text_layer); R.rd(hp.n_mels); R.rd(hp.ftype);
    if (!R.ok) { set_error("truncated model header"); return false; }
    if (hp.n_text_state != hp.n_audio_state) { set_error("n_text_state != n_audio_state is not supported"); return false; }
    if (hp.n_audio_state % hp.n_audio_head || hp.n_audio_state / hp.n_audio_head != 64 || hp.n_text_state / hp.n_text_head != 64) {
        set_error("head dimension must be 64 (n_state=%d n_head=%d)", hp.n_audio_state, hp.n_audio_head); return false;
    }
    m.mtype = hp.n_audio_layer == 4 ? 1 : hp.n_audio_layer == 6 ? 2 : hp.n_audio_layer == 12 ? 3 : hp.n_audio_layer == 24 ? 4 : hp.n_audio_layer == 32 ? 5 : 0;
    hp.ftype %= 1000; // strip GGML_QNT_VERSION (src/whisper.cpp:1549-1551)
    int host_dq = -1;
    switch (hp.ftype) {  // ggml_ftype_to_ggml_type (ggml/src/ggml.c:1426-1463)
        case 0: m.wtype = WT_F32; break;  case 1: m.wtype = WT_F16; break; case 2: m.wtype = WT_Q4_0; break;
        case 7: m.wtype = WT_Q8_0; break; case 8: m.wtype = WT_Q5_0; break; case 12: m.wtype = WT_Q4_K; break;
        case 13: m.wtype = WT_Q5_K; break; case 3: m.wtype = WT_Q4_1; break; case 9: m.wtype = WT_Q5_1; break;
        case 11: m.wtype = WT_Q3_K; break;
        // formats without device kernels: expanded on the host at load time, kept in HBM as F16 (wb_dequant_host.h)
        case 10: host_dq = HT_Q2_K; break; case 14: host_dq = HT_Q6_K; break; case 24: host_dq = HT_BF16; break;
        default: set_error("invalid model (ftype %d is not supported by this engine)", hp.ftype); return false;
    }
    if (wt_is_kquant(m.wtype) && getenv("WB200_KQUANT_AS_F16") && atoi(getenv("WB200_KQUANT_AS_F16")) != 0) {
        // opt-in: K-quants expanded to F16 (2 bytes per weight, F16 arithmetic); without it their blocks decode natively (Q8_K activations)
        host_dq = m.wtype;                                       // HostDqType ids are the ggml_type ids
    }
    if (host_dq >= 0) {
        m.wtype = WT_F16;
        logf(LOG_WARN, "%s: ftype %d (ggml type %d): matrices are expanded to F16 on the host at load time (%s)\n", __func__, hp.ftype, host_dq,
             wt_is_kquant(host_dq) ? "WB200_KQUANT_AS_F16" : "no device kernels for this block format");
    }
    const int file_wtype = host_dq >= 0 ? host_dq : m.wtype;
    const int wt = (m.wtype == WT_F32) ? WT_F16 : m.wtype;   // F32 matrices are stored as F16 in HBM
    logf(LOG_INFO, "%s: n_vocab=%d n_audio_ctx=%d n_audio_state=%d n_audio_head=%d n_audio_layer=%d n_text_ctx=%d n_text_state=%d n_text_head=%d n_text_layer=%d n_mels=%d ftype=%d\n",
         __func__, hp.n_vocab, hp.n_audio_ctx, hp.n_audio_state, hp.n_audio_head, hp.n_audio_layer, hp.n_text_ctx, hp.n_text_state, hp.n_text_head, hp.n_text_layer, hp.n_mels, hp.ftype);

    // mel filters (src/whisper.cpp:1577-1586)
    R.rd(m.n_filt_mel); R.rd(m.n_filt_fft);
    if (!R.ok || m.n_filt_mel <= 0 || m.n_filt_mel > 1024 || m.n_filt_fft != 201) { set_error("invalid mel filter header (%d x %d)", m.n_filt_mel, m.n_filt_fft); return false; }
    m.filters_host.resize((size_t) m.n_filt_mel * m.n_filt_fft);
    R.rdn(m.filters_host.data(), m.filters_host.size() * 4);

    // vocabulary (src/whisper.cpp:1589-1675)
    {
        int32_t n_vocab = 0; R.rd(n_vocab);
        if (!R.ok || n_vocab < 0 || n_vocab > (1 << 22)) { set_error("invalid vocab size"); return false; }
        std::vector<char> tmp;
        for (int i = 0; i < n_vocab; ++i) {
            uint32_t len = 0; R.rd(len);
            if (!R.ok || len > (1u << 20)) { set_error("invalid vocab entry"); return false; }
            std::string word;
            if (len > 0) { tmp.resize(len); R.rdn(tmp.data(), len); word.assign(tmp.data(), len); }
            vocab.token_to_id[word] = i;
            vocab.id_to_token[i] = word;
        }
        vocab.n_vocab = hp.n_vocab;
        if (vocab.is_multilingual()) {
            vocab.token_eot++; vocab.token_sot++;
            const int dt = vocab.num_languages() - 98;
            vocab.token_translate += dt; vocab.token_transcribe += dt; vocab.token_solm += dt; vocab.token_prev += dt;
            vocab.token_nosp += dt; vocab.token_not += dt; vocab.token_beg += dt;
        }
        for (int i = n_vocab; i < hp.n_vocab; ++i) {
            std::string word;
            if (i > vocab.token_beg)              word = "[_TT_" + std::to_string(i - vocab.token_beg) + "]";
            else if (i == vocab.token_eot)        word = "[_EOT_]";
            else if (i == vocab.token_sot)        word = "[_SOT_]";
            else if (i == vocab.token_translate)  word = "[_TRANSLATE_]";
            else if (i == vocab.token_transcribe) word = "[_TRANSCRIBE_]";
            else if (i == vocab.token_solm)       word = "[_SOLM_]";
            else if (i == vocab.token_prev)       word = "[_PREV_]";
            else if (i == vocab.token_nosp)       word = "[_NOSP_]";
            else if (i == vocab.token_not)        word = "[_NOT_]";
            else if (i == vocab.token_beg)        word = "[_BEG_]";
            else if (i > vocab.token_sot && i <= vocab.token_sot + vocab.num_languages()) {
                const int id = i - vocab.token_sot - 1;
                word = std::string("[_LANG_") + (id >= 0 && id < 100 ? g_lang_codes[id] : "??") + "]";
            } else                                word = "[_extra_token_" + std::to_string(i) + "]";
            vocab.token_to_id[word] = i;
            vocab.id_to_token[i] = word;
        }
    }
    if (!R.ok) { set_error("truncated model file (vocab)"); return false; }
    if (device < 0) return true;

    // ------------------------------------------------------------------ allocate the HBM image
    const int d = hp.n_audio_state, La = hp.n_audio_layer, Lt = hp.n_text_layer, V = hp.n_vocab, M = hp.n_mels;
    auto fvec = [&](size_t n) { return (float *) dalloc(m, n * 4); };
    std::map<std::string, Dest> dests;
    auto add_vec = [&](const std::string & name, float * p, int64_t n) { Dest x; x.kind = Dest::VEC_F32; x.vec = p; x.n = n; dests[name] = x; };
    auto add_mat = [&](const std::string & name, QMat * q, int row_off, int rows, int cols) { Dest x; x.kind = Dest::MAT; x.mat = q; x.row_off = row_off; x.rows = rows; x.cols = cols; dests[name] = x; };

    float * filt = fvec(m.filters_host.size());
    if (!filt) return false;
    WB_CUDA_OK(cudaMemcpy(filt, m.filters_host.data(), m.filters_host.size() * 4, cudaMemcpyHostToDevice));
    m.filters = filt;

    { float * p = fvec((size_t) hp.n_audio_ctx * d); if (!p) return false; m.e_pe = p; add_vec("encoder.positional_embedding", p, (int64_t) hp.n_audio_ctx * d); }
    { float * p = fvec((size_t) hp.n_text_ctx  * d); if (!p) return false; m.d_pe = p; add_vec("decoder.positional_embedding", p, (int64_t) hp.n_text_ctx * d); }
    {
        __half * c1 = (__half *) dalloc(m, (size_t) 3 * d * M * 2); __half * c2 = (__half *) dalloc(m, (size_t) 3 * d * d * 2);
        float * b1 = fvec(d), * b2 = fvec(d);
        if (!c1 || !c2 || !b1 || !b2) return false;
        m.conv1_w = c1; m.conv2_w = c2; m.conv1_b = b1; m.conv2_b = b2;
        Dest x; x.kind = Dest::CONV; x.conv = c1; x.oc = d; x.ic = M; dests["encoder.conv1.weight"] = x;
        x.conv = c2; x.ic = d; dests["encoder.conv2.weight"] = x;
        add_vec("encoder.conv1.bias", b1, d); add_vec("encoder.conv2.bias", b2, d);
    }
    auto add_ln = [&](const std::string & base, LNorm & ln) -> bool {
        float * w = fvec(d), * b = fvec(d); if (!w || !b) return false;
        ln.w = w; ln.b = b; add_vec(base + ".weight", w, d); add_vec(base + ".bias", b, d); return true;
    };
    if (!add_ln("encoder.ln_post", m.e_ln) || !add_ln("decoder.ln", m.d_ln)) return false;
    {   // the persistent decode kernel (wb_decode_mk.cu) reads the decoder matrices in the tile-major layout; WB200_MEGAKERNEL=0
        // keeps them planar for the kernel-per-op chain (odd shapes always use the chain; K-quants need whole super-blocks: d % 256)
        const char * e = getenv("WB200_MEGAKERNEL");
        m.dec_tm = (!e || atoi(e) != 0) && wt_tm_rec_bytes(wt) > 0 && d % 128 == 0 && (!wt_is_kquant(wt) || d % 256 == 0) &&
                   hp.n_text_head * 64 == d && hp.n_text_state == d;
    }
    if (!alloc_qmat(m, wt, V, d, m.d_te, m.dec_tm)) return false;
    add_mat("decoder.token_embedding.weight", &m.d_te, 0, V, d);

    m.enc.resize(La); m.dec.resize(Lt);
    for (int i = 0; i < La; ++i) {
        EncLayerW & L = m.enc[i];
        const std::string p = "encoder.blocks." + std::to_string(i) + ".";
        if (!add_ln(p + "attn_ln", L.ln0) || !add_ln(p + "mlp_ln", L.ln1)) return false;
        if (!alloc_qmat(m, wt, 2*d, d, L.qk) || !alloc_qmat(m, wt, d, d, L.v) || !alloc_qmat(m, wt, d, d, L.o) ||
            !alloc_qmat(m, wt, 4*d, d, L.fc1) || !alloc_qmat(m, wt, d, 4*d, L.fc2)) return false;
        float * qkb = fvec(2*d), * vb = fvec(d), * ob = fvec(d), * f1b = fvec(4*d), * f2b = fvec(d);
        if (!qkb || !vb || !ob || !f1b || !f2b) return false;
        L.qk_bias = qkb; L.v_bias = vb; L.o_bias = ob; L.fc1_bias = f1b; L.fc2_bias = f2b;
        add_mat(p + "attn.query.weight", &L.qk, 0, d, d); add_vec(p + "attn.query.bias", qkb, d);
        add_mat(p + "attn.key.weight",   &L.qk, d, d, d);
        add_mat(p + "attn.value.weight", &L.v,  0, d, d); add_vec(p + "attn.value.bias", vb, d);
        add_mat(p + "attn.out.weight",   &L.o,  0, d, d); add_vec(p + "attn.out.bias", ob, d);
        add_mat(p + "mlp.0.weight", &L.fc1, 0, 4*d, d);   add_vec(p + "mlp.0.bias", f1b, 4*d);
        add_mat(p + "mlp.2.weight", &L.fc2, 0, d, 4*d);   add_vec(p + "mlp.2.bias", f2b, d);
    }
    if (!alloc_qmat(m, wt, 2*Lt*d, d, m.cross_kv)) return false;
    float * cb = fvec((size_t) 2*Lt*d), * cs = fvec((size_t) 2*Lt*d);
    if (!cb || !cs) return false;
    m.cross_bias = cb; m.cross_scale = cs;
    const float kq_scale = powf(64.0f, -0.25f);
    k_fill<<<(Lt*d + 255)/256, 256>>>(cs, kq_scale, (int64_t) Lt*d);
    k_fill<<<(Lt*d + 255)/256, 256>>>(cs + (size_t) Lt*d, 1.0f, (int64_t) Lt*d);
    count_launch(2);
    for (int i = 0; i < Lt; ++i) {
        DecLayerW & L = m.dec[i];
        const std::string p = "decoder.blocks." + std::to_string(i) + ".";
        if (!add_ln(p + "attn_ln", L.ln0) || !add_ln(p + "cross_attn_ln", L.lnc) || !add_ln(p + "mlp_ln", L.lnm)) return false;
        if (!alloc_qmat(m, wt, 3*d, d, L.qkv, m.dec_tm) || !alloc_qmat(m, wt, d, d, L.o, m.dec_tm) || !alloc_qmat(m, wt, d, d, L.cq, m.dec_tm) ||
            !alloc_qmat(m, wt, d, d, L.co, m.dec_tm) || !alloc_qmat(m, wt, 4*d, d, L.fc1, m.dec_tm) || !alloc_qmat(m, wt, d, 4*d, L.fc2, m.dec_tm)) return false;
        float * qb = fvec(3*d), * qs = fvec(3*d), * ob = fvec(d), * cqb = fvec(d), * cob = fvec(d), * f1b = fvec(4*d), * f2b = fvec(d);
        if (!qb || !qs || !ob || !cqb || !cob || !f1b || !f2b) return false;
        k_fill<<<(2*d + 255)/256, 256>>>(qs, kq_scale, 2*d);
        k_fill<<<(d + 255)/256, 256>>>(qs + 2*d, 1.0f, d);
        count_launch(2);
        L.qkv_bias = qb; L.qkv_scale = qs; L.o_bias = ob; L.cq_bias = cqb; L.co_bias = cob; L.fc1_bias = f1b; L.fc2_bias = f2b;
        add_mat(p + "attn.query.weight", &L.qkv, 0,   d, d); add_vec(p + "attn.query.bias", qb, d);
        add_mat(p + "attn.key.weight",   &L.qkv, d,   d, d);
        add_mat(p + "attn.value.weight", &L.qkv, 2*d, d, d); add_vec(p + "attn.value.bias", qb + 2*d, d);
        add_mat(p + "attn.out.weight",   &L.o,   0,   d, d); add_vec(p + "attn.out.bias", ob, d);
        add_mat(p + "cross_attn.query.weight", &L.cq, 0, d, d); add_vec(p + "cross_attn.query.bias", cqb, d);
        add_mat(p + "cross_attn.key.weight",   &m.cross_kv, i*d,        d, d);
        add_mat(p + "cross_attn.value.weight", &m.cross_kv, (Lt + i)*d, d, d); add_vec(p + "cross_attn.value.bias", cb + (size_t) (Lt + i)*d, d);
        add_mat(p + "cross_attn.out.weight",   &L.co, 0, d, d); add_vec(p + "cross_attn.out.bias", cob, d);
        add_mat(p + "mlp.0.weight", &L.fc1, 0, 4*d, d); add_vec(p + "mlp.0.bias", f1b, 4*d);
        add_mat(p + "mlp.2.weight", &L.fc2, 0, d, 4*d); add_vec(p + "mlp.2.bias", f2b, d);
    }

    // ------------------------------------------------------------------ stream the tensor records
    size_t max_bytes = (size_t) V * d * 4;
    max_bytes = std::max(max_bytes, (size_t) 4 * d * d * 4);
    uint8_t * hstage = nullptr; uint8_t * dstage = nullptr;
    if (cudaMallocHost(&hstage, max_bytes) != cudaSuccess) { set_error("cudaMallocHost(%zu) failed", max_bytes); return false; }
    if (cudaMalloc(&dstage, max_bytes + 64) != cudaSuccess) { cudaFreeHost(hstage); set_error("cudaMalloc(staging) failed"); return false; }
    struct Cleanup { uint8_t * h, * d; ~Cleanup() { cudaFreeHost(h); cudaFree(d); } } cleanup{hstage, dstage};

    size_t total = 0;
    m.n_loaded = 0;
    while (true) {
        int32_t n_dims = 0, length = 0, ttype = 0;
        R.ok = true;
        R.rd(n_dims); R.rd(length); R.rd(ttype);
        if (loader->eof(loader->context) || !R.ok) break;
        if (n_dims < 0 || n_dims > 4) { set_error("invalid n_dims %d in model file", n_dims); return false; }
        int64_t ne[4] = { 1, 1, 1, 1 }; int64_t nelements = 1;
        for (int i = 0; i < n_dims; ++i) { int32_t v = 0; R.rd(v); ne[i] = v; nelements *= v; }
        if (length < 0 || length > 4096) { set_error("invalid tensor name length"); return false; }
        std::string name(length, '\0');
        R.rdn(&name[0], length);
        if (!R.ok) { set_error("truncated tensor header"); return false; }
        auto it = dests.find(name);
        if (it == dests.end()) { set_error("unknown tensor '%s' in model file", name.c_str()); return false; }
        Dest & D = it->second;

        size_t nbytes = 0;
        if (ttype == WT_F32) nbytes = (size_t) nelements * 4;
        else if (ttype == WT_F16) nbytes = (size_t) nelements * 2;
        else if (wt_is_block32(ttype) || wt_is_kquant(ttype)) {
            const int bs = wt_is_kquant(ttype) ? 256 : 32;
            if (ne[0] % bs) { set_error("tensor '%s': row length %lld not divisible by block size", name.c_str(), (long long) ne[0]); return false; }
            nbytes = (size_t) ((double) nelements * wt_bpw(ttype) + 0.5);
        } else if (host_dq_supported(ttype) && ttype == host_dq) {
            if (ne[0] % host_dq_block_values(ttype)) { set_error("tensor '%s': row length %lld not divisible by block size", name.c_str(), (long long) ne[0]); return false; }
            nbytes = (size_t) (nelements / host_dq_block_values(ttype)) * host_dq_block_bytes(ttype);
        } else { set_error("tensor '%s' has unsupported type %d", name.c_str(), ttype); return false; }
        const bool expand = host_dq >= 0 && ttype == host_dq;     // blocks -> f32 on the host, then the ordinary F32 -> F16 upload
        if (nbytes > max_bytes || (expand && (size_t) nelements * 4 > max_bytes)) { set_error("tensor '%s' is larger than expected", name.c_str()); return false; }
        const int file_ttype = ttype;                              // what the record says; `ttype` below is what is staged on the device
        const size_t file_bytes = nbytes;
        if (expand) {
            std::vector<uint8_t> blocks(nbytes);
            R.rdn(blocks.data(), nbytes);
            if (!R.ok) { set_error("truncated data for tensor '%s'", name.c_str()); return false; }
            host_dequantize(ttype, blocks.data(), reinterpret_cast<float *>(hstage), nelements);
            nbytes = (size_t) nelements * 4; ttype = WT_F32;
        } else {
            R.rdn(hstage, nbytes);
            if (!R.ok) { set_error("truncated data for tensor '%s'", name.c_str()); return false; }
        }
        WB_CUDA_OK(cudaMemcpy(dstage, hstage, nbytes, cudaMemcpyHostToDevice));

        if (D.kind == Dest::VEC_F32) {
            if (nelements != D.n) { set_error("tensor '%s' has wrong size in model file", name.c_str()); return false; }
            if (ttype == WT_F32) WB_CUDA_OK(cudaMemcpy(D.vec, dstage, nbytes, cudaMemcpyDeviceToDevice));
            else if (ttype == WT_F16) f16_to_f32((const __half *) dstage, D.vec, nelements, 0);
            else { set_error("tensor '%s' must be F32/F16", name.c_str()); return false; }
        } else if (D.kind == Dest::CONV) {
            if (ne[0] != 3 || ne[1] != D.ic || ne[2] != D.oc) { set_error("tensor '%s' has wrong shape in model file", name.c_str()); return false; }
            const __half * src = (const __half *) dstage;
            DevBuf<__half> tmp;
            if (ttype == WT_F32) { if (!tmp.alloc(nelements)) return false; f32_to_f16((const float *) dstage, tmp.p, nelements, 0); src = tmp.p; }
            else if (ttype != WT_F16) { set_error("tensor '%s' must be F16/F32", name.c_str()); return false; }
            k_conv_reorder<<<(int) ((nelements + 255) / 256), 256>>>(src, D.conv, D.oc, D.ic); count_launch();
            WB_CUDA_OK(cudaDeviceSynchronize());
        } else { // MAT
            if (ne[0] != D.cols || ne[1] != D.rows) {
                set_error("tensor '%s' has wrong shape in model file: got [%lld, %lld], expected [%d, %d]", name.c_str(), (long long) ne[0], (long long) ne[1], D.cols, D.rows);
                return false;
            }
            if (file_ttype != file_wtype) { set_error("tensor '%s' has type %d, expected %d", name.c_str(), file_ttype, file_wtype); return false; }
            QMat & q = *D.mat;
            const int K = q.K;
            if (q.layout == 1) {
                const uint8_t * src = dstage;
                DevBuf<__half> tmp;
                if (q.type == WT_F16 && ttype == WT_F32) { if (!tmp.alloc(nelements)) return false; f32_to_f16((const float *) dstage, tmp.p, nelements, 0); src = (const uint8_t *) tmp.p; }
                if (!repack_tile_major(q.type, src, q, D.row_off, D.rows, 0)) return false;
                WB_CUDA_OK(cudaDeviceSynchronize());
            } else if (q.type == WT_F16) {
                __half * dst = (__half *) q.base + (size_t) D.row_off * K;
                if (ttype == WT_F16) WB_CUDA_OK(cudaMemcpy(dst, dstage, nbytes, cudaMemcpyDeviceToDevice));
                else f32_to_f16((const float *) dstage, dst, nelements, 0);
            } else if (wt_is_block32(q.type)) {
                QMat sub = q;
                const size_t boff = (size_t) D.row_off * (K / 32);
                sub.qs = q.qs + boff * wt_qs_bytes(q.type); sub.d = q.d + boff; sub.qh = q.qh ? q.qh + boff : nullptr; sub.m = q.m ? q.m + boff : nullptr;
                if (!repack_block32_into(q.type, dstage, sub, D.rows, K, 0)) return false;
            } else {
                const size_t bpr = (size_t) (K / 256) * wt_kq_block_bytes(q.type);
                WB_CUDA_OK(cudaMemcpy((uint8_t *) q.base + (size_t) D.row_off * bpr, dstage, nbytes, cudaMemcpyDeviceToDevice));
            }
        }
        WB_CUDA_OK(cudaDeviceSynchronize());
        D.seen = true;
        total += file_bytes;
        m.n_loaded++;
    }
    logf(LOG_INFO, "%s: model size = %.2f MB (%d tensors), HBM image = %.2f MB\n", __func__, total / 1e6, m.n_loaded, m.bytes_weights / 1e6);
    if (m.n_loaded == 0) {
        logf(LOG_WARN, "%s: WARN no tensors loaded from model file - assuming empty model for testing\n", __func__);
    } else if (m.n_loaded != (int) dests.size()) {
        set_error("not all tensors loaded from model file - expected %zu, got %d", dests.size(), m.n_loaded);
        return false;
    }
    // Encoder-side matrices of a quantised model are kept a second time as f16 [N][K] (large-v3: 1.26 GB + 0.21 GB cross K/V projections
    // next to the 0.58 GB of blocks): the persistent tensor-core GEMM takes both operands through TMA, and a 30-s window multiplies every
    // weight by 1500 activations -- expanding once at load instead of once per launch (or, first generation, once per CTA) costs 1.5 GB
    // of the 80 GB.  WB200_ENC_F16=0 keeps only the blocks (the GEMM then expands each matrix into a scratch per launch).
    if (m.n_loaded > 0 && device >= 0 && m.wtype != WT_F16 && m.wtype != WT_F32 && !(getenv("WB200_ENC_F16") && atoi(getenv("WB200_ENC_F16")) == 0) &&
        getenv("WB200_GEMM_V1") == nullptr) {
        auto expand = [&](QMat & W) -> bool {
            void * p = nullptr;
            if (cudaMalloc(&p, (size_t) W.N * W.K * sizeof(__half)) != cudaSuccess) { set_error("cudaMalloc of the f16 expansion failed"); return false; }
            m.allocs.push_back(p);
            if (dequant_to_f16(W, W.N, (__half *) p, 0) != cudaSuccess) { set_error("dequant_to_f16 failed"); return false; }
            W.f16 = (const __half *) p;
            return true;
        };
        for (auto & L : m.enc) if (!expand(L.qk) || !expand(L.v) || !expand(L.o) || !expand(L.fc1) || !expand(L.fc2)) return false;
        if (!expand(m.cross_kv)) return false;
        WB_CUDA_OK(cudaDeviceSynchronize());
    }
    m.t_load_us = std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now() - t0).count();
    return true;
}

} // namespace wb

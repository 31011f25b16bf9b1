// ggml_b200_backend.cpp -- ggml backend PLUGIN in front of the engine (SURVEY.md section 8(b) "secondary seam", 8(f) rank 2).
//
// Built into libggml-b200.so and loaded by an UNMODIFIED reference program through GGML_BACKEND_PATH (ggml_backend_load_all,
// reference ggml/src/ggml-backend-reg.cpp:562-591).  It implements the plugin interface of ggml/src/ggml-backend-impl.h:17-267:
// a registry with one GPU-type device, a buffer type, a backend whose graph_compute receives whisper.cpp's four graphs WHOLE (the
// device claims every op, so ggml_backend_sched never splits them) and recognises them by the names of their inputs
// ("mel", "embd_conv", "embd_enc", "embd" / "position" / "KQ_mask": src/whisper.cpp:2004, 2023, 2031, 2507-2517).
//
// This engine does not execute ggml graphs node by node (stacked weight matrices, head-major cross K/V, one persistent kernel per decoder
// pass), so the plugin maps GRAPHS to engine calls:
//   conv graph     -> keeps the mel window of the graph's input
//   encoder graph  -> hands it on (matched through the "embd_conv" / "embd_enc" tensors the graphs share)
//   cross graph    -> whisper_set_mel + whisper_encode on the engine state that belongs to this host state (identified by the kv_cross
//                     tensor the graph copies into); the engine keeps the cross K/V in its own layout
//   decoder graph  -> wb200_decode_explicit: tokens and positions from "embd" / "position", the cells a row is stored in from the
//                     offset of the K-cache view the graph copies into (kv_head), the cells it attends to from the zeros of
//                     "KQ_mask" (src/whisper.cpp:2580-2599, 2928-2938); logits are written into the graph's last node.
// Tensors handed to this backend live in plain host memory owned by the buffer objects (the host program reads / writes them only through
// set_tensor / get_tensor); the weights the host uploads are NOT used: the engine builds its own layouts from the model FILE, which the
// plugin finds among the host's open file descriptors while the host is loading it (or WB200_PLUGIN_MODEL=<path>).
// libwhisper_b200.so exports the same whisper_* names as the host's own libwhisper, so it is opened with RTLD_LOCAL | RTLD_DEEPBIND and
// called through function pointers only.
// Not supported through this seam (the graphs are not executed node by node): a reduced audio_ctx, DTW token timestamps (the decoder
// graph's aheads_cross_QKs output is not produced; they need flash_attn = false anyway), the VAD graph (runs on the host's CPU backend:
// whisper_vad builds its own scheduler), models given as memory buffers unless WB200_PLUGIN_MODEL names the file, and more than ONE
// whisper model per process (the engine context is created once, from the first model file seen).
#include <dlfcn.h>
#include <dirent.h>
#include <unistd.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "ggml.h"
#include "ggml-backend.h"
#include "ggml-backend-impl.h"
#include "ggml-impl.h"
#include "whisper.h"

namespace {

#define PLOG(...) do { if (g.verbose) { fprintf(stderr, "ggml-b200: " __VA_ARGS__); fputc('\n', stderr); } } while (0)

struct Api {                                  // libwhisper_b200.so, through dlsym
    void * h = nullptr;
    whisper_context_params (*context_default_params)() = nullptr;
    whisper_context * (*init_from_file_no_state)(const char *, whisper_context_params) = nullptr;
    whisper_state * (*init_state)(whisper_context *) = nullptr;
    void (*free_state)(whisper_state *) = nullptr;
    void (*free_ctx)(whisper_context *) = nullptr;
    int (*set_mel_with_state)(whisper_context *, whisper_state *, const float *, int, int) = nullptr;
    int (*encode_with_state)(whisper_context *, whisper_state *, int, int) = nullptr;
    int (*n_vocab)(whisper_context *) = nullptr;
    int (*n_text_state)(whisper_context *) = nullptr;
    int (*n_text_layer)(whisper_context *) = nullptr;
    int (*n_audio_ctx)(whisper_context *) = nullptr;
    int (*decode_explicit)(whisper_context *, whisper_state *, const whisper_token *, const int *, int, const int *, const int *, int, const int *, int, float *) = nullptr;
    const char * (*last_error)() = nullptr;
};

struct Global {
    std::mutex mu;
    bool verbose = false, dry = false;
    Api api;
    std::string model_path;
    whisper_context * ctx = nullptr;          // engine context (weights in the engine's layouts)
    std::map<const ggml_tensor *, whisper_state *> state_of_cross;      // host kv_cross.k tensor -> engine state
    std::map<const ggml_tensor *, std::vector<float>> mel_of;           // "embd_conv" / "embd_enc" tensor of a host state -> its mel window
    std::map<const ggml_tensor *, std::pair<int, int>> mel_shape;       // (n_len, n_mel)
    int64_t n_conv = 0, n_enc = 0, n_cross = 0, n_dec = 0;
    int path_tries = 0;
} g;

bool load_api() {
    if (g.api.h) return true;
    Dl_info info;
    std::string dir = ".";
    if (dladdr((void *) &load_api, &info) && info.dli_fname) { dir = info.dli_fname; const size_t p = dir.find_last_of('/'); dir = p == std::string::npos ? "." : dir.substr(0, p); }
    const char * env = getenv("WB200_PLUGIN_ENGINE");
    const std::string path = env ? env : dir + "/libwhisper_b200.so";
    void * h = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL | RTLD_DEEPBIND);
    if (!h) { fprintf(stderr, "ggml-b200: cannot open %s: %s\n", path.c_str(), dlerror()); return false; }
    Api & a = g.api;
#define SYM(field, name) a.field = (decltype(a.field)) dlsym(h, name); if (!a.field) { fprintf(stderr, "ggml-b200: %s not found in %s\n", name, path.c_str()); return false; }
    SYM(context_default_params, "whisper_context_default_params")
    SYM(init_from_file_no_state, "whisper_init_from_file_with_params_no_state")
    SYM(init_state, "whisper_init_state")
    SYM(free_state, "whisper_free_state")
    SYM(free_ctx, "whisper_free")
    SYM(set_mel_with_state, "whisper_set_mel_with_state")
    SYM(encode_with_state, "whisper_encode_with_state")
    SYM(n_vocab, "whisper_model_n_vocab")
    SYM(n_text_state, "whisper_model_n_text_state")
    SYM(n_text_layer, "whisper_model_n_text_layer")
    SYM(n_audio_ctx, "whisper_model_n_audio_ctx")
    SYM(decode_explicit, "wb200_decode_explicit")
    SYM(last_error, "wb200_last_error")
#undef SYM
    a.h = h;
    return true;
}

// the model file the host is reading: an open descriptor on a regular file that starts with the ggml magic (src/whisper.cpp:1497-1505)
void find_model_path() {
    if (!g.model_path.empty()) return;
    if (const char * e = getenv("WB200_PLUGIN_MODEL")) { g.model_path = e; return; }
    DIR * d = opendir("/proc/self/fd");
    if (!d) return;
    while (dirent * e = readdir(d)) {
        if (e->d_name[0] == '.') continue;
        char link[64], target[4096];
        snprintf(link, sizeof(link), "/proc/self/fd/%s", e->d_name);
        const ssize_t n = readlink(link, target, sizeof(target) - 1);
        if (n <= 0 || target[0] != '/') continue;
        target[n] = 0;
        FILE * f = fopen(target, "rb");
        if (!f) continue;
        uint32_t magic = 0;
        const bool ok = fread(&magic, 4, 1, f) == 1 && magic == 0x67676d6c;
        fclose(f);
        if (ok) { g.model_path = target; break; }
    }
    closedir(d);
    PLOG("model file of the host: %s", g.model_path.empty() ? "(not found)" : g.model_path.c_str());
}

bool ensure_engine() {
    if (g.dry) return true;
    if (g.ctx) return true;
    if (g.model_path.empty()) { fprintf(stderr, "ggml-b200: the model file of the host process was not found (set WB200_PLUGIN_MODEL)\n"); return false; }
    if (!load_api()) return false;
    whisper_context_params cp = g.api.context_default_params();
    cp.use_gpu = true;
    g.ctx = g.api.init_from_file_no_state(g.model_path.c_str(), cp);
    if (!g.ctx) { fprintf(stderr, "ggml-b200: engine could not load %s: %s\n", g.model_path.c_str(), g.api.last_error()); return false; }
    PLOG("engine context ready");
    return true;
}

// ---------------------------------------------------------------------------------------------------------------- buffers
struct Buf { void * base; size_t size; };
const size_t ALIGN = 128;

void buf_free(ggml_backend_buffer_t b) { Buf * x = (Buf *) b->context; free(x->base); delete x; }
void * buf_base(ggml_backend_buffer_t b) { return ((Buf *) b->context)->base; }
void buf_memset(ggml_backend_buffer_t, ggml_tensor * t, uint8_t v, size_t off, size_t sz) { memset((char *) t->data + off, v, sz); }
void buf_set(ggml_backend_buffer_t b, ggml_tensor * t, const void * data, size_t off, size_t sz) {
    // the host uploads the weights while it still has the model file open (src/whisper.cpp:1900-1956): look for it during the first uploads
    if (g.model_path.empty() && g.path_tries < 64) { std::lock_guard<std::mutex> lk(g.mu); ++g.path_tries; find_model_path(); }
    (void) b;
    memcpy((char *) t->data + off, data, sz);
}
void buf_get(ggml_backend_buffer_t, const ggml_tensor * t, void * data, size_t off, size_t sz) { memcpy(data, (const char *) t->data + off, sz); }
void buf_clear(ggml_backend_buffer_t b, uint8_t v) { Buf * x = (Buf *) b->context; memset(x->base, v, x->size); }

const char * buft_name(ggml_backend_buffer_type_t) { return "B200"; }
ggml_backend_buffer_t buft_alloc(ggml_backend_buffer_type_t buft, size_t size) {
    Buf * x = new Buf();
    x->size = size;
    if (posix_memalign(&x->base, ALIGN, size ? size : ALIGN) != 0) { delete x; return nullptr; }
    ggml_backend_buffer_i i = {};
    i.free_buffer = buf_free; i.get_base = buf_base; i.memset_tensor = buf_memset; i.set_tensor = buf_set; i.get_tensor = buf_get; i.clear = buf_clear;
    return ggml_backend_buffer_init(buft, i, x, size);
}
size_t buft_align(ggml_backend_buffer_type_t) { return ALIGN; }
bool buft_is_host(ggml_backend_buffer_type_t) { return false; }

ggml_backend_buffer_type * the_buft();

// ---------------------------------------------------------------------------------------------------------------- graphs
std::string base_name(const ggml_tensor * t) {           // "B200#mel#0" (a copy the scheduler made of a graph input) -> "mel"
    std::string n = t->name;
    const size_t a = n.find('#');
    if (a == std::string::npos) return n;
    const size_t b = n.find('#', a + 1);
    return n.substr(a + 1, b == std::string::npos ? std::string::npos : b - a - 1);
}
const ggml_tensor * root_of(const ggml_tensor * t) { while (t->view_src) t = t->view_src; return t; }

// first source tensor of the graph (following views) whose name is `name`; `as_root`: return the viewed tensor instead of the view
const ggml_tensor * find_src(const ggml_cgraph * gr, const char * name, bool as_root) {
    for (int i = 0; i < gr->n_nodes; ++i)
        for (int s = 0; s < GGML_MAX_SRC; ++s) {
            const ggml_tensor * t = gr->nodes[i]->src[s];
            if (!t) continue;
            if (base_name(t) == name) return t;
            const ggml_tensor * r = root_of(t);
            if (r != t && base_name(r) == name) return as_root ? r : t;
        }
    return nullptr;
}
const ggml_tensor * find_node(const ggml_cgraph * gr, const char * name) {
    for (int i = 0; i < gr->n_nodes; ++i) if (base_name(gr->nodes[i]) == name) return gr->nodes[i];
    return nullptr;
}
const ggml_tensor * first_cpy_dst_root(const ggml_cgraph * gr, const ggml_tensor ** view_out) {
    for (int i = 0; i < gr->n_nodes; ++i) {
        const ggml_tensor * n = gr->nodes[i];
        if (n->op == GGML_OP_CPY && n->src[1] && n->src[1]->view_src) { if (view_out) *view_out = n->src[1]; return root_of(n->src[1]); }
    }
    return nullptr;
}

ggml_status compute_conv(const ggml_cgraph * gr) {
    const ggml_tensor * mel = find_src(gr, "mel", false);
    const ggml_tensor * out = find_node(gr, "embd_conv");
    if (!mel || !out || mel->type != GGML_TYPE_F32) { fprintf(stderr, "ggml-b200: conv graph not understood\n"); return GGML_STATUS_FAILED; }
    std::lock_guard<std::mutex> lk(g.mu);
    std::vector<float> & v = g.mel_of[out];
    v.assign((const float *) mel->data, (const float *) mel->data + ggml_nelements(mel));
    g.mel_shape[out] = { (int) mel->ne[0], (int) mel->ne[1] };                // n_len = 2 * n_ctx (mel-major rows), n_mel
    ++g.n_conv;
    return GGML_STATUS_SUCCESS;
}
ggml_status compute_encoder(const ggml_cgraph * gr) {
    const ggml_tensor * in = find_src(gr, "embd_conv", true);
    const ggml_tensor * out = gr->nodes[gr->n_nodes - 1];                      // wstate.embd_enc: the (unnamed) last node, src/whisper.cpp:2257-2259
    if (!in || !out) { fprintf(stderr, "ggml-b200: encoder graph not understood\n"); return GGML_STATUS_FAILED; }
    std::lock_guard<std::mutex> lk(g.mu);
    auto it = g.mel_of.find(in);
    if (it == g.mel_of.end()) { fprintf(stderr, "ggml-b200: encoder graph without a conv graph before it\n"); return GGML_STATUS_FAILED; }
    if (in != out) { g.mel_of[out] = std::move(it->second); g.mel_shape[out] = g.mel_shape[in]; g.mel_of.erase(in); g.mel_shape.erase(in); }
    ++g.n_enc;
    return GGML_STATUS_SUCCESS;
}
// the encoder output a graph reads (a view of wstate.embd_enc, src/whisper.cpp:2311): a source whose viewed tensor is one an encoder graph produced
const ggml_tensor * find_enc_out(const ggml_cgraph * gr) {
    std::lock_guard<std::mutex> lk(g.mu);
    for (int i = 0; i < gr->n_nodes; ++i)
        for (int s = 0; s < GGML_MAX_SRC; ++s) {
            const ggml_tensor * t = gr->nodes[i]->src[s];
            if (t && g.mel_of.count(root_of(t))) return root_of(t);
        }
    return nullptr;
}
ggml_status compute_cross(const ggml_cgraph * gr) {
    const ggml_tensor * in = find_enc_out(gr);
    const ggml_tensor * kc = first_cpy_dst_root(gr, nullptr);
    if (!in || !kc) { fprintf(stderr, "ggml-b200: cross graph not understood\n"); return GGML_STATUS_FAILED; }
    std::vector<float> mel; std::pair<int, int> shape;
    whisper_state * st = nullptr;
    {
        std::lock_guard<std::mutex> lk(g.mu);
        auto it = g.mel_of.find(in);
        if (it == g.mel_of.end()) { fprintf(stderr, "ggml-b200: cross graph without an encoder graph before it\n"); return GGML_STATUS_FAILED; }
        mel.swap(it->second); shape = g.mel_shape[in];
        g.mel_of.erase(in); g.mel_shape.erase(in);
        ++g.n_cross;
        if (!ensure_engine()) return GGML_STATUS_FAILED;
        if (g.dry) { g.state_of_cross[kc] = nullptr; return GGML_STATUS_SUCCESS; }
        auto is = g.state_of_cross.find(kc);
        if (is == g.state_of_cross.end()) {
            st = g.api.init_state(g.ctx);
            if (!st) { fprintf(stderr, "ggml-b200: whisper_init_state failed: %s\n", g.api.last_error()); return GGML_STATUS_FAILED; }
            g.state_of_cross[kc] = st;
            PLOG("engine state %zu for host kv_cross %p", g.state_of_cross.size(), (const void *) kc);
        } else st = is->second;
    }
    if (shape.first != 2 * g.api.n_audio_ctx(g.ctx)) {          // whisper_full_params.audio_ctx / whisper_set_audio_ctx: the engine state would need the same override
        fprintf(stderr, "ggml-b200: mel window of %d frames: a reduced audio_ctx is not supported through the plugin\n", shape.first); return GGML_STATUS_FAILED;
    }
    // the window of the host (already cut out of the clip and zero-padded, src/whisper.cpp:2389-2411) becomes the engine state's whole mel
    if (g.api.set_mel_with_state(g.ctx, st, mel.data(), shape.first, shape.second) != 0 || g.api.encode_with_state(g.ctx, st, 0, 1) != 0) {
        fprintf(stderr, "ggml-b200: encode failed: %s\n", g.api.last_error()); return GGML_STATUS_FAILED;
    }
    return GGML_STATUS_SUCCESS;
}
ggml_status compute_decoder(const ggml_cgraph * gr) {
    const ggml_tensor * embd = find_src(gr, "embd", false), * position = find_src(gr, "position", false), * mask = find_src(gr, "KQ_mask", false);
    const ggml_tensor * kview = nullptr;
    const ggml_tensor * kself = first_cpy_dst_root(gr, &kview);
    ggml_tensor * logits = gr->nodes[gr->n_nodes - 1];
    if (!embd || !position || !mask || !kself || embd->type != GGML_TYPE_I32 || position->type != GGML_TYPE_I32 || mask->type != GGML_TYPE_F32 || logits->type != GGML_TYPE_F32) {
        fprintf(stderr, "ggml-b200: decoder graph not understood\n"); return GGML_STATUS_FAILED;
    }
    whisper_state * st = nullptr; bool found = false;
    {
        std::lock_guard<std::mutex> lk(g.mu);
        ++g.n_dec;
        for (int i = 0; i < gr->n_nodes && !found; ++i)
            for (int s = 0; s < GGML_MAX_SRC && !found; ++s) {
                const ggml_tensor * t = gr->nodes[i]->src[s];
                if (!t || !t->view_src) continue;
                auto it = g.state_of_cross.find(root_of(t));
                if (it != g.state_of_cross.end()) { st = it->second; found = true; }
            }
    }
    if (!found) { fprintf(stderr, "ggml-b200: decoder graph of a state that never ran the cross graph\n"); return GGML_STATUS_FAILED; }
    const int n = (int) embd->ne[0], n_kv = (int) mask->ne[0];
    const int V = (int) logits->ne[0];
    if ((int) logits->ne[1] != n) { fprintf(stderr, "ggml-b200: logits shape\n"); return GGML_STATUS_FAILED; }
    if (g.dry) { memset(logits->data, 0, ggml_nbytes(logits)); return GGML_STATUS_SUCCESS; }
    const int d = g.api.n_text_state(g.ctx), L = g.api.n_text_layer(g.ctx);
    const int kv_head = (int) (kview->view_offs / (ggml_element_size(kself) * (size_t) d));        // layer 0: offset = elt * d * (0 * n_ctx + kv_head)
    const int n_ctx = (int) (kself->ne[0] / ((int64_t) d * L));
    if (V != g.api.n_vocab(g.ctx) || kv_head < 0 || kv_head + n > n_ctx) { fprintf(stderr, "ggml-b200: decoder graph geometry (V %d, kv_head %d, n %d, n_ctx %d)\n", V, kv_head, n, n_ctx); return GGML_STATUS_FAILED; }
    const float * m = (const float *) mask->data;
    std::vector<int> cells(n), nkv(n), idx((size_t) n * n_kv);
    for (int j = 0; j < n; ++j) {
        cells[j] = kv_head + j;
        int c = 0;
        for (int i = 0; i < n_kv; ++i) if (m[(size_t) j * n_kv + i] == 0.0f) idx[(size_t) j * n_kv + c++] = i;
        nkv[j] = c;
    }
    if (g.api.decode_explicit(g.ctx, st, (const whisper_token *) embd->data, (const int *) position->data, n, cells.data(), idx.data(), n_kv, nkv.data(), n_ctx,
                              (float *) logits->data) != 0) {
        fprintf(stderr, "ggml-b200: decode failed: %s\n", g.api.last_error()); return GGML_STATUS_FAILED;
    }
    return GGML_STATUS_SUCCESS;
}

// ---------------------------------------------------------------------------------------------------------------- backend / device / registry
const char * backend_name(ggml_backend_t) { return "B200"; }
void backend_free(ggml_backend_t b) { delete b; }
ggml_status backend_graph_compute(ggml_backend_t, ggml_cgraph * gr) {
    if (gr->n_nodes == 0) return GGML_STATUS_SUCCESS;
    if (find_src(gr, "mel", false)) return compute_conv(gr);
    if (find_src(gr, "embd", false) && find_src(gr, "KQ_mask", false)) return compute_decoder(gr);
    if (find_src(gr, "embd_conv", true)) return compute_encoder(gr);
    if (find_enc_out(gr)) return compute_cross(gr);
    fprintf(stderr, "ggml-b200: a graph of %d nodes that is none of whisper.cpp's four (this backend runs whisper graphs only)\n", gr->n_nodes);
    return GGML_STATUS_FAILED;
}
ggml_guid_t backend_guid() { static ggml_guid guid = { 0xb2, 0x00, 0x77, 0x68, 0x69, 0x73, 0x70, 0x65, 0x72, 0x2e, 0x63, 0x70, 0x70, 0x5f, 0x62, 0x32 }; return &guid; }

ggml_backend_reg * the_reg();
ggml_backend_device * the_dev();

const char * dev_name(ggml_backend_dev_t) { return "B200"; }
const char * dev_desc(ggml_backend_dev_t) { return "whisper.cpp_b200 engine (sm_90a) behind the ggml backend interface"; }
void dev_memory(ggml_backend_dev_t, size_t * free_b, size_t * total) { *free_b = (size_t) 160 << 30; *total = (size_t) 180 << 30; }
enum ggml_backend_dev_type dev_type(ggml_backend_dev_t) { return GGML_BACKEND_DEVICE_TYPE_GPU; }
void dev_props(ggml_backend_dev_t dev, ggml_backend_dev_props * p) {
    memset(p, 0, sizeof(*p));
    p->name = dev_name(dev); p->description = dev_desc(dev); p->type = dev_type(dev);
    dev_memory(dev, &p->memory_free, &p->memory_total);
    p->caps.async = false; p->caps.host_buffer = false; p->caps.buffer_from_host_ptr = false; p->caps.events = false;
}
ggml_backend_t dev_init(ggml_backend_dev_t dev, const char *) {
    ggml_backend_i i = {};
    i.get_name = backend_name; i.free = backend_free; i.graph_compute = backend_graph_compute;
    ggml_backend * b = new ggml_backend();
    b->guid = backend_guid(); b->iface = i; b->device = dev; b->context = nullptr;
    return b;
}
ggml_backend_buffer_type_t dev_buft(ggml_backend_dev_t) { return the_buft(); }
bool dev_supports_op(ggml_backend_dev_t, const ggml_tensor *) { return true; }                  // whole graphs come here: they are mapped to engine calls, not executed node by node
bool dev_supports_buft(ggml_backend_dev_t, ggml_backend_buffer_type_t buft) { return buft == the_buft(); }
bool dev_offload_op(ggml_backend_dev_t, const ggml_tensor *) { return false; }

const char * reg_name(ggml_backend_reg_t) { return "B200"; }
size_t reg_count(ggml_backend_reg_t) { return 1; }
ggml_backend_dev_t reg_device(ggml_backend_reg_t, size_t) { return the_dev(); }
void * reg_proc(ggml_backend_reg_t, const char *) { return nullptr; }

ggml_backend_buffer_type * the_buft() {
    static ggml_backend_buffer_type t = [] {
        ggml_backend_buffer_type x = {};
        x.iface.get_name = buft_name; x.iface.alloc_buffer = buft_alloc; x.iface.get_alignment = buft_align; x.iface.is_host = buft_is_host;
        x.device = the_dev(); x.context = nullptr;
        return x;
    }();
    return &t;
}
ggml_backend_device * the_dev() {
    static ggml_backend_device d = [] {
        ggml_backend_device x = {};
        x.iface.get_name = dev_name; x.iface.get_description = dev_desc; x.iface.get_memory = dev_memory; x.iface.get_type = dev_type; x.iface.get_props = dev_props;
        x.iface.init_backend = dev_init; x.iface.get_buffer_type = dev_buft; x.iface.supports_op = dev_supports_op; x.iface.supports_buft = dev_supports_buft;
        x.iface.offload_op = dev_offload_op;
        x.reg = the_reg(); x.context = nullptr;
        return x;
    }();
    return &d;
}
ggml_backend_reg * the_reg() {
    static ggml_backend_reg r = [] {
        ggml_backend_reg x = {};
        x.api_version = GGML_BACKEND_API_VERSION;
        x.iface.get_name = reg_name; x.iface.get_device_count = reg_count; x.iface.get_device = reg_device; x.iface.get_proc_address = reg_proc;
        x.context = nullptr;
        return x;
    }();
    return &r;
}

} // namespace

extern "C" {
__attribute__((visibility("default"))) ggml_backend_reg_t ggml_backend_init(void) {
    g.verbose = getenv("WB200_PLUGIN_VERBOSE") != nullptr;
    g.dry = getenv("WB200_PLUGIN_DRY") != nullptr;           // CPU-only check of the plugin plumbing: graphs are parsed, nothing is computed (logits = 0)
    PLOG("registered (api version %d)%s", GGML_BACKEND_API_VERSION, g.dry ? ", dry run" : "");
    return the_reg();
}
__attribute__((visibility("default"))) int ggml_backend_score(void) { return 1; }
// counters for the tests: graphs seen per kind
__attribute__((visibility("default"))) void wb200_plugin_counts(long long * out4) { out4[0] = g.n_conv; out4[1] = g.n_enc; out4[2] = g.n_cross; out4[3] = g.n_dec; }
}

// wb_api.cpp -- the whisper.h C ABI (include/whisper_b200.h) except whisper_full* (wb_full.cpp):
// context / state lifecycle, low-level mel/encode/decode entry points, tokenizer, language table, getters, timings.
// Behavioural reference: src/whisper.cpp:3284-3332 (tokenizer), 3386-3557 (state), 3618-4323 (API bodies).
#include <algorithm>
#include <chrono>
#include <cstring>
#include <fstream>
#include <regex>
#include <thread>
#include "wb_state.h"
#include "wb_dtw.h"
#include <linux/futex.h>
#include <sys/syscall.h>
#include <unistd.h>
#include "wb_kernels.cuh"
#include "wb_gemm.cuh"

using namespace wb;

namespace wb {
extern const char * const g_lang_codes[100];
extern const char * const g_lang_names[100];
void set_log_sink(void (*cb)(int, const char *, void *), void * ud);

bool & tls_pcm_is_device() { static thread_local bool f = false; return f; }

int64_t time_us() {
    return std::chrono::duration_cast<std::chrono::microseconds>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// ---------------------------------------------------------------------------------------------------- KV bookkeeping
bool KvCells::find_slot(const int * pos, const int * seq, uint32_t n_tokens) {       // whisper.cpp:1019-1068
    if (n_tokens > size) { set_error("kv: n_tokens=%u > n_ctx=%u", n_tokens, size); return false; }
    uint32_t tested = 0;
    for (;;) {
        if (head + n_tokens > size) { tested += size - head; head = 0; continue; }
        bool ok = true;
        for (uint32_t i = 0; i < n_tokens; ++i) {
            if (cells[head + i].pos >= 0) { ok = false; head += i + 1; tested += i + 1; break; }
        }
        if (ok) break;
        if (tested >= size) return false;
    }
    for (uint32_t i = 0; i < n_tokens; ++i) { cells[head + i].pos = pos[i]; cells[head + i].seqs |= 1u << seq[i]; }
    return true;
}
int KvCells::cell_max() const {                                                      // whisper.cpp:1071-1079
    for (uint32_t i = size - 1; i > 0; --i) if (cells[i].pos >= 0 && cells[i].seqs) return (int) i + 1;
    return 1;
}
void KvCells::seq_rm(int seq, int p0, int p1) {                                      // whisper.cpp:1091-1119
    uint32_t new_head = size;
    if (p0 < 0) p0 = 0;
    if (p1 < 0) p1 = INT32_MAX;
    for (uint32_t i = 0; i < size; ++i) {
        Cell & c = cells[i];
        if (c.pos >= p0 && c.pos < p1) {
            if (seq < 0) c.seqs = 0;
            else if (c.seqs & (1u << seq)) c.seqs &= ~(1u << seq);
            else continue;
            if (!c.seqs) { c.pos = -1; if (new_head == size) new_head = i; }
        }
    }
    if (new_head != size) head = new_head;
}
void KvCells::seq_cp(int src, int dst, int p0, int p1) {                             // whisper.cpp:1121-1137
    if (p0 < 0) p0 = 0;
    if (p1 < 0) p1 = INT32_MAX;
    head = 0;
    for (auto & c : cells) if ((c.seqs & (1u << src)) && c.pos >= p0 && c.pos < p1) c.seqs |= 1u << dst;
}

// host-only test hook: run a script of KV bookkeeping operations on a stand-alone cell table (same encoding as the oracle's
// wref_kv_script, oracle/ref_harness.cpp)
extern "C" WB_EXPORT int wb200_dbg_kv_script(int size, const int * ops, int n_ops, int * trace, int * cells_out) {
    if (size <= 0 || !ops || !trace || !cells_out) return -1;
    KvCells kv; kv.reset((uint32_t) size);
    for (int o = 0; o < n_ops; ++o) {
        const int * q = ops + 5 * o;
        int ret = 1;
        if (q[0] == 0) {
            std::vector<int> pos(q[1]), seq(q[1], q[3]);
            for (int i = 0; i < q[1]; ++i) pos[i] = q[2] + i;
            ret = kv.find_slot(pos.data(), seq.data(), (uint32_t) q[1]) ? 1 : 0;
        } else if (q[0] == 1) kv.seq_rm(q[1], q[2], q[3]);
        else if (q[0] == 2)   kv.seq_cp(q[1], q[2], q[3], q[4]);
        else                  kv.clear();
        trace[3 * o] = ret; trace[3 * o + 1] = (int) kv.head; trace[3 * o + 2] = kv.cell_max();
    }
    for (int i = 0; i < size; ++i) { cells_out[2 * i] = kv.cells[i].pos; cells_out[2 * i + 1] = (int) kv.cells[i].seqs; }
    return 0;
}

// ---------------------------------------------------------------------------------------------------- engine glue
namespace {
// host-side preparation of one decode request: KV slot search + attention index lists (whisper.cpp:2876-2948)
struct PreparedDecode {
    std::vector<DecToken> rows; std::vector<int> cells, nkv, idx; int ld = 0;
};
bool prepare_rows(KvCells & kv, const whisper_state & st, const int * tokens, const int * pos, const int * seq, const int8_t * want, int n_tokens, PreparedDecode & P) {
    if (!kv.find_slot(pos, seq, (uint32_t) n_tokens)) { set_error("decode: no KV slot for %d tokens", n_tokens); return false; }
    kv.n = (uint32_t) std::min<int>((int) kv.size, std::max(1, kv.cell_max()));      // padding 1 on this path (whisper.cpp:2884-2885)
    const int n_kv = (int) kv.n;
    P.ld = n_kv;
    P.rows.resize(n_tokens); P.cells.resize(n_tokens); P.nkv.resize(n_tokens); P.idx.assign((size_t) n_tokens * n_kv, 0);
    for (int j = 0; j < n_tokens; ++j) {
        P.rows[j] = { tokens[j], pos[j], seq[j], st.slot, want[j] != 0 };
        P.cells[j] = st.cell_off + (int) kv.head + j;
        int c = 0;
        for (int i = 0; i < n_kv; ++i) {                                              // KQ_mask rule, whisper.cpp:2928-2938
            const KvCells::Cell & cell = kv.cells[i];
            if ((cell.seqs & (1u << seq[j])) && cell.pos <= pos[j]) P.idx[(size_t) j * n_kv + c++] = st.cell_off + i;
        }
        P.nkv[j] = c;
    }
    return true;
}
bool prepare_decode(whisper_state & st, const int * tokens, const int * pos, const int * seq, const int8_t * want, int n_tokens, PreparedDecode & P) {
    return prepare_rows(st.kv, st, tokens, pos, seq, want, n_tokens, P);
}
// test hook (engine-less states): per row a hash of the positions it attends to, i.e. of the index list the kernels would get
void scripted_attended(whisper_state & st, const PreparedDecode & P, int n_tokens) {
    st.dbg_att.resize((size_t) n_tokens);
    std::vector<int> ps;
    for (int j = 0; j < n_tokens; ++j) {
        ps.clear();
        for (int c = 0; c < P.nkv[j]; ++c) ps.push_back(st.kv.cells[(size_t) (P.idx[(size_t) j * P.ld + c] - st.cell_off)].pos);
        std::sort(ps.begin(), ps.end());
        uint64_t h = 1469598103934665603ull;
        for (int v : ps) for (int k = 0; k < 4; ++k) { h ^= (uint64_t) ((v >> (8 * k)) & 0xff); h *= 1099511628211ull; }
        st.dbg_att[(size_t) j] = h;
    }
}
// keep whisper_state::lrows / row0_copy in step with what the reference's logits buffer would hold after this decode
void note_rows(const whisper_context & ctx, whisper_state & st, const int8_t * want, int n_tokens) {
    const int n = ctx.vocab.n_vocab, nosp = ctx.vocab.token_nosp;
    whisper_state::LogitRow zero; zero.mx = 0.0f; zero.sum = (float) n; zero.nosp = 0.0f;          // a zero-filled row
    st.lrows.resize((size_t) n_tokens, zero);
    const bool dev = !st.samp_out.empty();
    for (int j = 0; j < n_tokens; ++j) {
        if (!want[j]) continue;
        whisper_state::LogitRow & r = st.lrows[(size_t) j];
        if (dev) { const SampOut & o = st.samp_out[(size_t) j * st.samp_stride]; r.mx = o.raw_max; r.sum = o.raw_sum; r.nosp = o.raw_nosp; }
        else if (st.logits.size() >= (size_t) (j + 1) * n) {
            const float * l = st.logits.data() + (size_t) j * n;
            float mx = -INFINITY; for (int i = 0; i < n; ++i) mx = std::max(mx, l[i]);
            float sum = 0.0f; for (int i = 0; i < n; ++i) if (l[i] > -INFINITY) sum += expf(l[i] - mx);
            r.mx = mx; r.sum = sum; r.nosp = l[nosp];
        }
        if (j == 0) {
            st.row0_is_copy = !dev && st.logits.size() >= (size_t) n;
            if (st.row0_is_copy) st.row0_copy.assign(st.logits.begin(), st.logits.begin() + n);
        }
    }
}
void account_decode(whisper_state & st, int n_tokens, int64_t dt) {                    // whisper.cpp:2974-2983
    if (n_tokens == 1)      { st.t_decode_us += dt; st.n_decode++; }
    else if (n_tokens < 16) { st.t_batchd_us += dt; st.n_batchd += n_tokens; }
    else                    { st.t_prompt_us += dt; st.n_prompt += n_tokens; }
}
} // namespace

bool encode_window(whisper_context & ctx, whisper_state & st, int mel_offset) {
    const int n_ctx = st.exp_n_audio_ctx > 0 ? st.exp_n_audio_ctx : ctx.model.hp.n_audio_ctx;

    if (st.fe.n_mel != ctx.model.hp.n_mels) { set_error("encode: mel has %d bands, model expects %d", st.fe.n_mel, ctx.model.hp.n_mels); return false; }
    if (!st.group) { set_error("encode: the state is not attached to a device pool"); return false; }
    Group::Req r; r.kind = 0; r.ctx = &ctx; r.st = &st; r.seek = mel_offset; r.n_ctx = n_ctx;
    if (!st.group->submit(r)) return false;
    st.t_encode_us += r.dt_us;
    st.n_encode++;
    return true;
}

bool decode_batch(whisper_context & ctx, whisper_state & st, const int * tokens, const int * pos, const int * seq,
                  const int8_t * want, int n_tokens, const SampReq * samp, int dtw_n_ctx, int dtw_sot_len, int dtw_n_frames) {
    if (st.scripted) {                                                       // test hook: what was fed to the decoder (wb200_dbg_last_batch)
        st.dbg_tok.assign(tokens, tokens + n_tokens); st.dbg_pos.assign(pos, pos + n_tokens);
        st.dbg_seq.assign(seq, seq + n_tokens); st.dbg_want.assign(want, want + n_tokens);
    }
    if (!st.group) { set_error("decode: the state is not attached to a device pool"); return false; }
    Group::Req r; r.kind = 1; r.ctx = &ctx; r.st = &st; r.tokens = tokens; r.pos = pos; r.seq = seq; r.want = want; r.n = n_tokens; r.samp = samp;
    r.dtw_n_ctx = dtw_n_ctx; r.dtw_sot_len = dtw_sot_len; r.dtw_n_frames = dtw_n_frames;
    if (!st.group->submit(r)) return false;
    account_decode(st, n_tokens, r.dt_us);
    note_rows(ctx, st, want, n_tokens);
    return true;
}

// ---------------------------------------------------------------------------------------------------- batch group
// A member blocks on the futex word of its own request; the thread that completes the rendezvous runs the batch and wakes the
// others one by one.  (A condition variable made all 63 sleepers re-acquire one mutex after every decode step.)
static void req_wait(Group::Req & r) {
    while (r.done.load(std::memory_order_acquire) == 0)
        syscall(SYS_futex, reinterpret_cast<int *>(&r.done), FUTEX_WAIT_PRIVATE, 0, nullptr, nullptr, 0);
}
static void req_wake(Group::Req & r) {
    r.done.store(1, std::memory_order_release);
    syscall(SYS_futex, reinterpret_cast<int *>(&r.done), FUTEX_WAKE_PRIVATE, 1, nullptr, nullptr, 0);
}
// ---- pool management -----------------------------------------------------------------------------------------------------------
static int pool_cells_for(const Model & m, int n_decoders) {                          // whisper.cpp:3402, 7167-7172
    const int base = (m.hp.n_text_ctx + 255) / 256 * 256;
    return base * (n_decoders > 1 ? n_decoders + 2 : 1);
}

// Reallocate the pool for `new_cap` slots of `new_cps` cells.  Waits until no batch is executing and keeps `mu` so that none can start;
// states blocked in submit() keep their slot contents (Engine::resize copies them).
bool Group::grow_locked(std::unique_lock<std::mutex> & lk, int new_cap, int new_cps) {
    cv.wait(lk, [&] { return !running; });
    spec_drop();                                                                     // the relayout moves cells and cell_off
    if (!scripted) {
        if (cap == 0) {
            if (!eng.init(model, 1)) return false;                                   // one slot, GGML_PAD(n_text_ctx, 256) cells
            if (!eng.dtw_set_heads(dtw_heads)) return false;
            cap = 1; cps = eng.cps;
        }
        if ((new_cap != cap || new_cps != cps) && !eng.resize(new_cap, new_cps)) return false;
    }
    cap = new_cap; cps = new_cps;
    slot_used.resize((size_t) cap, 0);
    return true;
}

bool Group::attach(whisper_state * st) {
    std::unique_lock<std::mutex> lk(mu);
    int slot = -1;
    for (int i = 0; i < cap; ++i) if (!slot_used[(size_t) i]) { slot = i; break; }
    if (slot < 0) {
        const int base_cps = cps > 0 ? cps : pool_cells_for(*model, 1);
        const int new_cap = cap == 0 ? 1 : (cap < 8 ? cap * 2 : cap + std::max(8, cap / 4));     // 1 2 4 8 16 24 32 40 50 62 77 ...
        if (new_cap > 1024) { set_error("whisper_init_state: too many states on one context (%d)", cap); return false; }
        slot = cap;
        if (!grow_locked(lk, new_cap, base_cps)) return false;
    }
    slot_used[(size_t) slot] = 1;
    ++n_registered;
    st->group = this; st->eng = scripted ? nullptr : &eng; st->slot = slot; st->cell_off = slot * cps;
    st->kv.reset((uint32_t) pool_cells_for(*model, 1));
    st->kv_self_n_dec = 1;
    return true;
}

std::unique_ptr<FrontEnd> Group::take_fe() {
    std::lock_guard<std::mutex> lk(mu);
    if (fe_cache.empty()) return nullptr;
    std::unique_ptr<FrontEnd> f = std::move(fe_cache.back());
    fe_cache.pop_back();
    return f;
}

void Group::detach(whisper_state * st) {
    std::unique_lock<std::mutex> lk(mu);
    if (st->slot >= 0 && st->slot < cap) slot_used[(size_t) st->slot] = 0;
    --n_registered;
    if (st->fe_own && st->fe_own->st && fe_cache.size() < 256) fe_cache.push_back(std::move(st->fe_own));
    st->group = nullptr; st->eng = nullptr;
}

bool Group::ensure_cells(whisper_state * st, int cells) {
    std::unique_lock<std::mutex> lk(mu);
    cv.wait(lk, [&] { return !running; });
    spec_drop();                                                                     // kv.reset below rewrites the state's cell table
    if (cells > cps) {
        // another state may hold cells beyond `cells` only if cps already covered them, so growing never truncates anybody
        if (!grow_locked(lk, cap, cells)) return false;
    }
    st->cell_off = st->slot * cps;
    st->kv.reset((uint32_t) cells);
    return true;
}

// ---- rendezvous ------------------------------------------------------------------------------------------------------------------
// Gathering: callers of whisper_full_with_state on different states start within microseconds of each other but not at the same
// instant.  A complete batch that contains an encode request (the first request of a window) is held back for a moment while states
// are still entering, so that the windows of near-simultaneous callers share one batched encoder pass instead of chasing each other
// one step apart.  Costs a lone caller on a multi-state context at most kGatherUs once per 30-s window.
static const int64_t kGatherUs = 300;
int64_t Group::grace_left_us() const {
    if (n_registered <= n_active) return 0;                  // nobody left who could still join
    bool has_enc = false;
    for (const Req * q : pending) has_enc |= (q->kind == 0);
    if (!has_enc) return 0;
    return kGatherUs - (time_us() - t_last_enter_us);
}

void Group::enter(whisper_state * st) {
    std::lock_guard<std::mutex> lk(mu);
    ++n_active; t_last_enter_us = time_us();
    st->in_group_call = true;
    st->cell_off = st->slot * cps;
}

bool Group::submit(Req & r) {
    std::vector<Req *> batch;
    {
        std::unique_lock<std::mutex> lk(mu);
        r.st->cell_off = r.st->slot * cps;                    // the pool may have been re-laid out since the last request
        pending.push_back(&r);
        for (;;) {
            if (r.taken || (int) pending.size() < n_active) { lk.unlock(); req_wait(r); return r.ok; }   // somebody else runs (or ran) it
            const int64_t w = grace_left_us();
            if (w <= 0) break;
            lk.unlock();
            std::this_thread::sleep_for(std::chrono::microseconds(w));
            lk.lock();
        }
        batch.swap(pending);
        for (Req * q : batch) q->taken = true;
        running = true;
    }
    run(batch);
    { std::lock_guard<std::mutex> lk(mu); running = false; }
    cv.notify_all();
    for (Req * q : batch) if (q != &r) req_wake(*q);             // q may be gone as soon as it is woken: nothing of it is touched afterwards
    return r.ok;
}

void Group::deactivate(whisper_state * st, bool clear_flag) {
    std::vector<Req *> batch;
    {
        std::lock_guard<std::mutex> lk(mu);
        if (clear_flag) st->in_group_call = false;
        n_active--;
        if (!pending.empty() && (int) pending.size() >= n_active) {      // everybody else was only waiting for this state
            batch.swap(pending);
            for (Req * q : batch) q->taken = true;
            running = true;
        }
    }
    if (!batch.empty()) {
        run(batch);
        { std::lock_guard<std::mutex> lk(mu); running = false; }
        cv.notify_all();
        for (Req * q : batch) req_wake(*q);
    }
}
void Group::leave(whisper_state * st)   { deactivate(st, true); }
void Group::suspend(whisper_state * st) { deactivate(st, false); }
void Group::resume(whisper_state *)     { std::lock_guard<std::mutex> lk(mu); ++n_active; }

static thread_local std::vector<whisper_state *> tls_call_stack;       // states this thread is executing a whisper.h call for, innermost last
GroupCall::GroupCall(whisper_state * s) : st(s) {
    if (!st || !st->group) return;
    if (!tls_call_stack.empty() && tls_call_stack.back() != st && tls_call_stack.back()->group == st->group && tls_call_stack.back()->in_group_call) {
        suspended = tls_call_stack.back();
        st->group->suspend(suspended);
    }
    if (!st->in_group_call) { st->group->enter(st); entered = true; }
    tls_call_stack.push_back(st);
}
GroupCall::~GroupCall() {
    if (!st || !st->group) return;
    tls_call_stack.pop_back();
    if (entered) st->group->leave(st);
    if (suspended) suspended->group->resume(suspended);
}

void Group::spec_drop() {
    if (!scripted) for (int s = 0; s < Engine::PASS_SLOTS; ++s) eng.pass_wait(s);
    spec_pass = -1; spec_rows.clear();
}

void Group::run(std::vector<Req *> & batch) {
    for (Req * q : batch) q->st->cell_off = q->st->slot * cps;      // the pool may have been re-laid out since the request was queued
    // encode requests first (they only touch the encoder workspaces and the members' cross-KV slots)
    std::vector<Req *> enc, dec;
    for (Req * q : batch) (q->kind == 0 ? enc : dec).push_back(q);
    auto by_slot = [](const Req * a, const Req * b) { return a->st->slot < b->st->slot; };
    std::sort(enc.begin(), enc.end(), by_slot);                      // slots 0..n-1 in order: the cross K/V of all windows is one launch
    std::sort(dec.begin(), dec.end(), by_slot);                      // and the row order of a pass does not depend on thread timing
    if (!enc.empty()) {
        const int64_t t0 = time_us();
        bool same_ctx = true;
        for (Req * q : enc) same_ctx &= (q->n_ctx == enc[0]->n_ctx);
        bool ok = true;
        if (scripted) {
            // test hook: nothing to encode
        } else if (same_ctx) {
            std::vector<EncSrc> srcs;
            for (Req * q : enc) srcs.push_back({ q->st->fe.mel.p, q->st->fe.n_len, q->st->fe.n_mel, q->seek, q->st->slot });
            ok = eng.encode(srcs.data(), (int) srcs.size(), enc[0]->n_ctx);
        } else {
            for (Req * q : enc) { const EncSrc s = { q->st->fe.mel.p, q->st->fe.n_len, q->st->fe.n_mel, q->seek, q->st->slot }; ok &= eng.encode(&s, 1, q->n_ctx); }
        }
        const int64_t dt = (time_us() - t0) / (int64_t) enc.size();
        for (Req * q : enc) { q->ok = ok; q->dt_us = dt; }
    }
    if (!dec.empty()) {
        const int64_t t0 = time_us();
        const int n_vocab = dec[0]->ctx->model.hp.n_vocab;
        std::vector<PreparedDecode> preps(dec.size());
        bool ok = true; int total = 0, ld = 1;
        for (size_t i = 0; i < dec.size(); ++i) {
            Req * q = dec[i];
            if (q->x_cells) {                                          // explicit cells (ggml-backend plugin): no bookkeeping on this side
                PreparedDecode & P = preps[i];
                P.ld = q->x_ld; P.rows.resize(q->n); P.cells.resize(q->n); P.nkv.assign(q->x_nkv, q->x_nkv + q->n); P.idx.assign((size_t) q->n * q->x_ld, 0);
                for (int j = 0; j < q->n; ++j) {
                    P.rows[j] = { q->tokens[j], q->pos[j], 0, q->st->slot, q->want[j] != 0 };
                    P.cells[j] = q->st->cell_off + q->x_cells[j];
                    for (int c = 0; c < q->x_nkv[j]; ++c) P.idx[(size_t) j * q->x_ld + c] = q->st->cell_off + q->x_idx[(size_t) j * q->x_ld + c];
                }
            } else
            ok &= prepare_decode(*q->st, q->tokens, q->pos, q->seq, q->want, q->n, preps[i]);
            total += q->n; ld = std::max(ld, preps[i].ld);
        }
        // the on-device filter + pick serves the pass only if EVERY request asked for it with the same configuration (a member that fell
        // back to temperature > 0 samples on the host and needs full logits, so the whole pass returns logits then).  A DTW pass samples
        // nothing: the one row it wants needs only the raw summary (max, sum, no-speech logit) of the sampler output, which does not depend
        // on the filter configuration, so it rides on whatever configuration the other requests share (its own, when it offers one and
        // only DTW passes are in the batch).
        const Req * cfg0 = nullptr;
        for (Req * q : dec) if (!q->dtw_n_ctx) { cfg0 = q; break; }
        if (!cfg0) for (Req * q : dec) if (q->samp) { cfg0 = q; break; }
        bool all_samp = cfg0 != nullptr && cfg0->samp != nullptr;
        auto same_cfg = [](const SampCfg & a, const SampCfg & b) {            // field by field: the struct has padding bytes
            return a.token_eot == b.token_eot && a.token_beg == b.token_beg && a.token_nosp == b.token_nosp && a.space_id == b.space_id &&
                   a.suppress_blank == b.suppress_blank && a.no_timestamps == b.no_timestamps && a.max_initial_tid == b.max_initial_tid;
        };
        for (Req * q : dec) if (!q->dtw_n_ctx) all_samp = all_samp && q->samp != nullptr && q->samp->mask_key == cfg0->samp->mask_key && same_cfg(q->samp->cfg, cfg0->samp->cfg);
        // DTW requests: capture indices [cap0, cap0 + n) of the engine's capture buffer, one region per request
        std::vector<int> dtw_req, dtw_path; std::vector<Req *> dtw_of;
        int n_cap = 0;
        for (Req * q : dec) if (q->dtw_n_ctx > 0) {
            dtw_req.insert(dtw_req.end(), { n_cap, q->st->slot, q->n, q->dtw_n_ctx });
            dtw_path.insert(dtw_path.end(), { q->dtw_n_frames / 2, q->dtw_sot_len });
            dtw_of.push_back(q); n_cap += q->n;
        }
        if (scripted) {                                               // test hook: KV bookkeeping done above, logits are the callback's business
            for (size_t i = 0; i < dec.size(); ++i) {
                Req * q = dec[i];
                if (ok) scripted_attended(*q->st, preps[i], q->n);
                q->st->samp_out.clear(); q->st->logits.assign((size_t) q->n * n_vocab, 0.0f);
            }
        } else {
        if (ok && all_samp) ok = eng.set_samp_mask(cfg0->samp->mask_key, *cfg0->samp->mask_bits);
        if (ok && n_cap > 0) ok = eng.dtw_reserve(n_cap);
        // run-ahead: greedy rows of one decoder, sampled on the device, on the persistent kernel; never while per-launch profiling or
        // tracing is on (those runs attribute every launch to its pass), never with DTW (its passes capture queries and sample nothing)
        int stride = 1;                                                // entries per row of the sampler output: the widest request decides
        auto own_stride = [](const Req * q) { return (q->samp && q->samp->draws) ? q->samp->stride : 1; };
        if (all_samp) for (Req * q : dec) stride = std::max(stride, own_stride(q));
        const bool ahead = ok && run_ahead && all_samp && stride == 1 && n_cap == 0 && dtw_heads.empty() && eng.use_mk && !prof_enabled() && !eng.mk_trace.p;
        // requests the queued run-ahead pass already computed: acc[i] = its row, -1: run in an ordinary pass
        std::vector<int> acc(dec.size(), -1);
        int n_acc = 0;
        if (ahead && spec_pass >= 0 && spec_mask_key == cfg0->samp->mask_key && same_cfg(spec_cfg, cfg0->samp->cfg)) {
            for (size_t i = 0; i < dec.size(); ++i) {
                const Req * q = dec[i]; const PreparedDecode & P = preps[i];
                if (q->n != 1 || q->x_cells || q->dtw_n_ctx || !q->want[0] || q->samp->draws) continue;
                for (size_t k = 0; k < spec_rows.size(); ++k) {
                    const SpecRow & r = spec_rows[k];
                    if (r.st != q->st) continue;
                    if (r.token == q->tokens[0] && r.pos == q->pos[0] && r.seq == q->seq[0] && r.slot == q->st->slot && r.cell == P.cells[0] &&
                        r.n_ctx == eng.slot_n_ctx(r.slot) && (r.rowinfo[0] & 0xff) == (q->samp->rowinfo[0] & 0xff) && r.rowinfo[1] == q->samp->rowinfo[1] &&
                        (int) r.idx.size() == P.nkv[0] && std::equal(r.idx.begin(), r.idx.end(), P.idx.begin())) { acc[i] = (int) k; ++n_acc; }
                    break;
                }
            }
        }
        if (ok) {
            std::vector<int> cap0(dec.size(), -1);
            for (size_t i = 0, c = 0; i < dec.size(); ++i) if (dec[i]->dtw_n_ctx > 0) { cap0[i] = dtw_req[4 * c]; ++c; }
            for (Req * q : dec) { if (all_samp) { q->st->samp_stride = own_stride(q); q->st->samp_out.assign((size_t) q->n * q->st->samp_stride, SampOut()); } else { q->st->samp_out.clear(); q->st->logits.resize((size_t) q->n * n_vocab); } }
            // one decode call per encoded context length (a pass attends to one number of cross keys), requests in slot order within each
            std::vector<std::vector<size_t>> groups; std::vector<int> group_ctx;
            for (size_t i = 0; i < dec.size(); ++i) {
                if (acc[i] >= 0) continue;
                const int T = eng.slot_n_ctx(dec[i]->st->slot);
                size_t g = 0;
                while (g < groups.size() && group_ctx[g] != T) ++g;
                if (g == groups.size()) { groups.emplace_back(); group_ctx.push_back(T); }
                groups[g].push_back(i);
            }
            // with run-ahead, a batch whose ordinary rows fit one pass only enqueues it here: the next run-ahead pass goes in behind it
            int o_pass = -1; std::vector<std::pair<Req *, int>> o_origin;
            for (const std::vector<size_t> & grp : groups) {
                if (!ok) break;
                int gtotal = 0; for (size_t i : grp) gtotal += dec[i]->n;
                std::vector<DecToken> rows; std::vector<int> cells, nkv, idx((size_t) gtotal * ld, 0); std::vector<float *> outs;
                std::vector<int> rowinfo, capidx; std::vector<SampOut> souts((size_t) gtotal * stride); std::vector<std::pair<Req *, int>> origin;
                std::vector<double> draws; if (stride > 1) draws.assign((size_t) gtotal * stride, 0.0);
                rows.reserve(gtotal);
                // interleave: row k of every request first, so that single-token steps of all members share one pass (<= Engine::max_rows rows)
                // and multi-token prompts advance in lock-step (causal order inside each member is preserved)
                int maxn = 0; for (size_t i : grp) maxn = std::max(maxn, dec[i]->n);
                for (int k = 0; k < maxn; ++k) {
                    for (size_t i : grp) {
                        Req * q = dec[i]; if (k >= q->n) continue;
                        const PreparedDecode & P = preps[i];
                        const size_t r = rows.size();
                        rows.push_back(P.rows[k]); cells.push_back(P.cells[k]); nkv.push_back(P.nkv[k]);
                        memcpy(idx.data() + r * ld, P.idx.data() + (size_t) k * P.ld, (size_t) P.nkv[k] * sizeof(int));
                        outs.push_back(all_samp ? nullptr : q->st->logits.data() + (size_t) k * n_vocab);
                        capidx.push_back(cap0[i] >= 0 ? cap0[i] + k : -1);
                        if (all_samp && q->dtw_n_ctx > 0) {               // DTW row: greedy pick without draws, only its raw summary is read
                            rowinfo.push_back(0); rowinfo.push_back(0);
                        } else if (all_samp) {
                            const bool has_draws = q->samp->draws != nullptr;
                            rowinfo.push_back(has_draws ? q->samp->rowinfo[2*k] : (q->samp->rowinfo[2*k] & 0xff)); rowinfo.push_back(q->samp->rowinfo[2*k + 1]);
                            if (has_draws) memcpy(draws.data() + r * stride, q->samp->draws + (size_t) k * q->samp->stride, (size_t) q->samp->stride * sizeof(double));
                        }
                        origin.emplace_back(q, k);
                    }
                }
                if (ahead && groups.size() == 1 && gtotal <= eng.max_rows) {
                    ok = eng.pass_enqueue(rows.data(), gtotal, cells.data(), idx.data(), ld, nkv.data(), &cfg0->samp->cfg, rowinfo.data(), nullptr, 1,
                                          nullptr, nullptr, &o_pass);
                    o_origin.swap(origin);
                } else if (all_samp) {
                    ok = eng.decode(rows.data(), gtotal, cells.data(), idx.data(), ld, nkv.data(), nullptr, &cfg0->samp->cfg, rowinfo.data(), souts.data(),
                                    stride > 1 ? draws.data() : nullptr, stride, n_cap > 0 ? capidx.data() : nullptr);
                    for (int r = 0; r < gtotal; ++r) {
                        Req * q = origin[r].first; const int own = own_stride(q);
                        for (int j = 0; j < own; ++j) q->st->samp_out[(size_t) origin[r].second * own + j] = souts[(size_t) r * stride + j];
                    }
                } else {
                    ok = eng.decode(rows.data(), gtotal, cells.data(), idx.data(), ld, nkv.data(), outs.data(), nullptr, nullptr, nullptr, nullptr, 1,
                                    n_cap > 0 ? capidx.data() : nullptr);
                }
            }
            // the next run-ahead pass: the single-token step after the last row of every request whose member may continue, its token
            // taken on the device from this batch's sampler output (the accepted run-ahead rows, or the ordinary pass enqueued above)
            // A mispredicted row costs a whole ordinary pass behind the run-ahead pass (two passes for the step instead of one), a
            // taken pass saves one host turnaround.  Where predictions fail often (timestamps sampled every few tokens) the pool runs
            // lock-step and tries again every 256th batch: spec_miss is the running share of run-ahead batches with a mispredicted row.
            if (spec_pass >= 0) {
                bool miss = false;
                for (size_t i = 0; i < dec.size() && !miss; ++i)
                    if (acc[i] < 0 && dec[i]->n == 1)
                        for (const SpecRow & r : spec_rows) miss |= r.st == dec[i]->st;
                spec_miss += ((miss ? 1.0f : 0.0f) - spec_miss) / 8.0f;
            }
            const bool try_ahead = spec_miss < 0.25f || ++spec_idle >= 256;
            int next_pass = -1; std::vector<SpecRow> next;
            if (ok && ahead && try_ahead) {
                auto predict = [&](Req * q, int src_pass, int src_row) {
                    const int k = q->n - 1;
                    if (!q->samp->next_step || q->x_cells || !q->want[k] || q->seq[k] != 0) return;
                    KvCells kv = q->st->kv;                               // what find_slot and the KQ-mask rule will give the real request
                    const int pos = q->pos[k] + 1, seq = 0, tok = 0; const int8_t want = 1;
                    PreparedDecode P;
                    if (pos >= q->ctx->model.hp.n_text_ctx || !prepare_rows(kv, *q->st, &tok, &pos, &seq, &want, 1, P)) return;
                    SpecRow r{ q->st, -1, pos, seq, q->st->slot, P.cells[0], eng.slot_n_ctx(q->st->slot), { q->samp->next_rowinfo[0], q->samp->next_rowinfo[1] },
                               std::vector<int>(P.idx.begin(), P.idx.begin() + P.nkv[0]), src_pass, src_row };
                    next.push_back(std::move(r));
                };
                for (size_t i = 0; i < dec.size(); ++i) if (acc[i] >= 0) predict(dec[i], spec_pass, acc[i]);
                for (size_t r = 0; r < o_origin.size(); ++r) if (o_origin[r].second == o_origin[r].first->n - 1) predict(o_origin[r].first, o_pass, (int) r);
                bool one_ctx = true;
                for (const SpecRow & r : next) one_ctx &= r.n_ctx == next[0].n_ctx;
                if (!next.empty() && one_ctx && (int) next.size() <= eng.max_rows) {
                    std::sort(next.begin(), next.end(), [](const SpecRow & a, const SpecRow & b) { return a.slot < b.slot; });   // row order of a pass
                    const int nn = (int) next.size();
                    int nld = 1; for (const SpecRow & r : next) nld = std::max(nld, (int) r.idx.size());
                    std::vector<DecToken> rows; std::vector<int> cells, nkv, idx((size_t) nn * nld, 0), rowinfo, src;
                    for (int j = 0; j < nn; ++j) {
                        const SpecRow & r = next[j];
                        rows.push_back({ 0, r.pos, r.seq, r.slot, true }); cells.push_back(r.cell); nkv.push_back((int) r.idx.size());
                        std::copy(r.idx.begin(), r.idx.end(), idx.begin() + (size_t) j * nld);
                        rowinfo.push_back(r.rowinfo[0] & 0xff); rowinfo.push_back(r.rowinfo[1]);
                        src.push_back((int) (eng.dsamp_of(r.src_pass) - eng.dsamp.p) + r.src_row);   // stride-1 passes: entry 0 of row src_row
                    }
                    ok = eng.pass_enqueue(rows.data(), nn, cells.data(), idx.data(), nld, nkv.data(), &cfg0->samp->cfg, rowinfo.data(), nullptr, 1,
                                          nullptr, src.data(), &next_pass);
                    if (ok) counter_add(12, nn);
                    spec_idle = 0;
                } else {
                    next.clear();
                }
            }
            // results: the accepted rows of the previous run-ahead pass, then the ordinary pass; each fills in the tokens it fed forward
            auto harvest = [&](int pass) {
                if (pass < 0) return;
                if (!eng.pass_wait(pass)) { ok = false; return; }
                for (SpecRow & r : next) if (r.src_pass == pass) r.token = eng.pslot[pass].hsamp[r.src_row].id;
            };
            if (spec_pass >= 0) {
                harvest(spec_pass);
                if (ok) for (size_t i = 0; i < dec.size(); ++i) if (acc[i] >= 0) dec[i]->st->samp_out[0] = eng.pslot[spec_pass].hsamp[acc[i]];
                counter_add(13, n_acc);
            }
            harvest(o_pass);
            if (ok) for (size_t r = 0; r < o_origin.size(); ++r) o_origin[r].first->st->samp_out[(size_t) o_origin[r].second] = eng.pslot[o_pass].hsamp[r];
            spec_pass = -1; spec_rows.clear();
            if (ok && next_pass >= 0) { spec_pass = next_pass; spec_rows.swap(next); spec_mask_key = cfg0->samp->mask_key; spec_cfg = cfg0->samp->cfg; }
            // alignment weights and warping paths of every DTW request of the batch, one launch per kernel (dtw_assign runs on each state's
            // own thread)
            if (ok && n_cap > 0) {
                std::vector<std::vector<float> *> outw; std::vector<std::vector<int32_t> *> outt, outj;
                for (Req * q : dtw_of) { outw.push_back(&q->st->dtw_qk_last); outt.push_back(&q->st->dtw_tok); outj.push_back(&q->st->dtw_time); }
                ok = eng.dtw_weights(dtw_req, dtw_path, outw, outt, outj);
                for (Req * q : dtw_of) { whisper_state & s = *q->st; s.dtw_last_shape[0] = q->n; s.dtw_last_shape[1] = q->dtw_n_ctx; s.dtw_last_shape[2] = eng.dtw_n_heads; }
            }
        }
        if (!ok) spec_drop();
        }
        const int64_t dt = (time_us() - t0) / (int64_t) dec.size();
        for (Req * q : dec) { q->ok = ok; q->dt_us = dt; }
    }
}

static std::vector<whisper_token> tokenize(const Vocab & vocab, const std::string & text) {   // whisper.cpp:3284-3332
    std::vector<std::string> words;
    {
        std::string str = text;
        static const std::regex re(R"('s|'t|'re|'ve|'m|'ll|'d| ?[[:alpha:]]+| ?[[:digit:]]+| ?[^\s[:alpha:][:digit:]]+|\s+(?!\S)|\s+)");
        std::smatch mt;
        while (std::regex_search(str, mt, re)) {
            for (auto x : mt) words.push_back(x);
            str = mt.suffix();
        }
    }
    std::vector<whisper_token> out;
    for (const auto & word : words) {
        if (word.empty()) continue;
        int i = 0; const int n = (int) word.size();
        while (i < n) {
            int j = n; bool found = false;
            while (j > i) {
                auto it = vocab.token_to_id.find(word.substr(i, j - i));
                if (it != vocab.token_to_id.end()) { out.push_back(it->second); i = j; found = true; break; }
                --j;
            }
            if (!found) { logf(LOG_ERROR, "unknown token\n"); ++i; }
        }
    }
    return out;
}

} // namespace wb

// =====================================================================================================================
extern "C" {

WB_EXPORT const char * whisper_version(void) { return "1.9.3-b200"; }

WB_EXPORT struct whisper_context_params whisper_context_default_params(void) {       // whisper.cpp:3618-3634
    struct whisper_context_params p;
    memset(&p, 0, sizeof(p));
    p.use_gpu = true; p.flash_attn = true; p.gpu_device = 0;
    p.dtw_token_timestamps = false; p.dtw_aheads_preset = WHISPER_AHEADS_NONE; p.dtw_n_top = -1;
    p.dtw_aheads.n_heads = 0; p.dtw_aheads.heads = nullptr; p.dtw_mem_size = 1024 * 1024 * 128;
    return p;
}
WB_EXPORT struct whisper_context_params * whisper_context_default_params_by_ref(void) {
    auto * p = new whisper_context_params(); *p = whisper_context_default_params(); return p;
}
WB_EXPORT void whisper_free_context_params(struct whisper_context_params * p) { delete p; }
WB_EXPORT void whisper_free_params(struct whisper_full_params * p) { delete p; }

// ---------------------------------------------------------------------------------------------------- init / free
WB_EXPORT struct whisper_context * whisper_init_with_params_no_state(struct whisper_model_loader * loader, struct whisper_context_params params) {
    if (!loader) return nullptr;
    whisper_context * ctx = nullptr;
    bool ok = false;
    try {
        if (!params.use_gpu) {
            set_error("this engine runs on the GPU only: whisper_context_params.use_gpu=false is not supported (no CPU fallback)");
        } else {
            int ndev = 0;
            if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
                set_error("no CUDA device available: libwhisper_b200 has no CPU fallback");
            } else if (params.gpu_device < 0 || params.gpu_device >= ndev) {
                set_error("gpu_device %d out of range (%d devices)", params.gpu_device, ndev);
            } else {
                if (params.flash_attn && params.dtw_token_timestamps) {
                    logf(LOG_WARN, "%s: dtw_token_timestamps is not supported with flash_attn - disabling\n", __func__);
                    params.dtw_token_timestamps = false;
                }
                ctx = new whisper_context();
                ctx->params = params;
                ctx->t_start_us = time_us();
                ok = model_load(loader, ctx->model, ctx->vocab, params.gpu_device);
                ctx->t_load_us = ctx->model.t_load_us;
            }
        }
    } catch (const std::exception & e) {
        set_error("exception during model load: %s", e.what());
    } catch (...) {
        set_error("unknown exception during model load");
    }
    loader->close(loader->context);                                                  // always, whisper.cpp:3750,3756
    if (!ok) { logf(LOG_ERROR, "%s: failed to load model\n", __func__); delete ctx; return nullptr; }
    return ctx;
}

WB_EXPORT struct whisper_context * whisper_init_from_file_with_params_no_state(const char * path_model, struct whisper_context_params params) {
    if (!path_model) return nullptr;
    logf(LOG_INFO, "%s: loading model from '%s'\n", __func__, path_model);
    std::ifstream fin(path_model, std::ios::binary);
    if (!fin) { set_error("failed to open '%s'", path_model); return nullptr; }
    whisper_model_loader loader = {};
    loader.context = &fin;
    loader.read  = [](void * c, void * out, size_t n) -> size_t { auto * f = (std::ifstream *) c; f->read((char *) out, (std::streamsize) n); return (size_t) f->gcount(); };
    loader.eof   = [](void * c) -> bool { return ((std::ifstream *) c)->eof(); };
    loader.close = [](void * c) { ((std::ifstream *) c)->close(); };
    whisper_context * ctx = whisper_init_with_params_no_state(&loader, params);
    if (ctx) ctx->path_model = path_model;
    if (ctx && !ctx->params.dtw_token_timestamps) {
        // WB200_DEVICES = "all" | "0,1,5": one more copy of the weights per listed GPU (the context's own device is always first)
        if (const char * e = getenv("WB200_DEVICES")) {
            int ndev = 0; cudaGetDeviceCount(&ndev);
            std::vector<int> devs;
            if (!strcmp(e, "all")) { for (int d = 0; d < ndev; ++d) devs.push_back(d); }
            else { for (const char * q = e; *q; ) { char * end = nullptr; const long d = strtol(q, &end, 10); if (end == q) break; if (d >= 0 && d < ndev) devs.push_back((int) d); q = (*end == ',') ? end + 1 : end; } }
            for (int d : devs) {
                if (d == params.gpu_device) continue;
                std::ifstream f2(path_model, std::ios::binary);
                if (!f2) break;
                whisper_model_loader l2 = {};
                l2.context = &f2;
                l2.read  = [](void * c, void * out, size_t n) -> size_t { auto * f = (std::ifstream *) c; f->read((char *) out, (std::streamsize) n); return (size_t) f->gcount(); };
                l2.eof   = [](void * c) -> bool { return ((std::ifstream *) c)->eof(); };
                l2.close = [](void * c) { ((std::ifstream *) c)->close(); };
                std::unique_ptr<Replica> r(new Replica());
                Vocab vtmp;
                if (!model_load(&l2, r->model, vtmp, d)) { logf(LOG_WARN, "%s: no replica on GPU %d: %s\n", __func__, d, last_error()); continue; }
                logf(LOG_INFO, "%s: replica of the weights on GPU %d\n", __func__, d);
                ctx->replicas.push_back(std::move(r));
            }
            cudaSetDevice(params.gpu_device);
        }
    }
    return ctx;
}

WB_EXPORT struct whisper_context * whisper_init_from_buffer_with_params_no_state(void * buffer, size_t buffer_size, struct whisper_context_params params) {
    struct Buf { const uint8_t * p; size_t size, off; } b = { (const uint8_t *) buffer, buffer_size, 0 };
    logf(LOG_INFO, "%s: loading model from buffer\n", __func__);
    whisper_model_loader loader = {};
    loader.context = &b;
    loader.read  = [](void * c, void * out, size_t n) -> size_t { auto * q = (Buf *) c; size_t k = std::min(n, q->size - q->off); memcpy(out, q->p + q->off, k); q->off += k; return k; };
    loader.eof   = [](void * c) -> bool { auto * q = (Buf *) c; return q->off >= q->size; };
    loader.close = [](void *) {};
    return whisper_init_with_params_no_state(&loader, params);
}

WB_EXPORT struct whisper_state * whisper_init_state(struct whisper_context * ctx) {  // whisper.cpp:3386-3557
    if (!ctx) return nullptr;
    whisper_state * st = nullptr;
    if (ctx->params.dtw_token_timestamps && !ctx->scripted && ctx->dtw_heads.empty()) {     // aheads_masks_init, src/whisper.cpp:3442-3450: a bad selection fails the state
        if (!dtw_resolve_heads(ctx->params, ctx->model.hp.n_text_layer, ctx->model.hp.n_text_head, ctx->dtw_heads)) {
            logf(LOG_ERROR, "%s: aheads_masks_init() failed for alignment heads masks: %s\n", __func__, last_error());
            return nullptr;
        }
        logf(LOG_INFO, "%s: alignment heads masks: %d heads\n", __func__, (int) ctx->dtw_heads.size());
    }
    try {
        // every state is a slot of a device pool of the context (created with the first state); see wb_state.h.  With replicas on
        // several GPUs the new state goes to the GPU that holds the fewest states (ties: the context's own device first).
        Group * pool = nullptr; const Model * model = &ctx->model;
        {
            std::lock_guard<std::mutex> lk(ctx->replicas_mu);
            if (!ctx->pool) { ctx->pool.reset(new Group()); ctx->pool->model = &ctx->model; ctx->pool->scripted = ctx->scripted; ctx->pool->dtw_heads = ctx->dtw_heads; ctx->pool->run_ahead = ctx->run_ahead; }
            pool = ctx->pool.get();
            for (auto & r : ctx->replicas) {
                if (!r->pool) { r->pool.reset(new Group()); r->pool->model = &r->model; r->pool->run_ahead = ctx->run_ahead; }
                if (r->pool->n_registered < pool->n_registered) { pool = r->pool.get(); model = &r->model; }
            }
        }
        std::unique_ptr<FrontEnd> fe = pool->take_fe();
        st = fe ? new whisper_state(std::move(fe)) : new whisper_state();
        st->scripted = ctx->scripted;
        if (!ctx->scripted && !st->fe.st && !st->fe.init(model)) { delete st; return nullptr; }
        if (!pool->attach(st)) { logf(LOG_ERROR, "%s: %s\n", __func__, last_error()); delete st; return nullptr; }
        st->decoders[0].rng = std::mt19937(0);
    } catch (...) { set_error("whisper_init_state: allocation failed"); delete st; return nullptr; }
    return st;
}

#define WB_INIT_WITH_STATE(call) \
    whisper_context * ctx = call; if (!ctx) return nullptr; \
    ctx->state = whisper_init_state(ctx); if (!ctx->state) { whisper_free(ctx); return nullptr; } return ctx;

WB_EXPORT void whisper_free_state(struct whisper_state * st) {
    if (!st) return;
    if (st->group) st->group->detach(st);          // the slot and the front end go back to the context's pool
    delete st;
}
WB_EXPORT void whisper_free(struct whisper_context * ctx) {
    if (!ctx) return;
    whisper_free_state(ctx->state);
    delete ctx;
}
} // extern "C"
whisper_context::~whisper_context() {}
extern "C" {

WB_EXPORT struct whisper_context * whisper_init_from_file_with_params(const char * path, struct whisper_context_params p)            { WB_INIT_WITH_STATE(whisper_init_from_file_with_params_no_state(path, p)) }
WB_EXPORT struct whisper_context * whisper_init_from_buffer_with_params(void * b, size_t n, struct whisper_context_params p)           { WB_INIT_WITH_STATE(whisper_init_from_buffer_with_params_no_state(b, n, p)) }
WB_EXPORT struct whisper_context * whisper_init_with_params(struct whisper_model_loader * l, struct whisper_context_params p)          { WB_INIT_WITH_STATE(whisper_init_with_params_no_state(l, p)) }
WB_EXPORT struct whisper_context * whisper_init_from_file(const char * path)                      { return whisper_init_from_file_with_params(path, whisper_context_default_params()); }
WB_EXPORT struct whisper_context * whisper_init_from_buffer(void * b, size_t n)                   { return whisper_init_from_buffer_with_params(b, n, whisper_context_default_params()); }
WB_EXPORT struct whisper_context * whisper_init(struct whisper_model_loader * l)                  { return whisper_init_with_params(l, whisper_context_default_params()); }
WB_EXPORT struct whisper_context * whisper_init_from_file_no_state(const char * path)             { return whisper_init_from_file_with_params_no_state(path, whisper_context_default_params()); }
WB_EXPORT struct whisper_context * whisper_init_from_buffer_no_state(void * b, size_t n)          { return whisper_init_from_buffer_with_params_no_state(b, n, whisper_context_default_params()); }
WB_EXPORT struct whisper_context * whisper_init_no_state(struct whisper_model_loader * l)         { return whisper_init_with_params_no_state(l, whisper_context_default_params()); }

WB_EXPORT int whisper_ctx_init_openvino_encoder_with_state(struct whisper_context *, struct whisper_state *, const char *, const char *, const char *) { return 1; }
WB_EXPORT int whisper_ctx_init_openvino_encoder(struct whisper_context *, const char *, const char *, const char *) { return 1; }

// ---------------------------------------------------------------------------------------------------- low-level pipeline
WB_EXPORT int whisper_pcm_to_mel_with_state(struct whisper_context * ctx, struct whisper_state * st, const float * samples, int n_samples, int) {
    if (!ctx || !st || n_samples < 0) return -1;     // samples == NULL is legal after wb200_pcm_upload (device-resident input)
    const int64_t t0 = time_us();
    if (st->scripted) {                                                      // test hook: only the frame counts of whisper.cpp:3202-3220
        st->fe.n_mel = ctx->model.hp.n_mels; st->fe.n_len = (n_samples + 480000) / 160; st->fe.n_len_org = 1 + (n_samples + 200 - 400) / 160;
        return 0;
    }
    if (!st->fe.pcm_to_mel(samples, n_samples, wb::tls_pcm_is_device())) { logf(LOG_ERROR, "%s: failed to compute mel spectrogram\n", __func__); return -1; }
    st->t_mel_us += time_us() - t0;
    return 0;
}
WB_EXPORT int whisper_pcm_to_mel(struct whisper_context * ctx, const float * samples, int n_samples, int n_threads) {
    return ctx ? whisper_pcm_to_mel_with_state(ctx, ctx->state, samples, n_samples, n_threads) : -1;
}
WB_EXPORT int whisper_set_mel_with_state(struct whisper_context * ctx, struct whisper_state * st, const float * data, int n_len, int n_mel) {
    if (!ctx || !st) return -1;
    if (n_mel != ctx->model.n_filt_mel) { logf(LOG_ERROR, "%s: invalid number of mel bands: %d (expected %d)\n", __func__, n_mel, ctx->model.n_filt_mel); return -1; }
    return st->fe.set_mel(data, n_len, n_mel) ? 0 : -1;
}
WB_EXPORT int whisper_set_mel(struct whisper_context * ctx, const float * data, int n_len, int n_mel) {
    return ctx ? whisper_set_mel_with_state(ctx, ctx->state, data, n_len, n_mel) : -1;
}
WB_EXPORT int whisper_encode_with_state(struct whisper_context * ctx, struct whisper_state * st, int offset, int) {
    if (!ctx || !st) return -1;
    GroupCall gc(st);
    if (!encode_window(*ctx, *st, offset)) { logf(LOG_ERROR, "%s: failed to eval\n", __func__); return -1; }
    return 0;
}
WB_EXPORT int whisper_encode(struct whisper_context * ctx, int offset, int n_threads) { return ctx ? whisper_encode_with_state(ctx, ctx->state, offset, n_threads) : -1; }

WB_EXPORT int whisper_decode_with_state(struct whisper_context * ctx, struct whisper_state * st, const whisper_token * tokens, int n_tokens, int n_past, int) {
    if (!ctx || !st || !tokens || n_tokens <= 0) return 1;
    std::vector<int> pos(n_tokens), seq(n_tokens, 0); std::vector<int8_t> want(n_tokens, 0);
    for (int i = 0; i < n_tokens; ++i) pos[i] = n_past + i;
    want[n_tokens - 1] = 1;                                                          // whisper_batch_prep_legacy, whisper.cpp:511-523
    GroupCall gc(st);
    st->kv.seq_rm(0, n_past, -1);
    if (!decode_batch(*ctx, *st, tokens, pos.data(), seq.data(), want.data(), n_tokens)) { logf(LOG_ERROR, "%s: failed to eval\n", __func__); return 1; }
    return 0;
}
// Decode with the self-KV cells spelled out by the caller: row j is written to cell cells[j] of the state's range and attends to
// idx[j*ld .. j*ld + nkv[j]) (whisper_build_graph_decoder's kv_head and KQ_mask, src/whisper.cpp:2580-2599, 2928-2938).  Entry point of the
// ggml-backend plugin (plugin/ggml_b200_backend.cpp), whose host keeps the whisper_kv_cache bookkeeping itself.  logits: [n_tokens][n_vocab].
WB_EXPORT int wb200_decode_explicit(struct whisper_context * ctx, struct whisper_state * st, const whisper_token * tokens, const int * pos, int n_tokens,
                                    const int * cells, const int * idx, int ld, const int * nkv, int n_cells_needed, float * logits) {
    if (!ctx || !st || !tokens || !pos || !cells || !idx || !nkv || n_tokens <= 0 || !st->group) return 1;
    GroupCall gc(st);
    if ((int) st->kv.size < n_cells_needed) {                                  // the host's kv_self is larger than this state's cell range so far
        if (!st->group->ensure_cells(st, n_cells_needed)) { logf(LOG_ERROR, "%s: KV cache allocation failed: %s\n", __func__, last_error()); return 1; }
    }
    std::vector<int8_t> want((size_t) n_tokens, 1);
    Group::Req r; r.kind = 1; r.ctx = ctx; r.st = st; r.tokens = tokens; r.pos = pos; r.seq = nullptr; r.want = want.data(); r.n = n_tokens;
    r.x_cells = cells; r.x_idx = idx; r.x_nkv = nkv; r.x_ld = ld;
    if (!st->group->submit(r)) { logf(LOG_ERROR, "%s: failed to eval: %s\n", __func__, last_error()); return 1; }
    if (logits) memcpy(logits, st->logits.data(), (size_t) n_tokens * ctx->model.hp.n_vocab * sizeof(float));
    return 0;
}
WB_EXPORT int whisper_decode(struct whisper_context * ctx, const whisper_token * tokens, int n_tokens, int n_past, int n_threads) {
    if (!ctx || !ctx->state) { logf(LOG_ERROR, "%s: ERROR state was not loaded.\n", __func__); return -1; }
    return whisper_decode_with_state(ctx, ctx->state, tokens, n_tokens, n_past, n_threads);
}
WB_EXPORT float * whisper_get_logits(struct whisper_context * ctx) { return ctx->state->logits.data(); }
WB_EXPORT float * whisper_get_logits_from_state(struct whisper_state * st) { return st->logits.data(); }

// ---------------------------------------------------------------------------------------------------- tokenizer / languages
WB_EXPORT int whisper_tokenize(struct whisper_context * ctx, const char * text, whisper_token * tokens, int n_max_tokens) {
    const auto res = tokenize(ctx->vocab, text);
    if (n_max_tokens < (int) res.size()) { logf(LOG_ERROR, "%s: too many resulting tokens: %d (max %d)\n", __func__, (int) res.size(), n_max_tokens); return -(int) res.size(); }
    for (size_t i = 0; i < res.size(); ++i) tokens[i] = res[i];
    return (int) res.size();
}
WB_EXPORT int whisper_token_count(struct whisper_context * ctx, const char * text) { return -whisper_tokenize(ctx, text, nullptr, 0); }
WB_EXPORT int whisper_lang_max_id(void) { return 99; }
WB_EXPORT int whisper_lang_id(const char * lang) {
    if (lang) {
        for (int i = 0; i < 100; ++i) if (!strcmp(lang, g_lang_codes[i])) return i;
        for (int i = 0; i < 100; ++i) if (!strcmp(lang, g_lang_names[i])) return i;
    }
    logf(LOG_ERROR, "%s: unknown language '%s'\n", __func__, lang ? lang : "(null)");
    return -1;
}
WB_EXPORT const char * whisper_lang_str(int id)      { if (id >= 0 && id < 100) return g_lang_codes[id]; logf(LOG_ERROR, "%s: unknown language id %d\n", __func__, id); return nullptr; }
WB_EXPORT const char * whisper_lang_str_full(int id) { if (id >= 0 && id < 100) return g_lang_names[id]; logf(LOG_ERROR, "%s: unknown language id %d\n", __func__, id); return nullptr; }

WB_EXPORT int whisper_lang_auto_detect_with_state(struct whisper_context * ctx, struct whisper_state * st, int offset_ms, int n_threads, float * lang_probs) {
    const int seek = offset_ms / 10;                                                 // whisper.cpp:4047-4120
    if (seek < 0) { logf(LOG_ERROR, "%s: offset %dms is before the start of the audio\n", __func__, offset_ms); return -1; }
    if (seek >= st->fe.n_len_org) { logf(LOG_ERROR, "%s: offset %dms is past the end of the audio (%dms)\n", __func__, offset_ms, st->fe.n_len_org * 10); return -2; }
    if (whisper_encode_with_state(ctx, st, seek, n_threads) != 0) return -6;
    const whisper_token sot = ctx->vocab.token_sot;
    if (whisper_decode_with_state(ctx, st, &sot, 1, 0, n_threads) != 0) return -7;
    std::vector<std::pair<double, int>> li;
    for (int id = 0; id < 100; ++id) {
        const int tok = sot + 1 + id;
        if (tok >= ctx->vocab.n_vocab) continue;
        li.emplace_back(st->logits[tok], id);
    }
    if (li.empty()) return -7;
    std::sort(li.begin(), li.end(), [](const std::pair<double, int> & a, const std::pair<double, int> & b) { return a.first > b.first; });
    const double mx = li[0].first; double sum = 0.0;
    for (auto & kv : li) { kv.first = exp(kv.first - mx); sum += kv.first; }
    for (auto & kv : li) kv.first /= sum;
    if (lang_probs) for (auto & kv : li) lang_probs[kv.second] = (float) kv.first;
    return li[0].second;
}
WB_EXPORT int whisper_lang_auto_detect(struct whisper_context * ctx, int offset_ms, int n_threads, float * lang_probs) {
    return whisper_lang_auto_detect_with_state(ctx, ctx->state, offset_ms, n_threads, lang_probs);
}

// ---------------------------------------------------------------------------------------------------- getters
WB_EXPORT int whisper_n_len(struct whisper_context * ctx)              { return ctx->state->fe.n_len_org; }
WB_EXPORT int whisper_n_len_from_state(struct whisper_state * st)      { return st->fe.n_len_org; }
WB_EXPORT int whisper_n_vocab(struct whisper_context * ctx)            { return ctx->vocab.n_vocab; }
WB_EXPORT int whisper_n_text_ctx(struct whisper_context * ctx)         { return ctx->model.hp.n_text_ctx; }
WB_EXPORT int whisper_n_audio_ctx(struct whisper_context * ctx)        { return ctx->model.hp.n_audio_ctx; }
WB_EXPORT int whisper_is_multilingual(struct whisper_context * ctx)    { return ctx->vocab.is_multilingual() ? 1 : 0; }
WB_EXPORT int whisper_model_n_vocab(struct whisper_context * ctx)       { return ctx->model.hp.n_vocab; }
WB_EXPORT int whisper_model_n_audio_ctx(struct whisper_context * ctx)   { return ctx->model.hp.n_audio_ctx; }
WB_EXPORT int whisper_model_n_audio_state(struct whisper_context * ctx) { return ctx->model.hp.n_audio_state; }
WB_EXPORT int whisper_model_n_audio_head(struct whisper_context * ctx)  { return ctx->model.hp.n_audio_head; }
WB_EXPORT int whisper_model_n_audio_layer(struct whisper_context * ctx) { return ctx->model.hp.n_audio_layer; }
WB_EXPORT int whisper_model_n_text_ctx(struct whisper_context * ctx)    { return ctx->model.hp.n_text_ctx; }
WB_EXPORT int whisper_model_n_text_state(struct whisper_context * ctx)  { return ctx->model.hp.n_text_state; }
WB_EXPORT int whisper_model_n_text_head(struct whisper_context * ctx)   { return ctx->model.hp.n_text_head; }
WB_EXPORT int whisper_model_n_text_layer(struct whisper_context * ctx)  { return ctx->model.hp.n_text_layer; }
WB_EXPORT int whisper_model_n_mels(struct whisper_context * ctx)        { return ctx->model.hp.n_mels; }
WB_EXPORT int whisper_model_ftype(struct whisper_context * ctx)         { return ctx->model.hp.ftype; }
WB_EXPORT int whisper_model_type(struct whisper_context * ctx)          { return ctx->model.mtype; }
WB_EXPORT const char * whisper_model_type_readable(struct whisper_context * ctx) {
    static const char * const names[] = { "unknown", "tiny", "base", "small", "medium", "large" };
    const int t = ctx->model.mtype; return names[t >= 0 && t <= 5 ? t : 0];
}
WB_EXPORT const char * whisper_token_to_str(struct whisper_context * ctx, whisper_token token) {
    auto it = ctx->vocab.id_to_token.find(token);
    return it == ctx->vocab.id_to_token.end() ? "" : it->second.c_str();
}
WB_EXPORT whisper_token whisper_token_eot (struct whisper_context * ctx) { return ctx->vocab.token_eot; }
WB_EXPORT whisper_token whisper_token_sot (struct whisper_context * ctx) { return ctx->vocab.token_sot; }
WB_EXPORT whisper_token whisper_token_solm(struct whisper_context * ctx) { return ctx->vocab.token_solm; }
WB_EXPORT whisper_token whisper_token_prev(struct whisper_context * ctx) { return ctx->vocab.token_prev; }
WB_EXPORT whisper_token whisper_token_nosp(struct whisper_context * ctx) { return ctx->vocab.token_nosp; }
WB_EXPORT whisper_token whisper_token_not (struct whisper_context * ctx) { return ctx->vocab.token_not; }
WB_EXPORT whisper_token whisper_token_beg (struct whisper_context * ctx) { return ctx->vocab.token_beg; }
WB_EXPORT whisper_token whisper_token_lang(struct whisper_context * ctx, int lang_id) { return ctx->vocab.token_sot + 1 + lang_id; }
WB_EXPORT whisper_token whisper_token_translate (struct whisper_context * ctx) { return ctx->vocab.token_translate; }
WB_EXPORT whisper_token whisper_token_transcribe(struct whisper_context * ctx) { return ctx->vocab.token_transcribe; }

// ---------------------------------------------------------------------------------------------------- timings / diagnostics
WB_EXPORT struct whisper_timings * whisper_get_timings(struct whisper_context * ctx) {
    if (!ctx || !ctx->state) return nullptr;
    const whisper_state & s = *ctx->state;
    auto * t = new whisper_timings();
    t->sample_ms = 1e-3f * s.t_sample_us / std::max(1, s.n_sample);
    t->encode_ms = 1e-3f * s.t_encode_us / std::max(1, s.n_encode);
    t->decode_ms = 1e-3f * s.t_decode_us / std::max(1, s.n_decode);
    t->batchd_ms = 1e-3f * s.t_batchd_us / std::max(1, s.n_batchd);
    t->prompt_ms = 1e-3f * s.t_prompt_us / std::max(1, s.n_prompt);
    return t;
}
WB_EXPORT void whisper_print_timings(struct whisper_context * ctx) {
    const int64_t t_end = time_us();
    logf(LOG_INFO, "\n");
    logf(LOG_INFO, "%s:     load time = %8.2f ms\n", __func__, ctx->t_load_us / 1000.0f);
    if (ctx->state) {
        const whisper_state & s = *ctx->state;
        const int ns = std::max(1, s.n_sample), ne = std::max(1, s.n_encode), nd = std::max(1, s.n_decode), nb = std::max(1, s.n_batchd), np = std::max(1, s.n_prompt);
        logf(LOG_INFO, "%s:     fallbacks = %3d p / %3d h\n", __func__, s.n_fail_p, s.n_fail_h);
        logf(LOG_INFO, "%s:      mel time = %8.2f ms\n", __func__, s.t_mel_us / 1000.0f);
        logf(LOG_INFO, "%s:   sample time = %8.2f ms / %5d runs ( %8.2f ms per run)\n", __func__, 1e-3f * s.t_sample_us, ns, 1e-3f * s.t_sample_us / ns);
        logf(LOG_INFO, "%s:   encode time = %8.2f ms / %5d runs ( %8.2f ms per run)\n", __func__, 1e-3f * s.t_encode_us, ne, 1e-3f * s.t_encode_us / ne);
        logf(LOG_INFO, "%s:   decode time = %8.2f ms / %5d runs ( %8.2f ms per run)\n", __func__, 1e-3f * s.t_decode_us, nd, 1e-3f * s.t_decode_us / nd);
        logf(LOG_INFO, "%s:   batchd time = %8.2f ms / %5d runs ( %8.2f ms per run)\n", __func__, 1e-3f * s.t_batchd_us, nb, 1e-3f * s.t_batchd_us / nb);
        logf(LOG_INFO, "%s:   prompt time = %8.2f ms / %5d runs ( %8.2f ms per run)\n", __func__, 1e-3f * s.t_prompt_us, np, 1e-3f * s.t_prompt_us / np);
    }
    logf(LOG_INFO, "%s:    total time = %8.2f ms\n", __func__, (t_end - ctx->t_start_us) / 1000.0f);
}
WB_EXPORT void whisper_reset_timings(struct whisper_context * ctx) {
    ctx->t_start_us = time_us();
    if (ctx->state) {
        whisper_state & s = *ctx->state;
        s.t_mel_us = s.t_sample_us = s.t_encode_us = s.t_decode_us = s.t_batchd_us = s.t_prompt_us = 0;
        s.n_sample = s.n_encode = s.n_decode = s.n_batchd = s.n_prompt = 0;
    }
}
WB_EXPORT const char * whisper_print_system_info(void) {
    static std::string s;
    s = "WHISPER_B200 : CUDA = 1 | ARCH = sm_90a | WGMMA = 1 | TMA = 1 | CPU_FALLBACK = 0 | ";
    int ndev = 0; if (cudaGetDeviceCount(&ndev) == cudaSuccess) s += "DEVICES = " + std::to_string(ndev) + " | ";
    return s.c_str();
}
WB_EXPORT void whisper_log_set(ggml_log_callback cb, void * user_data) {
    set_log_sink(reinterpret_cast<void (*)(int, const char *, void *)>(cb), user_data);
}
// whisper_bench_memcpy / whisper_bench_ggml_mul_mat (whisper.h:746-753; `whisper-bench -w 1|2`): the reference measures its CPU backend's
// memcpy and ggml_mul_mat; here the same entry points measure what this engine runs on -- device copy bandwidth and the wgmma GEMM.
static std::string bench_memcpy_str() {
    std::string out;
    char line[256];
    int dev = 0; cudaGetDevice(&dev);
    const size_t bytes = (size_t) 1 << 30;
    DevBuf<uint8_t> a, b;
    if (!a.alloc(bytes, true) || !b.alloc(bytes)) return "memcpy: device allocation failed\n";
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    double best = 0.0;
    for (int it = 0; it < 6; ++it) {
        cudaEventRecord(e0); cudaMemcpyAsync(b.p, a.p, bytes, cudaMemcpyDeviceToDevice); cudaEventRecord(e1); cudaEventSynchronize(e1);
        float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
        if (it) best = std::max(best, 2.0 * bytes / 1e9 / (ms * 1e-3));
    }
    snprintf(line, sizeof(line), "memcpy: %8.2f GB/s (device %d, HBM read + write, 1 GiB copy, best of 5)\n", best, dev); out += line;
    std::vector<uint8_t> h((size_t) 256 << 20, 1);
    double h2d = 0.0;
    for (int it = 0; it < 3; ++it) {
        const int64_t t0 = time_us(); cudaMemcpy(a.p, h.data(), h.size(), cudaMemcpyHostToDevice); const int64_t t1 = time_us();
        h2d = std::max(h2d, h.size() / 1e9 / ((t1 - t0) * 1e-6));
    }
    snprintf(line, sizeof(line), "memcpy: %8.2f GB/s (pageable host -> device, 256 MiB)\n", h2d); out += line;
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    return out;
}
static std::string bench_mul_mat_str() {
    std::string out;
    char line[256];
    out += "wgmma GEMM, f16 x f16 -> f32 (persistent kernel, wb_gemm.cu); C[N][M] = A[M][K] . B[N][K]^T\n";
    const int sizes[] = { 256, 512, 1024, 2048, 4096, 8192 };
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    for (int n : sizes) {
        DevBuf<__half> A, B; DevBuf<float> Cd;
        if (!A.alloc((size_t) n * n, true) || !B.alloc((size_t) n * n, true) || !Cd.alloc((size_t) n * n)) break;
        GemmDesc g; g.M = n; g.N = n; g.K = n; g.BN = 256; g.v2 = 1; g.A.type = WT_F16; g.A.base = A.p;
        if (!make_tmap_f16(&g.tmA, A.p, n, n, 1, 1, n, 0, 0, 128) || !make_tmap_f16(&g.tmB, B.p, n, n, 1, 1, n, 0, 0, 256)) break;
        g.ep.out = Cd.p; g.ep.ldo = n;
        double best = 0.0;
        for (int it = 0; it < 6; ++it) {
            cudaEventRecord(e0); if (gemm_launch(g, 0) != cudaSuccess) break; cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms = 0; cudaEventElapsedTime(&ms, e0, e1);
            if (it) best = std::max(best, 2.0 * n * n * (double) n / 1e12 / (ms * 1e-3));
        }
        snprintf(line, sizeof(line), "%5d x %5d x %5d: %8.1f TFLOP/s\n", n, n, n, best); out += line;
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    return out;
}
WB_EXPORT const char * whisper_bench_memcpy_str(int)       { static std::string s; s = bench_memcpy_str(); return s.c_str(); }
WB_EXPORT int          whisper_bench_memcpy(int n)         { logf(LOG_INFO, "%s", whisper_bench_memcpy_str(n)); return 0; }
WB_EXPORT const char * whisper_bench_ggml_mul_mat_str(int) { static std::string s; s = bench_mul_mat_str(); return s.c_str(); }
WB_EXPORT int          whisper_bench_ggml_mul_mat(int n)   { logf(LOG_INFO, "%s", whisper_bench_ggml_mul_mat_str(n)); return 0; }

// ---------------------------------------------------------------------------------------------------- results
#define SEG(st, i) ((st)->result_all[(size_t) (i)])
WB_EXPORT int whisper_full_n_segments_from_state(struct whisper_state * st) { return (int) st->result_all.size(); }
WB_EXPORT int whisper_full_n_segments(struct whisper_context * ctx)         { return (int) ctx->state->result_all.size(); }
WB_EXPORT int whisper_full_lang_id_from_state(struct whisper_state * st)    { return st->lang_id; }
WB_EXPORT int whisper_full_lang_id(struct whisper_context * ctx)            { return ctx->state->lang_id; }
// with VAD the stored times are on the cut timeline; map them back to the original audio (whisper.cpp:8001-8033)
WB_EXPORT int64_t whisper_full_get_segment_t0_from_state(struct whisper_state * st, int i) {
    const int64_t t0 = SEG(st, i).t0;
    return (!st->vad.has_segments || st->vad.table.empty()) ? t0 : vad_map_segment_time(t0, st->vad.table);
}
WB_EXPORT int64_t whisper_full_get_segment_t1_from_state(struct whisper_state * st, int i) {
    const int64_t t1 = SEG(st, i).t1;
    if (!st->vad.has_segments || st->vad.table.empty()) return t1;
    const int64_t o0 = whisper_full_get_segment_t0_from_state(st, i);
    return std::max(vad_map_segment_time(t1, st->vad.table), o0 + 10);               // never a zero-length segment
}
WB_EXPORT int64_t whisper_full_get_segment_t0(struct whisper_context * ctx, int i)         { return whisper_full_get_segment_t0_from_state(ctx->state, i); }
WB_EXPORT int64_t whisper_full_get_segment_t1(struct whisper_context * ctx, int i)         { return whisper_full_get_segment_t1_from_state(ctx->state, i); }
WB_EXPORT bool whisper_full_get_segment_speaker_turn_next_from_state(struct whisper_state * st, int i) { return SEG(st, i).speaker_turn_next; }
WB_EXPORT bool whisper_full_get_segment_speaker_turn_next(struct whisper_context * ctx, int i)         { return SEG(ctx->state, i).speaker_turn_next; }
WB_EXPORT const char * whisper_full_get_segment_text_from_state(struct whisper_state * st, int i) { return SEG(st, i).text.c_str(); }
WB_EXPORT const char * whisper_full_get_segment_text(struct whisper_context * ctx, int i)         { return SEG(ctx->state, i).text.c_str(); }
WB_EXPORT float whisper_full_get_segment_no_speech_prob_from_state(struct whisper_state * st, int i) { return SEG(st, i).no_speech_prob; }
WB_EXPORT float whisper_full_get_segment_no_speech_prob(struct whisper_context * ctx, int i)         { return SEG(ctx->state, i).no_speech_prob; }
WB_EXPORT int whisper_full_n_tokens_from_state(struct whisper_state * st, int i) { return (int) SEG(st, i).tokens.size(); }
WB_EXPORT int whisper_full_n_tokens(struct whisper_context * ctx, int i)         { return (int) SEG(ctx->state, i).tokens.size(); }
WB_EXPORT const char * whisper_full_get_token_text_from_state(struct whisper_context * ctx, struct whisper_state * st, int i, int t) { return whisper_token_to_str(ctx, SEG(st, i).tokens[t].id); }
WB_EXPORT const char * whisper_full_get_token_text(struct whisper_context * ctx, int i, int t) { return whisper_token_to_str(ctx, SEG(ctx->state, i).tokens[t].id); }
WB_EXPORT whisper_token whisper_full_get_token_id_from_state(struct whisper_state * st, int i, int t) { return SEG(st, i).tokens[t].id; }
WB_EXPORT whisper_token whisper_full_get_token_id(struct whisper_context * ctx, int i, int t)         { return SEG(ctx->state, i).tokens[t].id; }
WB_EXPORT whisper_token_data whisper_full_get_token_data_from_state(struct whisper_state * st, int i, int t) { return SEG(st, i).tokens[t]; }
WB_EXPORT whisper_token_data whisper_full_get_token_data(struct whisper_context * ctx, int i, int t)         { return SEG(ctx->state, i).tokens[t]; }
WB_EXPORT int64_t whisper_full_get_token_t0_from_state(struct whisper_state * st, int i, int t) {       // whisper.cpp:8132-8158
    const int64_t t0 = SEG(st, i).tokens[t].t0;
    return (!st->vad.has_segments || st->vad.segments.empty()) ? t0 : vad_map_token_time(t0, st->vad.segments);
}
WB_EXPORT int64_t whisper_full_get_token_t1_from_state(struct whisper_state * st, int i, int t) {
    const int64_t t1 = SEG(st, i).tokens[t].t1;
    if (!st->vad.has_segments || st->vad.segments.empty()) return t1;
    return std::max(vad_map_token_time(t1, st->vad.segments), whisper_full_get_token_t0_from_state(st, i, t) + 1);
}
WB_EXPORT int64_t whisper_full_get_token_t0(struct whisper_context * ctx, int i, int t)         { return whisper_full_get_token_t0_from_state(ctx->state, i, t); }
WB_EXPORT int64_t whisper_full_get_token_t1(struct whisper_context * ctx, int i, int t)         { return whisper_full_get_token_t1_from_state(ctx->state, i, t); }
WB_EXPORT float whisper_full_get_token_p_from_state(struct whisper_state * st, int i, int t) { return SEG(st, i).tokens[t].p; }
WB_EXPORT float whisper_full_get_token_p(struct whisper_context * ctx, int i, int t)         { return SEG(ctx->state, i).tokens[t].p; }

WB_EXPORT int     whisper_full_n_vad_segments_from_state(struct whisper_state * st)               { return (int) st->vad.segments.size(); }   // whisper.cpp:8133-8158
WB_EXPORT int     whisper_full_n_vad_segments(struct whisper_context * ctx)                       { return (int) ctx->state->vad.segments.size(); }
WB_EXPORT int64_t whisper_full_get_vad_segment_t0_from_state(struct whisper_state * st, int i)    { return st->vad.segments[(size_t) i].orig_start; }
WB_EXPORT int64_t whisper_full_get_vad_segment_t0(struct whisper_context * ctx, int i)            { return ctx->state->vad.segments[(size_t) i].orig_start; }
WB_EXPORT int64_t whisper_full_get_vad_segment_t1_from_state(struct whisper_state * st, int i)    { return st->vad.segments[(size_t) i].orig_end; }
WB_EXPORT int64_t whisper_full_get_vad_segment_t1(struct whisper_context * ctx, int i)            { return ctx->state->vad.segments[(size_t) i].orig_end; }
// whisper_vad_* : wb_vad.cpp

// host-only test hook: the last decode request of an engine-less (scripted) state
WB_EXPORT int wb200_dbg_last_batch(struct whisper_state * st, int * tok, int * pos, int * seq, int8_t * want, int cap) {
    if (!st || !st->scripted || (int) st->dbg_tok.size() > cap) return -1;
    const int n = (int) st->dbg_tok.size();
    for (int i = 0; i < n; ++i) { tok[i] = st->dbg_tok[i]; pos[i] = st->dbg_pos[i]; seq[i] = st->dbg_seq[i]; want[i] = st->dbg_want[i]; }
    return n;
}

WB_EXPORT int wb200_dbg_last_attended(struct whisper_state * st, uint64_t * out, int cap) {
    if (!st || !st->scripted || (int) st->dbg_att.size() > cap) return -1;
    for (size_t i = 0; i < st->dbg_att.size(); ++i) out[i] = st->dbg_att[i];
    return (int) st->dbg_att.size();
}

// test hook: the window of the last DTW pass of this state: {mel frames, sot_len, seek, DTW passes of the state so far}
WB_EXPORT int wb200_dbg_last_dtw_window(struct whisper_state * st, int * out) {
    if (!st || !out) return -1;
    for (int i = 0; i < 4; ++i) out[i] = st->dtw_last_window[i];
    return 0;
}

// test hook: alignment-head weights of the last DTW pass of this state [heads][n_audio_ctx][tokens]; shape = {tokens, n_audio_ctx, heads}
WB_EXPORT int64_t wb200_dbg_last_dtw_qks(struct whisper_state * st, float * out, int64_t cap, int * shape) {
    if (!st) return -1;
    if (shape) { shape[0] = st->dtw_last_shape[0]; shape[1] = st->dtw_last_shape[1]; shape[2] = st->dtw_last_shape[2]; }
    const int64_t n = (int64_t) st->dtw_qk_last.size();
    if (!out) return n;
    if (n > cap) return -2;
    memcpy(out, st->dtw_qk_last.data(), (size_t) n * sizeof(float));
    return n;
}

// ---------------------------------------------------------------------------------------------------- engine extensions
WB_EXPORT int64_t wb200_read_tensor(struct whisper_state * st, int which, float * out, int64_t cap) {
    if (!st) return -1;
    if (!st->eng) return -1;
    Engine & E = *st->eng;
    const HParams & hp = E.m->hp;
    if (cudaSetDevice(E.m->device) != cudaSuccess) return -1;
    const int T = E.enc_n_ctx > 0 ? E.enc_n_ctx : hp.n_audio_ctx, d = hp.n_audio_state, Lt = hp.n_text_layer;
    if (which == 0) {
        const int64_t n = (int64_t) st->fe.n_mel * st->fe.n_len;
        if (!out) return n;
        if (n > cap) return -2;
        return cudaMemcpy(out, st->fe.mel.p, n * 4, cudaMemcpyDeviceToHost) == cudaSuccess ? n : -3;
    }
    if (which == 1 || which == 2) {
        const int64_t n = (int64_t) T * d;
        if (!out) return n;
        if (n > cap) return -2;
        const float * src = which == 1 ? E.conv32.p : E.enc32.p;
        if (!src) { set_error("wb200_read_tensor: set WB200_DEBUG_TAPS=1 before creating the state"); return -4; }
        return cudaMemcpy(out, src, n * 4, cudaMemcpyDeviceToHost) == cudaSuccess ? n : -3;
    }
    if (which == 3 || which == 4) {
        const int64_t n = (int64_t) Lt * E.Tp_max * d;
        if (!out) return n;
        if (n > cap) return -2;
        std::vector<__half> tmp((size_t) n);
        const __half * src = E.kv_cross.p + (size_t) st->slot * 2 * n + (which == 4 ? n : 0);
        if (cudaMemcpy(tmp.data(), src, (size_t) n * 2, cudaMemcpyDeviceToHost) != cudaSuccess) return -3;
        if (E.use_mk && mk_cross_head_major()) {                          // head-major in HBM: hand out the [Lt][Tp][d] view the tests expect
            const int Tp = E.Tp_max;
            for (int l = 0; l < Lt; ++l) for (int hh = 0; hh < d / 64; ++hh) for (int k = 0; k < Tp; ++k) for (int f = 0; f < 64; ++f)
                out[((size_t) l * Tp + k) * d + hh * 64 + f] = __half2float(tmp[(((size_t) l * (d / 64) + hh) * Tp + k) * 64 + f]);
        } else
        for (int64_t i = 0; i < n; ++i) out[i] = __half2float(tmp[(size_t) i]);
        return n;
    }
    return -5;
}
WB_EXPORT int wb200_last_encode_ms(struct whisper_state * st, float * out4) {
    if (!st || !out4 || !st->eng) return -1;
    for (int i = 0; i < 4; ++i) out4[i] = st->eng->last_ms[i];
    out4[0] = st->fe.last_mel_ms;
    return 0;
}
WB_EXPORT struct whisper_state * wb200_ctx_state(struct whisper_context * ctx) { return ctx ? ctx->state : nullptr; }
WB_EXPORT int wb200_state_device(struct whisper_state * st) { return (st && st->eng && st->eng->m) ? st->eng->m->device : -1; }
WB_EXPORT int wb200_n_devices(struct whisper_context * ctx) { return ctx ? 1 + (int) ctx->replicas.size() : 0; }
WB_EXPORT int wb200_pcm_upload(struct whisper_state * st, const float * samples, int n_samples) {
    if (!st || !samples || n_samples <= 0) return -1;
    return st->fe.pcm_upload(samples, n_samples) ? 0 : -1;
}
WB_EXPORT void wb200_profile_enable(int on) { wb::prof_enable(on != 0); }
WB_EXPORT void wb200_profile_collect(double * ms4, uint64_t * launches4, double * bytes4, double * flops4) { wb::prof_collect(ms4, launches4, bytes4, flops4); }
// test hook: run-ahead decode passes on (default) or off for every pool of the context, so that tests can compare both in one process
WB_EXPORT int wb200_dbg_run_ahead(struct whisper_context * ctx, int on) {
    if (!ctx) return -1;
    ctx->run_ahead = on != 0;
    if (ctx->pool) ctx->pool->run_ahead = on != 0;
    for (auto & r : ctx->replicas) if (r->pool) r->pool->run_ahead = on != 0;
    return 0;
}
WB_EXPORT void wb200_counters(double * out, int n) { for (int i = 0; i < n && i < 16; ++i) out[i] = wb::counter_get(i); }
WB_EXPORT void wb200_traffic(uint64_t * h2d, uint64_t * d2h) { if (h2d) *h2d = wb::h2d_bytes(); if (d2h) *d2h = wb::d2h_bytes(); }
WB_EXPORT const char * wb200_last_error(void) { return wb::last_error(); }
WB_EXPORT uint64_t wb200_launch_count(void)   { return wb::launch_count(); }

} // extern "C"

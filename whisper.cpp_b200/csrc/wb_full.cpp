// wb_full.cpp -- whisper_full / whisper_full_with_state / whisper_full_parallel and the host-side decoding policy:
// logits filtering, greedy / temperature / beam sampling, timestamp-driven window advance, fallback ladder, segment
// emission.  Semantics follow src/whisper.cpp:5947-6053 (defaults), 6156-6667 (filters, samplers, scoring),
// 6831-7788 (seek loop) and 7813-7941 (parallel); the device work goes through wb::encode_window / wb::decode_batch.
#include <numeric>
#include <algorithm>
#include <atomic>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <map>
#include <regex>
#include <thread>
#include <fstream>
#include <memory>
#include <mutex>
#include "wb_state.h"
#include "wb_dtw.h"

using namespace wb;

namespace {

const char * const k_non_speech[] = {   // src/whisper.cpp:6149-6154
    "\"", "#", "(", ")", "*", "+", "/", ":", ";", "<", "=", ">", "@", "[", "\\", "]", "^",
    "_", "`", "{", "|", "}", "~", "「", "」", "『", "』", "<<", ">>", "<<<", ">>>", "--",
    "---", "-(", "-[", "('", "(\"", "((", "))", "(((", ")))", "[[", "]]", "{{", "}}", "♪♪",
    "♪♪♪", "♩", "♪", "♫", "♬", "♭", "♮", "♯" };

// log-softmax over the finite entries (src/whisper.cpp:6156-6176)
void compute_logprobs(const std::vector<float> & logits, int n, std::vector<float> & logprobs) {
    const float mx = *std::max_element(logits.begin(), logits.begin() + n);
    float lse = 0.0f;
    for (int i = 0; i < n; ++i) if (logits[i] > -INFINITY) lse += expf(logits[i] - mx);
    lse = logf(lse) + mx;
    for (int i = 0; i < n; ++i) logprobs[i] = logits[i] > -INFINITY ? logits[i] - lse : -INFINITY;
}
void compute_probs(const std::vector<float> & logits, int n, const std::vector<float> & logprobs, std::vector<float> & probs) {
    for (int i = 0; i < n; ++i) probs[i] = logits[i] == -INFINITY ? 0.0f : expf(logprobs[i]);
}

// src/whisper.cpp:6196-6471
void process_logits(whisper_context & ctx, whisper_state & st, Decoder & dec, const whisper_full_params & params, float temperature) {
    const Vocab & vocab = ctx.vocab;
    const auto & cur = dec.sequence.tokens;
    const bool is_initial = cur.empty();
    const int n = vocab.n_vocab;
    auto & probs = dec.probs; auto & logits = dec.logits; auto & logprobs = dec.logprobs;
    logits.resize(n); probs.resize(n); logprobs.resize(n);
    memcpy(logits.data(), st.logits.data() + (size_t) dec.i_batch * n, (size_t) n * sizeof(float));
    if (temperature > 0.0f) for (int i = 0; i < n; ++i) logits[i] /= temperature;

    auto suppress = [&](int id) { if (id >= 0 && id < n) logits[id] = -INFINITY; };
    if (params.suppress_blank && is_initial) {
        suppress(vocab.token_eot);
        auto it = vocab.token_to_id.find(" ");
        if (it != vocab.token_to_id.end()) suppress(it->second);
    }
    suppress(vocab.token_not);
    if (params.no_timestamps) for (int i = vocab.token_beg; i < n; ++i) logits[i] = -INFINITY;
    if (!params.no_timestamps && !params.single_segment && params.max_tokens > 0 && (int) cur.size() >= params.max_tokens)
        for (int i = 0; i < vocab.token_eot; ++i) logits[i] = -INFINITY;
    suppress(vocab.token_sot); suppress(vocab.token_nosp);
    if (!params.tdrz_enable) suppress(vocab.token_solm);
    suppress(vocab.token_translate); suppress(vocab.token_transcribe); suppress(vocab.token_prev);
    for (int i = 0; i < 100; ++i) suppress(vocab.token_sot + 1 + i);       // one per entry of the language table
    suppress(vocab.token_prev);

    if (params.logits_filter_callback)
        params.logits_filter_callback(&ctx, &st, cur.data(), (int) cur.size(), logits.data(), params.logits_filter_callback_user_data);

    if (params.suppress_regex) {
        std::regex re(params.suppress_regex);
        for (const auto & kv : vocab.token_to_id) if (std::regex_match(kv.first, re)) suppress(kv.second);
    }
    if (params.suppress_nst) {
        for (const char * t : k_non_speech) {
            const std::string a = t, b = std::string(" ") + t;
            auto it = vocab.token_to_id.find(a); if (it != vocab.token_to_id.end()) suppress(it->second);
            it = vocab.token_to_id.find(b);      if (it != vocab.token_to_id.end()) suppress(it->second);
        }
        auto it = vocab.token_to_id.find(" -"); if (it != vocab.token_to_id.end()) suppress(it->second);
        it = vocab.token_to_id.find(" '");      if (it != vocab.token_to_id.end()) suppress(it->second);
    }
    { // timestamps come in pairs, except right before EOT
        const bool last_ts = !cur.empty() && cur.back().id >= vocab.token_beg;
        const bool penult_ts = cur.size() < 2 || cur[cur.size() - 2].id >= vocab.token_beg;
        if (last_ts) {
            if (penult_ts) for (int i = vocab.token_beg; i < n; ++i) logits[i] = -INFINITY;
            else           for (int i = 0; i < vocab.token_eot; ++i) logits[i] = -INFINITY;
        }
    }
    if (is_initial && params.max_initial_ts > 0.0f) {
        const float precision = float(WB_CHUNK_SIZE) / ctx.model.hp.n_audio_ctx;
        const int tid0 = (int) std::round(params.max_initial_ts / precision);
        for (int i = vocab.token_beg + tid0 + 1; i < n; ++i) logits[i] = -INFINITY;
    }
    if (dec.has_ts) {
        const int tid0 = dec.seek_delta / 2;
        for (int i = vocab.token_beg; i < vocab.token_beg + tid0 && i < n; ++i) logits[i] = -INFINITY;
    }
    compute_logprobs(logits, n, logprobs);
    { // if the timestamp mass beats every text token, force a timestamp
        float ts_logprob = -INFINITY;
        {
            float lse = 0.0f;
            const float mx = *std::max_element(logprobs.begin() + vocab.token_beg, logprobs.begin() + n);
            for (int i = vocab.token_beg; i < n; ++i) if (logprobs[i] > -INFINITY) lse += expf(logprobs[i] - mx);
            if (lse > 0.0f) ts_logprob = logf(lse) + mx;
        }
        const float max_text = *std::max_element(logprobs.begin(), logprobs.begin() + vocab.token_beg);
        if (ts_logprob > max_text) for (int i = 0; i < vocab.token_beg; ++i) { logits[i] = -INFINITY; logprobs[i] = -INFINITY; }
        else if (params.n_grammar_rules > 0) {                   // whisper.cpp:6388-6410: penalise what the grammar cannot continue with
            grammar_penalize(vocab, dec.grammar, params.grammar_penalty, logits);
            compute_logprobs(logits, n, logprobs);
        }
    }
    compute_probs(logits, n, logprobs, probs);
}

whisper_token_data blank_token() { whisper_token_data t; memset(&t, 0, sizeof(t)); t.t0 = t.t1 = t.t_dtw = -1; return t; }

void timestamp_stats(const Vocab & vocab, const std::vector<float> & probs, whisper_token & tid, float & pt, float & ptsum) {
    double sum_ts = 0.0, max_ts = 0.0;
    for (int i = vocab.token_beg; i < vocab.n_vocab; ++i) {
        if (probs[i] == -INFINITY) continue;
        sum_ts += probs[i];
        if (max_ts < probs[i]) { max_ts = probs[i]; tid = i; }
    }
    pt = (float) (max_ts / (sum_ts + 1e-10)); ptsum = (float) sum_ts;
}

// src/whisper.cpp:6486-6543
whisper_token_data sample_token(whisper_context & ctx, Decoder & dec, bool best) {
    const Vocab & vocab = ctx.vocab;
    whisper_token_data r = blank_token();
    timestamp_stats(vocab, dec.probs, r.tid, r.pt, r.ptsum);
    if (best) {
        for (int i = 0; i < vocab.n_vocab; ++i) if (r.p < dec.probs[i]) { r.id = i; r.p = dec.probs[i]; r.plog = dec.logprobs[i]; }
    } else {
        std::discrete_distribution<> dist(dec.probs.begin(), dec.probs.end());
        r.id = dist(dec.rng); r.p = dec.probs[r.id]; r.plog = dec.logprobs[r.id];
    }
    if (r.id >= vocab.token_beg) { r.tid = r.id; r.pt = r.p; }
    return r;
}

// src/whisper.cpp:6545-6618: k draws from the categorical distribution (the partial sort of the reference has no effect on the result)
std::vector<whisper_token_data> sample_token_topk(whisper_context & ctx, Decoder & dec, int k) {
    const Vocab & vocab = ctx.vocab;
    whisper_token tid = vocab.token_beg; float pt = 0.0f, ptsum = 0.0f;
    timestamp_stats(vocab, dec.probs, tid, pt, ptsum);
    std::discrete_distribution<> dist(dec.probs.begin(), dec.probs.end());
    std::vector<whisper_token_data> out; out.reserve(k);
    for (int i = 0; i < k; ++i) {
        const int id = dist(dec.rng);
        whisper_token_data t = blank_token();
        t.id = id; t.tid = tid; t.p = dec.probs[id]; t.plog = dec.logprobs[id]; t.pt = pt; t.ptsum = ptsum;
        if (t.id >= vocab.token_beg) { t.tid = t.id; t.pt = t.p; }
        out.push_back(t);
    }
    return out;
}

// the same k draws with the uniforms already taken from dec.rng: std::discrete_distribution (libstdc++) normalises the probabilities by
// their sum, forms the running sums (the last one forced to 1) and returns lower_bound(cp, u)
std::vector<whisper_token_data> sample_token_topk_u(whisper_context & ctx, Decoder & dec, int k, const double * u) {
    const Vocab & vocab = ctx.vocab;
    whisper_token tid = vocab.token_beg; float pt = 0.0f, ptsum = 0.0f;
    timestamp_stats(vocab, dec.probs, tid, pt, ptsum);
    std::vector<double> cp(dec.probs.begin(), dec.probs.end());
    const double sum = std::accumulate(cp.begin(), cp.end(), 0.0);
    for (double & v : cp) v /= sum;
    std::partial_sum(cp.begin(), cp.end(), cp.begin());
    if (!cp.empty()) cp.back() = 1.0;
    std::vector<whisper_token_data> out; out.reserve(k);
    for (int i = 0; i < k; ++i) {
        const int id = (int) (std::lower_bound(cp.begin(), cp.end(), u[i]) - cp.begin());
        whisper_token_data t = blank_token();
        t.id = id; t.tid = tid; t.p = dec.probs[id]; t.plog = dec.logprobs[id]; t.pt = pt; t.ptsum = ptsum;
        if (t.id >= vocab.token_beg) { t.tid = t.id; t.pt = t.p; }
        out.push_back(t);
    }
    return out;
}

// src/whisper.cpp:6621-6667
void sequence_score(const whisper_full_params & params, Sequence & s) {
    if (s.result_len == 0) return;
    double r = 0.0;
    for (int i = 0; i < s.result_len; ++i) r += s.tokens[i].plog;
    s.sum_logprobs = r; s.avg_logprobs = r / s.result_len;
    double penalty = s.result_len;
    if (params.length_penalty > 0.0f) penalty = pow((5.0 + penalty) / 6.0, params.length_penalty);
    s.score = r / penalty;
    std::map<whisper_token, int> counts; int cnt = 0;
    for (int i = std::max(0, s.result_len - 32); i < s.result_len; ++i) { counts[s.tokens[i].id]++; cnt++; }
    double ent = 0.0;
    for (const auto & kv : counts) { const double p = kv.second / (double) cnt; ent -= p * log(p); }
    s.entropy = ent;
}

bool tokens_equal(const Sequence & a, const Sequence & b) {
    if (a.tokens.size() != b.tokens.size()) return false;
    for (int i = (int) a.tokens.size() - 1; i >= 0; --i) if (a.tokens[i].id != b.tokens[i].id) return false;
    return true;
}

std::string to_timestamp(int64_t t, bool comma = false) {
    int64_t msec = t * 10;
    const int64_t hr = msec / 3600000; msec -= hr * 3600000;
    const int64_t mn = msec / 60000;   msec -= mn * 60000;
    const int64_t sec = msec / 1000;   msec -= sec * 1000;
    char buf[32];
    snprintf(buf, sizeof(buf), "%02d:%02d:%02d%s%03d", (int) hr, (int) mn, (int) sec, comma ? "," : ".", (int) msec);
    return buf;
}

// ---- experimental token-level timestamps (params.token_timestamps; src/whisper.cpp:8500-8820) and max_len wrapping (6096-6147) ----
// weight of a token's text in the split of a time interval: spaces ~0, letters 1, commas 2, sentence marks and digits 3
// (UTF-8 aware, full-width forms count like their ASCII twins; src/whisper.cpp:8512-8590)
float voice_length(const std::string & text) {
    const unsigned char * s = (const unsigned char *) text.data();
    const size_t n = text.size();
    float res = 0.0f;
    size_t i = 0;
    while (i < n) {
        const unsigned char c = s[i];
        int len = c < 0x80 ? 1 : (c >> 5) == 0x6 ? 2 : (c >> 4) == 0xE ? 3 : (c >> 3) == 0x1E ? 4 : 1;
        uint32_t cp = len == 1 ? c : len == 2 ? (c & 0x1Fu) : len == 3 ? (c & 0x0Fu) : (c & 0x07u);
        bool ok = i + (size_t) len <= n;
        for (int k = 1; ok && k < len; ++k) {
            if ((s[i + k] & 0xC0) != 0x80) ok = false; else cp = (cp << 6) | (s[i + k] & 0x3Fu);
        }
        if (!ok) { cp = c; len = 1; }                            // invalid sequence: the lead byte counts as one symbol
        i += (size_t) len;
        if (cp == ' ' || cp == 0x3000) res += 0.01f;
        else if (cp == ',' || cp == 0xFF0C || cp == 0x3001 || cp == 0xFF1B || cp == 0xFF1A) res += 2.00f;
        else if (cp == '.' || cp == '!' || cp == '?' || cp == 0x3002 || cp == 0xFF0E || cp == 0xFF01 || cp == 0xFF1F || cp == 0x2026) res += 3.00f;
        else if ((cp >= '0' && cp <= '9') || (cp >= 0xFF10 && cp <= 0xFF19)) res += 3.00f;
        else res += 1.00f;
    }
    return res;
}

// mean |signal| over a window of 2*hw+1 samples, window clipped at the ends but always divided by 2*hw+1 (whisper.cpp:8593-8609)
std::vector<float> signal_energy(const float * signal, int n_samples, int hw) {
    std::vector<float> out((size_t) std::max(n_samples, 0));
    for (int i = 0; i < n_samples; ++i) {
        float sum = 0;
        for (int j = std::max(0, i - hw); j <= std::min(n_samples - 1, i + hw); ++j) sum += fabs(signal[j]);
        out[i] = sum / (2 * hw + 1);
    }
    return out;
}

// token t0/t1 of segment `i_segment`: anchor on confident timestamp predictions (pt, ptsum), share the gaps in proportion to the
// voice length, then snap to the signal energy.  state.t_beg / t_last / tid_last carry over between segments.
void token_level_timestamps(whisper_context & ctx, whisper_state & st, int i_segment, float thold_pt, float thold_ptsum) {
    Segment & seg = st.result_all[i_segment];
    auto & tk = seg.tokens;
    const int n_samples = (int) st.energy.size(), n = (int) tk.size();
    if (n_samples == 0) { logf(LOG_ERROR, "%s: no signal data available\n", __func__); return; }
    if (n == 0) return;
    const int64_t t0 = seg.t0, t1 = seg.t1;
    if (n == 1) { tk[0].t0 = t0; tk[0].t1 = t1; return; }
    const whisper_token beg = ctx.vocab.token_beg, eot = ctx.vocab.token_eot;

    for (int j = 0; j < n; ++j) {
        if (j == 0) {
            if (tk[0].id == beg) { tk[0].t0 = t0; tk[0].t1 = t0; tk[1].t0 = t0; st.t_beg = t0; st.t_last = t0; st.tid_last = beg; }
            else tk[0].t0 = st.t_last;
        }
        const int64_t tt = st.t_beg + 2 * (tk[j].tid - beg);
        tk[j].vlen = voice_length(whisper_token_to_str(&ctx, tk[j].id));
        if (tk[j].pt > thold_pt && tk[j].ptsum > thold_ptsum && tk[j].tid > st.tid_last && tt <= t1) {
            if (j > 0) tk[j - 1].t1 = tt;
            tk[j].t0 = tt;
            st.tid_last = tk[j].tid;
        }
    }
    tk[n - 2].t1 = t1; tk[n - 1].t0 = t1; tk[n - 1].t1 = t1;
    st.t_last = t1;

    // runs of tokens without an end time share [t0 of the first, t1 of the last] in proportion to their voice length
    for (int p0 = 0; p0 < n; ) {
        int p1 = p0;
        while (p1 < n && tk[p1].t1 < 0) ++p1;
        if (p1 >= n) p1 = n - 1;
        if (p1 > p0) {
            double psum = 0.0;
            for (int j = p0; j <= p1; ++j) psum += tk[j].vlen;
            const double dt = tk[p1].t1 - tk[p0].t0;
            for (int j = p0 + 1; j <= p1; ++j) {
                const double ct = tk[j - 1].t0 + dt * tk[j - 1].vlen / psum;
                tk[j - 1].t1 = ct; tk[j].t0 = ct;
            }
        }
        p0 = p1 + 1;
    }
    for (int j = 0; j < n - 1; ++j) {                            // keep the intervals ordered
        if (tk[j].t1 < 0) tk[j + 1].t0 = tk[j].t1;
        if (j > 0 && tk[j - 1].t1 > tk[j].t0) { tk[j].t0 = tk[j - 1].t1; tk[j].t1 = std::max(tk[j].t0, tk[j].t1); }
    }

    // stretch or shrink every text token to the region where the signal is above half of its local mean
    auto to_sample = [&](int64_t t) { return std::max(0, std::min(n_samples - 1, (int) (((t - seg.t0) * WB_SAMPLE_RATE) / 100))); };
    auto to_time   = [&](int k) -> int64_t { return (100ll * k) / WB_SAMPLE_RATE + seg.t0; };
    const int hw = WB_SAMPLE_RATE / 8;
    for (int j = 0; j < n; ++j) {
        if (tk[j].id >= eot) continue;
        int s0 = to_sample(tk[j].t0), s1 = to_sample(tk[j].t1);
        const int ss0 = std::max(s0 - hw, 0), ss1 = std::min(s1 + hw, n_samples);
        float sum = 0.0f;
        for (int k = ss0; k < ss1; ++k) sum += st.energy[k];
        const float thold = 0.5 * sum / (ss1 - ss0);
        {
            int k = s0;
            if (st.energy[k] > thold && j > 0) {
                while (k > 0 && st.energy[k] > thold) --k;
                tk[j].t0 = to_time(k);
                if (tk[j].t0 < tk[j - 1].t1) tk[j].t0 = tk[j - 1].t1; else s0 = k;
            } else {
                while (st.energy[k] < thold && k < s1) ++k;
                s0 = k;
                tk[j].t0 = to_time(k);
            }
        }
        {
            int k = s1;
            if (st.energy[k] > thold) {
                while (k < n_samples - 1 && st.energy[k] > thold) ++k;
                tk[j].t1 = to_time(k);
                if (j < n - 1 && tk[j].t1 > tk[j + 1].t0) tk[j].t1 = tk[j + 1].t0; else s1 = k;
            } else {
                while (st.energy[k] < thold && k > s0) --k;
                s1 = k;
                tk[j].t1 = to_time(k);
            }
        }
    }
}

// split the last segment so that no piece has more than max_len characters (UTF-8 code points); returns the number of pieces
int wrap_segment(whisper_context & ctx, whisper_state & st, int max_len, bool split_on_word) {
    Segment cur = st.result_all.back();
    int pieces = 1, acc = 0;
    std::string text;
    for (int i = 0; i < (int) cur.tokens.size(); ++i) {
        const whisper_token_data & tok = cur.tokens[i];
        if (tok.id >= ctx.vocab.token_eot) continue;
        const char * txt = whisper_token_to_str(&ctx, tok.id);
        int chars = 0;
        for (const char * q = txt; *q; ++q) if ((*q & 0xC0) != 0x80) ++chars;
        if (acc + chars > max_len && i > 0 && (!split_on_word || txt[0] == ' ')) {
            Segment & head = st.result_all.back();
            head.text = std::move(text); head.t1 = tok.t0; head.tokens.resize(i); head.speaker_turn_next = false;
            Segment tail;
            tail.t0 = tok.t0; tail.t1 = cur.t1; tail.tokens.assign(cur.tokens.begin() + i, cur.tokens.end()); tail.speaker_turn_next = cur.speaker_turn_next;
            st.result_all.push_back(tail);
            acc = 0; text.clear();
            cur = st.result_all.back();
            i = -1;
            ++pieces;
        } else {
            acc += chars; text += txt;
        }
    }
    st.result_all.back().text = std::move(text);
    return pieces;
}

// static part of the logits filter as a bit mask for the on-device sampler (same ids process_logits suppresses)
void build_static_mask(const whisper_context & ctx, const whisper_full_params & params, std::vector<uint32_t> & bits, uint64_t & key) {
    const Vocab & vocab = ctx.vocab;
    const int n = vocab.n_vocab;
    bits.assign((size_t) (n + 31) / 32, 0u);
    auto sup = [&](int id) { if (id >= 0 && id < n) bits[id >> 5] |= 1u << (id & 31); };
    sup(vocab.token_not); sup(vocab.token_sot); sup(vocab.token_nosp);
    if (!params.tdrz_enable) sup(vocab.token_solm);
    sup(vocab.token_translate); sup(vocab.token_transcribe); sup(vocab.token_prev);
    for (int i = 0; i < 100; ++i) sup(vocab.token_sot + 1 + i);
    if (params.suppress_regex) {
        std::regex re(params.suppress_regex);
        for (const auto & kv : vocab.token_to_id) if (std::regex_match(kv.first, re)) sup(kv.second);
    }
    if (params.suppress_nst) {
        for (const char * t : k_non_speech) {
            auto it = vocab.token_to_id.find(t); if (it != vocab.token_to_id.end()) sup(it->second);
            it = vocab.token_to_id.find(std::string(" ") + t); if (it != vocab.token_to_id.end()) sup(it->second);
        }
        auto it = vocab.token_to_id.find(" -"); if (it != vocab.token_to_id.end()) sup(it->second);
        it = vocab.token_to_id.find(" '");      if (it != vocab.token_to_id.end()) sup(it->second);
    }
    uint64_t h = 1469598103934665603ull;
    for (uint32_t w : bits) { h ^= w; h *= 1099511628211ull; }
    key = h | 1ull;
}

whisper_token_data from_samp(const SampOut & o) {
    whisper_token_data t = blank_token();
    t.id = o.id; t.tid = o.tid; t.p = o.p; t.plog = o.plog; t.pt = o.pt; t.ptsum = o.ptsum;
    return t;
}

// uniform part of the on-device filter: special ids and the switches of whisper_full_params (whisper.cpp:6205-6346)
void make_samp_cfg(const whisper_context & ctx, const whisper_full_params & params, SampCfg & cfg) {
    const Vocab & vocab = ctx.vocab;
    cfg.token_eot = vocab.token_eot; cfg.token_beg = vocab.token_beg; cfg.token_nosp = vocab.token_nosp;
    { auto it = vocab.token_to_id.find(" "); cfg.space_id = it == vocab.token_to_id.end() ? -1 : it->second; }
    cfg.suppress_blank = params.suppress_blank ? 1 : 0;
    cfg.no_timestamps = params.no_timestamps ? 1 : 0;
    cfg.max_initial_tid = params.max_initial_ts > 0.0f ? (int) std::round(params.max_initial_ts / (float(WB_CHUNK_SIZE) / ctx.model.hp.n_audio_ctx)) : -1;
}

// state of the logits filter for the NEXT token of a decoder (whisper.cpp:6205, 6252, 6319-6320, 6350-6351)
void samp_rowinfo(const Vocab & vocab, const whisper_full_params & params, const Decoder & d, int * out2) {
    const auto & cur = d.sequence.tokens;
    int f = 0;
    if (cur.empty()) f |= 1;
    if (!cur.empty() && cur.back().id >= vocab.token_beg) f |= 2;
    if (cur.size() < 2 || cur[cur.size() - 2].id >= vocab.token_beg) f |= 4;
    if (d.has_ts) f |= 8;
    if (!params.no_timestamps && !params.single_segment && params.max_tokens > 0 && (int) cur.size() >= params.max_tokens) f |= 16;
    out2[0] = f; out2[1] = d.seek_delta / 2;
}

// samp_rowinfo of the step after the one being submitted, were the token sampled now a text token (< token_beg) appended to `d`
void samp_rowinfo_next(const Vocab & vocab, const whisper_full_params & params, const Decoder & d, int * out2) {
    const auto & cur = d.sequence.tokens;
    int f = 0;
    if (cur.empty() || cur.back().id >= vocab.token_beg) f |= 4;
    if (d.has_ts) f |= 8;
    if (!params.no_timestamps && !params.single_segment && params.max_tokens > 0 && (int) cur.size() + 1 >= params.max_tokens) f |= 16;
    out2[0] = f; out2[1] = d.seek_delta / 2;
}

// P(no-speech token) exactly as whisper.cpp:7190-7200 computes it: row 0 of the logits buffer, normalised with the log-sum-exp that
// whisper_compute_logprobs (whisper.cpp:6156-6176) forms against the maximum of the WHOLE buffer (see whisper_state::lrows)
float row0_nosp(const whisper_context & ctx, const whisper_state & st) {
    const int n = ctx.vocab.n_vocab;
    if (st.lrows.empty()) return 1.0f / (float) n;
    float mx_all = -INFINITY;
    for (const auto & r : st.lrows) mx_all = std::max(mx_all, r.mx);
    float lse, l_nosp;
    if (st.row0_is_copy && (int) st.row0_copy.size() >= n) {                  // the row itself is here: the reference's loop, term by term
        float s = 0.0f;
        for (int i = 0; i < n; ++i) if (st.row0_copy[i] > -INFINITY) s += expf(st.row0_copy[i] - mx_all);
        lse = logf(s) + mx_all; l_nosp = st.row0_copy[ctx.vocab.token_nosp];
    } else {                                                                   // summary of the row (on-device sampler, or a zero-filled row)
        const auto & r = st.lrows[0];
        lse = logf(r.sum * expf(r.mx - mx_all)) + mx_all; l_nosp = r.nosp;     // underflows to log(0) where the reference's sum does
    }
    if (l_nosp == -INFINITY) return 0.0f;
    return expf(l_nosp - lse);
}

template <typename F> void run_parallel(int n_threads, F && fn) {
    if (n_threads <= 1) { fn(); return; }
    std::vector<std::thread> th(n_threads - 1);
    for (auto & t : th) t = std::thread(fn);
    fn();
    for (auto & t : th) t.join();
}


// One extra decoder pass over [sot, (lang), no_timestamps, text tokens of the window's segments, eot].  It is an ordinary decode request of the
// pool that also captures the cross-attention queries of the alignment heads; the batch it joins computes the softmax weights of every
// DTW request on the device in one launch, and then the warping path of each (normalisation, median filter, mean over heads, DTW and
// backtrace: DtwPaths, Group::run); only the assignment of the path to the tokens (dtw_assign) runs here, on the state's own thread.
bool dtw_window(whisper_context & ctx, whisper_state & st, const whisper_full_params & params, int i_segment, int n_segments, int seek, int n_frames) {
    const Vocab & vocab = ctx.vocab;
    const int n_audio_ctx = st.exp_n_audio_ctx > 0 ? st.exp_n_audio_ctx : ctx.model.hp.n_audio_ctx;
    if (n_frames > 2 * n_audio_ctx) { set_error("dtw: %d frames exceed the audio context", n_frames); return false; }
    std::vector<int> tokens = { vocab.token_sot };
    if (vocab.is_multilingual()) { const int lang_id = whisper_lang_id(params.language); st.lang_id = lang_id; tokens.push_back(vocab.token_sot + 1 + lang_id); }
    const int sot_len = (int) tokens.size();
    tokens.push_back(vocab.token_not);
    for (int i = i_segment; i < i_segment + n_segments; ++i) for (const auto & t : st.result_all[(size_t) i].tokens) if (t.id < vocab.token_eot) tokens.push_back(t.id);
    tokens.push_back(vocab.token_eot);
    const int n = (int) tokens.size();
    if (n > ctx.model.hp.n_text_ctx) { set_error("dtw: %d tokens exceed the text context", n); return false; }
    std::vector<int> pos((size_t) n), seq((size_t) n, 0); std::vector<int8_t> want((size_t) n, 0);
    for (int i = 0; i < n; ++i) pos[(size_t) i] = i;
    want[(size_t) n - 1] = 1;
    st.kv.clear();
    st.kv.seq_rm(0, 0, -1);
    // where the window's own steps use the device sampler, the pass offers the same configuration: a batch of DTW passes alone then still
    // returns the raw summary of its logits rows instead of full logits
    std::vector<uint32_t> mask_bits; SampReq sreq; std::vector<int> rowinfo((size_t) 2 * n, 0);
    const bool dev = !params.logits_filter_callback && !(params.grammar_rules && params.n_grammar_rules > 0) && getenv("WB200_HOST_SAMPLER") == nullptr;
    if (dev) {
        build_static_mask(ctx, params, mask_bits, sreq.mask_key);
        sreq.mask_bits = &mask_bits; sreq.rowinfo = rowinfo.data();
        make_samp_cfg(ctx, params, sreq.cfg);
    }
    st.dtw_tok.clear(); st.dtw_time.clear();
    if (!decode_batch(ctx, st, tokens.data(), pos.data(), seq.data(), want.data(), n, dev ? &sreq : nullptr, n_audio_ctx, sot_len, n_frames)) return false;
    if (st.dtw_qk_last.size() != (size_t) n * n_audio_ctx * ctx.dtw_heads.size()) { set_error("dtw: the pass returned no alignment weights"); return false; }
    st.dtw_last_window[0] = n_frames; st.dtw_last_window[1] = sot_len; st.dtw_last_window[2] = seek; st.dtw_last_window[3]++;
    const int64_t t0 = time_us();
    dtw_assign(st.dtw_tok, st.dtw_time, seek, vocab.token_eot, st.result_all, i_segment, n_segments);
    counter_add(10, 1e-3 * (double) (time_us() - t0));           // host DTW ms (wb200_counters): the assignment of the device's path
    return true;
}
} // namespace

extern "C" {

WB_EXPORT struct whisper_full_params whisper_full_default_params(enum whisper_sampling_strategy strategy) {   // whisper.cpp:5947-6053
    struct whisper_full_params p;
    memset(&p, 0, sizeof(p));
    p.strategy = strategy;
    p.n_threads = std::min(4, (int) std::thread::hardware_concurrency());
    p.n_max_text_ctx = 16384;
    p.no_context = true; p.print_progress = true; p.print_timestamps = true;
    p.thold_pt = 0.01f; p.thold_ptsum = 0.01f;
    p.language = "en";
    p.suppress_blank = true;
    p.temperature = 0.0f; p.max_initial_ts = 1.0f; p.length_penalty = -1.0f;
    p.temperature_inc = 0.2f; p.entropy_thold = 2.4f; p.logprob_thold = -1.0f; p.no_speech_thold = 0.6f;
    p.greedy.best_of = -1; p.beam_search.beam_size = -1; p.beam_search.patience = -1.0f;
    p.grammar_penalty = 100.0f;
    p.vad_params = whisper_vad_default_params();
    if (strategy == WHISPER_SAMPLING_GREEDY) p.greedy.best_of = 5;
    else if (strategy == WHISPER_SAMPLING_BEAM_SEARCH) { p.beam_search.beam_size = 5; p.beam_search.patience = -1.0f; }
    return p;
}
WB_EXPORT struct whisper_full_params * whisper_full_default_params_by_ref(enum whisper_sampling_strategy strategy) {
    auto * p = new whisper_full_params(); *p = whisper_full_default_params(strategy); return p;
}

WB_EXPORT int whisper_full_with_state(struct whisper_context * ctx, struct whisper_state * state, struct whisper_full_params params,
                                      const float * samples, int n_samples) {
    if (!ctx || !state) return -1;
    GroupCall group_call(state);                  // this state takes part in the context's lock-step passes until the call returns
    auto & result_all = state->result_all;
    result_all.clear();
    const Vocab & vocab = ctx->vocab;

    if (n_samples > 0) {
        if (whisper_pcm_to_mel_with_state(ctx, state, samples, n_samples, params.n_threads) != 0) {
            logf(LOG_ERROR, "%s: failed to compute log mel spectrogram\n", __func__);
            return -2;
        }
    }
    if (params.language == nullptr || strlen(params.language) == 0 || strcmp(params.language, "auto") == 0 || params.detect_language) {
        std::vector<float> probs(whisper_lang_max_id() + 1, 0.0f);
        const int lang_id = whisper_lang_auto_detect_with_state(ctx, state, 0, params.n_threads, probs.data());
        if (lang_id < 0) { logf(LOG_ERROR, "%s: failed to auto-detect language\n", __func__); return -3; }
        state->lang_id = lang_id;
        params.language = whisper_lang_str(lang_id);
        logf(LOG_INFO, "%s: auto-detected language: %s (p = %f)\n", __func__, params.language, probs[lang_id]);
        if (params.detect_language) return 0;
    }
    if (params.token_timestamps) {                               // whisper.cpp:6868-6875
        state->t_beg = 0; state->t_last = 0; state->tid_last = 0;
        if (n_samples > 0) {
            std::vector<float> host;
            const float * pcm = samples;
            if (!samples || wb::tls_pcm_is_device()) {            // PCM lives in HBM (wb200_pcm_upload / device-pointer batch): bring it back once
                host.resize((size_t) n_samples);
                const float * src = samples ? samples : state->fe.pcm.p;
                if (!src || cudaMemcpy(host.data(), src, (size_t) n_samples * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess) {
                    logf(LOG_ERROR, "%s: cannot read the PCM back for token_timestamps\n", __func__); return -2;
                }
                pcm = host.data();
            }
            state->energy = signal_energy(pcm, n_samples, 32);
        }
    }

    const int seek_start = params.offset_ms / 10;
    const int seek_end = params.duration_ms == 0 ? whisper_n_len_from_state(state) : seek_start + params.duration_ms / 10;
    const int delta_min = 10;
    if (seek_end < seek_start + delta_min) {
        logf(LOG_WARN, "%s: input is too short - %d ms < 100 ms. consider padding the input audio with silence\n", __func__, (seek_end - seek_start) * 10);
        return 0;
    }

    std::vector<float> temperatures;
    if (params.temperature_inc > 0.0f) for (float t = params.temperature; t < 1.0f + 1e-6f; t += params.temperature_inc) temperatures.push_back(t);
    else temperatures.push_back(params.temperature);

    int n_decoders = 1;
    if (params.strategy == WHISPER_SAMPLING_GREEDY) n_decoders = params.greedy.best_of;
    else if (params.strategy == WHISPER_SAMPLING_BEAM_SEARCH) n_decoders = std::max(params.greedy.best_of, params.beam_search.beam_size);
    n_decoders = std::max(1, n_decoders);
    if (n_decoders > MAX_DECODERS) { logf(LOG_ERROR, "%s: too many decoders requested (%d), max = %d\n", __func__, n_decoders, MAX_DECODERS); return -4; }
    for (int j = 1; j < n_decoders; ++j) state->decoders[j].rng = std::mt19937(j);

    auto & past0 = state->prompt_past0; auto & past1 = state->prompt_past1;
    if (params.no_context) { past0.clear(); past1.clear(); }
    const int n_text_ctx = ctx->model.hp.n_text_ctx;
    const int max_prompt_ctx = std::min(params.n_max_text_ctx, n_text_ctx / 2);

    std::vector<whisper_token> init_prompt_tokens;
    if (!params.prompt_tokens && params.initial_prompt) {
        init_prompt_tokens.resize(1024);
        int need = whisper_tokenize(ctx, params.initial_prompt, init_prompt_tokens.data(), (int) init_prompt_tokens.size());
        if (need < 0) { init_prompt_tokens.resize(-need); need = whisper_tokenize(ctx, params.initial_prompt, init_prompt_tokens.data(), (int) init_prompt_tokens.size()); }
        init_prompt_tokens.resize(std::max(0, need));
        params.prompt_tokens = init_prompt_tokens.data(); params.prompt_n_tokens = (int) init_prompt_tokens.size();
    }
    if (params.prompt_tokens && params.prompt_n_tokens > 0) {
        if (params.carry_initial_prompt) {
            if (past0.empty()) {
                const int max_tokens = std::max(1, max_prompt_ctx - 1);
                if (params.prompt_n_tokens > max_tokens)
                    logf(LOG_WARN, "%s: initial prompt is too long (%d tokens), will use only the last %d tokens\n", __func__, params.prompt_n_tokens, max_tokens);
                const int nt = std::min(params.prompt_n_tokens, max_tokens);
                past0.assign(params.prompt_tokens + (params.prompt_n_tokens - nt), params.prompt_tokens + params.prompt_n_tokens);
            }
        } else {
            for (int i = 0; i < params.prompt_n_tokens; ++i) past1.push_back(params.prompt_tokens[i]);
            std::rotate(past1.begin(), past1.end() - params.prompt_n_tokens, past1.end());
        }
    }

    if (params.audio_ctx > ctx->model.hp.n_audio_ctx) {
        logf(LOG_ERROR, "%s: audio_ctx is larger than the maximum allowed (%d > %d)\n", __func__, params.audio_ctx, ctx->model.hp.n_audio_ctx);
        return -5;
    }
    state->exp_n_audio_ctx = params.audio_ctx;

    std::vector<whisper_token> prompt_init = { vocab.token_sot };
    if (vocab.is_multilingual()) {
        const int lang_id = whisper_lang_id(params.language);
        state->lang_id = lang_id;
        prompt_init.push_back(vocab.token_sot + 1 + lang_id);
        prompt_init.push_back(params.translate ? vocab.token_translate : vocab.token_transcribe);
    }
    {
        const bool is_distil = ctx->model.hp.n_text_layer == 2 && ctx->model.hp.n_vocab != 51866;
        if (is_distil && !params.no_timestamps) {
            logf(LOG_WARN, "%s: using first release distilled models - forcing no_timestamps\n", __func__);
            params.no_timestamps = true;
        }
    }
    if (params.no_timestamps) prompt_init.push_back(vocab.token_not);

    int seek = seek_start;
    std::vector<whisper_token> prompt; prompt.reserve(n_text_ctx);

    // on-device logits filter + greedy pick (decode results come back as 32 bytes per sequence instead of n_vocab floats);
    // used whenever the step is a pure argmax: greedy strategy at temperature 0 without a user logits callback
    const bool dev_any_ok = !params.logits_filter_callback && !(params.grammar_rules && params.n_grammar_rules > 0) && getenv("WB200_HOST_SAMPLER") == nullptr;
    const bool dev_samp_ok = dev_any_ok && params.strategy == WHISPER_SAMPLING_GREEDY;
    // beam search at temperature 0: filter + the k categorical draws per decoder on the device (k candidates come back instead of n_vocab floats)
    const bool dev_beam_ok = dev_any_ok && params.strategy == WHISPER_SAMPLING_BEAM_SEARCH && params.beam_search.beam_size >= 1 &&
                             params.beam_search.beam_size * n_decoders <= SAMP_MAX_DRAWS && getenv("WB200_HOST_BEAM") == nullptr;
    std::vector<uint32_t> mask_bits; SampReq sreq; std::vector<int> rowinfo; std::vector<double> draws;
    if (dev_samp_ok || dev_beam_ok) {
        build_static_mask(*ctx, params, mask_bits, sreq.mask_key);
        sreq.mask_bits = &mask_bits;
        make_samp_cfg(*ctx, params, sreq.cfg);
    }

    // run-ahead (SampReq::next_step): whether step i of the loop below submits a decode for `d` when the token it samples is a text token
    // (neither end-of-text nor a timestamp): not if max_tokens, the loop or the end of the audio ends the sequence there, or its last
    // step fails it
    const int n_max_steps = n_text_ctx / 2 - 4;
    auto step_follows = [&](const Decoder & d, int i) {
        if (i >= n_max_steps || (params.max_tokens > 0 && i >= params.max_tokens) || (d.has_ts && seek + d.seek_delta + delta_min >= seek_end)) return false;
        return i < n_max_steps - 1 || (d.sequence.result_len != 0 && d.seek_delta >= 100 * WB_CHUNK_SIZE / 2);
    };
    struct BeamCand { int decoder_idx; int seek_delta; bool has_ts; Sequence sequence; Grammar grammar; };
    std::vector<std::vector<BeamCand>> bc_per_dec(n_decoders);
    std::vector<BeamCand> cands;
    std::vector<int> b_tok, b_pos, b_seq; std::vector<int8_t> b_want;

    while (true) {
        if (params.progress_callback)
            params.progress_callback(ctx, state, (100 * (seek - seek_start)) / (seek_end - seek_start), params.progress_callback_user_data);
        if (seek + delta_min >= seek_end) break;
        if (params.encoder_begin_callback && !params.encoder_begin_callback(ctx, state, params.encoder_begin_callback_user_data)) {
            logf(LOG_ERROR, "%s: encoder_begin_callback returned false - aborting\n", __func__);
            break;
        }
        if (!encode_window(*ctx, *state, seek)) { logf(LOG_ERROR, "%s: failed to encode\n", __func__); return -6; }
        if (params.abort_callback && params.abort_callback(params.abort_callback_user_data)) { logf(LOG_ERROR, "%s: failed to encode\n", __func__); return -6; }

        if (seek > seek_start && seek + 500 >= seek_end) { past0.clear(); past1.clear(); }

        int best_decoder_id = 0;
        for (int it = 0; it < (int) temperatures.size(); ++it) {
            const float t_cur = temperatures[it];
            int n_cur = 1;
            if (params.strategy == WHISPER_SAMPLING_GREEDY) { if (t_cur > 0.0f) n_cur = params.greedy.best_of; }
            else if (params.strategy == WHISPER_SAMPLING_BEAM_SEARCH) n_cur = t_cur > 0.0f ? params.greedy.best_of : params.beam_search.beam_size;
            n_cur = std::max(1, n_cur);

            for (int j = 0; j < n_cur; ++j) {
                Decoder & d = state->decoders[j];
                d.sequence.tokens.clear(); d.sequence.result_len = 0; d.sequence.sum_logprobs_all = 0.0;
                d.sequence.sum_logprobs = -INFINITY; d.sequence.avg_logprobs = -INFINITY; d.sequence.entropy = 0.0; d.sequence.score = -INFINITY;
                d.seek_delta = 100 * WB_CHUNK_SIZE;
                d.failed = d.completed = d.has_ts = false;
                d.grammar = params.grammar_rules ? grammar_init(params.grammar_rules, params.n_grammar_rules, params.i_start_rule) : Grammar();   // whisper.cpp:7117-7121
            }

            { // prompt + KV cache for this attempt (whisper.cpp:7126-7221)
                prompt.clear();
                if (params.n_max_text_ctx > 0 && t_cur < 0.5f) {
                    const bool take0 = params.carry_initial_prompt && !past0.empty();
                    const bool take1 = !past1.empty();
                    if (max_prompt_ctx > 0 && (take0 || take1)) {
                        prompt.push_back(vocab.token_prev);
                        int n0 = 0;
                        if (take0) { n0 = (int) past0.size(); prompt.insert(prompt.end(), past0.end() - n0, past0.end()); }
                        const int n1 = std::min<int>(max_prompt_ctx - n0 - 1, (int) past1.size());
                        prompt.insert(prompt.end(), past1.end() - n1, past1.end());
                    }
                }
                prompt.insert(prompt.end(), prompt_init.begin(), prompt_init.end());

                if (state->kv_self_n_dec < n_cur) {
                    const int factor = n_cur > 1 ? n_cur + 2 : 1;
                    const int cells = ((n_text_ctx + 255) / 256 * 256) * factor;
                    if (state->group) {                                                // pool state: more cells per slot (contents of all slots preserved)
                        if (!state->group->ensure_cells(state, cells)) { logf(LOG_ERROR, "%s: KV cache allocation failed: %s\n", __func__, last_error()); return -7; }
                    } else {
                        if (!(state->scripted || state->eng->set_cells(cells))) { logf(LOG_ERROR, "%s: KV cache allocation failed\n", __func__); return -7; }
                        state->kv.reset((uint32_t) cells);
                    }
                    state->kv_self_n_dec = n_cur;
                }
                state->kv.clear();

                const int np = (int) prompt.size();
                b_tok.assign(prompt.begin(), prompt.end()); b_pos.resize(np); b_seq.assign(np, 0); b_want.assign(np, 0);
                for (int i = 0; i < np; ++i) b_pos[i] = i;
                b_want[np - 1] = 1;
                const bool dev_beam = dev_beam_ok && t_cur < 1e-6f;
                const bool dev_samp = (dev_samp_ok && t_cur < 1e-6f) || dev_beam;
                const int bk = params.beam_search.beam_size;
                for (int j = 0; j < n_cur; ++j) { Decoder & d = state->decoders[j]; d.have_pending = false; d.have_pending_k = false; d.predrawn.clear(); }
                sreq.draws = nullptr; sreq.stride = 1;
                if (dev_samp) { rowinfo.assign((size_t) 2 * np, 0); samp_rowinfo(vocab, params, state->decoders[0], &rowinfo[2 * (np - 1)]); sreq.rowinfo = rowinfo.data(); }
                sreq.next_step = dev_samp && !dev_beam && n_cur == 1 && step_follows(state->decoders[0], 0);      // step 0 of the loop below
                if (sreq.next_step) samp_rowinfo_next(vocab, params, state->decoders[0], sreq.next_rowinfo);
                if (dev_beam) {      // every decoder draws its k candidates from the distribution of the prompt's last row, each with its own generator (whisper.cpp:7212-7221, 7270-7290)
                    const int nd = n_cur * bk;
                    draws.assign((size_t) np * nd, 0.0);
                    for (int j = 0; j < n_cur; ++j) for (int q = 0; q < bk; ++q) {
                        const double u = std::generate_canonical<double, std::numeric_limits<double>::digits>(state->decoders[j].rng);
                        draws[(size_t) (np - 1) * nd + j * bk + q] = u; state->decoders[j].predrawn.push_back(u);
                    }
                    rowinfo[2 * (np - 1)] |= nd << 8;
                    sreq.draws = draws.data(); sreq.stride = nd;
                }
                if (!decode_batch(*ctx, *state, b_tok.data(), b_pos.data(), b_seq.data(), b_want.data(), np, dev_samp ? &sreq : nullptr)) { logf(LOG_ERROR, "%s: failed to decode\n", __func__); return -8; }
                if (params.abort_callback && params.abort_callback(params.abort_callback_user_data)) return -8;

                // no_speech probability (whisper.cpp:7190-7200).  The reference takes it from ROW 0 of state->logits, a buffer in which a
                // decode only refreshes the rows it was asked logits for (whisper.cpp:2957-2963): for a one-token prompt that is the SOT
                // row of this decode; for longer prompts (language / task tokens, previous context) it is whatever the last decode with a
                // flagged row 0 left there -- the last single-token step of the previous window, or zeros on a fresh state (p = 1/n_vocab).
                // row0_nosp() follows exactly that rule on both the host-logits and the device-sampler path.
                state->no_speech_prob = row0_nosp(*ctx, *state);
                if (!state->samp_out.empty() && dev_beam) {     // the device already filtered and drew: k candidates per decoder
                    const int nd = n_cur * bk;
                    for (int j = 0; j < n_cur; ++j) {
                        Decoder & d = state->decoders[j];
                        d.pending_k.clear();
                        for (int q = 0; q < bk; ++q) d.pending_k.push_back(from_samp(state->samp_out[(size_t) (np - 1) * nd + j * bk + q]));
                        d.have_pending_k = true; d.predrawn.clear();
                        if (j > 0) state->kv.seq_cp(0, j, -1, -1);
                    }
                } else if (!state->samp_out.empty()) {      // the device already filtered and picked
                    state->decoders[0].pending = from_samp(state->samp_out[(size_t) (np - 1) * state->samp_stride]);
                    state->decoders[0].have_pending = true;
                }
                if (state->samp_out.empty()) {
                    const int64_t ts = time_us();
                    state->decoders[0].i_batch = np - 1;
                    process_logits(*ctx, *state, state->decoders[0], params, t_cur);
                    for (int j = 1; j < n_cur; ++j) {
                        Decoder & d = state->decoders[j];
                        state->kv.seq_cp(0, j, -1, -1);
                        d.probs = state->decoders[0].probs; d.logits = state->decoders[0].logits; d.logprobs = state->decoders[0].logprobs;
                    }
                    state->t_sample_us += time_us() - ts;
                }
            }

            for (int i = 0, n_max = n_text_ctx / 2 - 4; i < n_max; ++i) {
                const int64_t ts0 = time_us();
                if (params.strategy == WHISPER_SAMPLING_BEAM_SEARCH) for (auto & bc : bc_per_dec) bc.clear();

                { // sampling
                    std::atomic<int> j_cur(0);
                    auto work = [&]() {
                        for (;;) {
                            const int j = j_cur.fetch_add(1);
                            if (j >= n_cur) break;
                            Decoder & d = state->decoders[j];
                            if (d.completed || d.failed) continue;
                            if (params.strategy == WHISPER_SAMPLING_GREEDY) {
                                if (d.have_pending) { d.sequence.tokens.push_back(d.pending); d.have_pending = false; }
                                else d.sequence.tokens.push_back(sample_token(*ctx, d, t_cur < 1e-6f));
                                d.sequence.sum_logprobs_all += d.sequence.tokens.back().plog;
                            } else {
                                std::vector<whisper_token_data> toks;
                                if (d.have_pending_k) { toks.swap(d.pending_k); d.have_pending_k = false; }
                                else if ((int) d.predrawn.size() >= params.beam_search.beam_size) toks = sample_token_topk_u(*ctx, d, params.beam_search.beam_size, d.predrawn.data());
                                else toks = sample_token_topk(*ctx, d, params.beam_search.beam_size);
                                d.predrawn.clear();
                                for (const auto & tk : toks) {
                                    bc_per_dec[j].push_back({ j, d.seek_delta, d.has_ts, d.sequence, d.grammar });
                                    bc_per_dec[j].back().sequence.tokens.push_back(tk);
                                    bc_per_dec[j].back().sequence.sum_logprobs_all += tk.plog;
                                }
                            }
                        }
                    };
                    run_parallel(std::min(params.n_threads, n_cur), work);
                }
                cands.clear();
                for (const auto & bc : bc_per_dec) { cands.insert(cands.end(), bc.begin(), bc.end()); if (!bc.empty()) state->n_sample += 1; }

                if (params.strategy == WHISPER_SAMPLING_BEAM_SEARCH) {                 // whisper.cpp:7305-7357
                    std::sort(cands.begin(), cands.end(), [](const BeamCand & a, const BeamCand & b) {
                        if (a.sequence.sum_logprobs_all != b.sequence.sum_logprobs_all) return a.sequence.sum_logprobs_all > b.sequence.sum_logprobs_all;
                        return a.decoder_idx < b.decoder_idx;
                    });
                    uint32_t cur_c = 0;
                    for (int j = 0; j < n_cur; ++j) {
                        Decoder & d = state->decoders[j];
                        if (d.completed || d.failed) continue;
                        if (cur_c >= cands.size()) cur_c = 0;
                        BeamCand & c = cands[cur_c++];
                        while (cands.size() > cur_c && tokens_equal(cands[cur_c].sequence, c.sequence) && i > 0) ++cur_c;
                        d.seek_delta = c.seek_delta; d.has_ts = c.has_ts; d.sequence = c.sequence; d.grammar = c.grammar;
                        state->kv.seq_cp(c.decoder_idx, MAX_DECODERS + j, -1, -1);
                    }
                    for (int j = 0; j < n_cur; ++j) {
                        Decoder & d = state->decoders[j];
                        if (d.completed || d.failed) continue;
                        state->kv.seq_rm(j, -1, -1);
                        state->kv.seq_cp(MAX_DECODERS + j, j, -1, -1);
                        state->kv.seq_rm(MAX_DECODERS + j, -1, -1);
                    }
                }

                for (int j = 0; j < n_cur; ++j) {                                     // whisper.cpp:7363-7445
                    Decoder & d = state->decoders[j];
                    if (d.completed || d.failed) continue;
                    int & result_len = d.sequence.result_len;
                    {
                        const whisper_token_data & tk = d.sequence.tokens.back();
                        if (tk.id > vocab.token_beg) {
                            const int sd_new = 2 * (tk.id - vocab.token_beg);
                            if (d.has_ts && d.seek_delta > sd_new && result_len < i) { d.failed = true; continue; }
                            d.seek_delta = sd_new; result_len = i + 1; d.has_ts = true;
                        }
                        grammar_accept_token(vocab, d.grammar, tk.id);       // whisper.cpp:7395
                        if (tk.id == vocab.token_eot || (params.max_tokens > 0 && i >= params.max_tokens) ||
                            (d.has_ts && seek + d.seek_delta + delta_min >= seek_end)) {
                            if (result_len == 0 && !params.no_timestamps) {
                                if (seek + d.seek_delta + delta_min >= seek_end) result_len = i + 1;
                                else { d.failed = true; continue; }
                            }
                            if (params.single_segment || params.no_timestamps) { result_len = i + 1; d.seek_delta = 100 * WB_CHUNK_SIZE; }
                            d.completed = true;
                            continue;
                        }
                        if (ctx->model.n_loaded == 0) { d.seek_delta = 100 * WB_CHUNK_SIZE; d.completed = true; continue; }   // weight-less test stubs
                    }
                    if (i == n_max - 1 && (result_len == 0 || d.seek_delta < 100 * WB_CHUNK_SIZE / 2)) { d.failed = true; continue; }
                }
                {
                    bool all_done = true;
                    for (int j = 0; j < n_cur; ++j) { const Decoder & d = state->decoders[j]; if (!(d.completed || d.failed)) all_done = false; }
                    if (all_done) break;
                }
                state->t_sample_us += time_us() - ts0;

                { // next-token logits for every live decoder (whisper.cpp:7469-7546)
                    b_tok.clear(); b_pos.clear(); b_seq.clear(); b_want.clear();
                    const int n_past = (int) prompt.size() + i;
                    for (int j = 0; j < n_cur; ++j) {
                        Decoder & d = state->decoders[j];
                        if (d.failed || d.completed) continue;
                        d.i_batch = (int) b_tok.size();
                        b_tok.push_back(d.sequence.tokens.back().id); b_pos.push_back(n_past); b_seq.push_back(j); b_want.push_back(1);
                    }
                    const bool dev_beam = dev_beam_ok && t_cur < 1e-6f && i + 1 < n_max;      // (after the last step nothing is sampled from these logits)
                    const bool dev_samp = (dev_samp_ok && t_cur < 1e-6f) || dev_beam;
                    const int bk = params.beam_search.beam_size;
                    sreq.draws = nullptr; sreq.stride = 1;
                    if (dev_samp) {
                        rowinfo.assign(2 * b_tok.size(), 0);
                        for (int j = 0; j < n_cur; ++j) { const Decoder & d = state->decoders[j]; if (!(d.failed || d.completed)) samp_rowinfo(vocab, params, d, &rowinfo[2 * d.i_batch]); }
                        sreq.rowinfo = rowinfo.data();
                    }
                    sreq.next_step = dev_samp && !dev_beam && n_cur == 1 && step_follows(state->decoders[0], i + 1);
                    if (sreq.next_step) samp_rowinfo_next(vocab, params, state->decoders[0], sreq.next_rowinfo);
                    if (dev_beam) {
                        draws.assign(b_tok.size() * (size_t) bk, 0.0);
                        for (int j = 0; j < n_cur; ++j) {
                            Decoder & d = state->decoders[j];
                            if (d.failed || d.completed) continue;
                            d.predrawn.clear();
                            for (int q = 0; q < bk; ++q) {
                                const double u = std::generate_canonical<double, std::numeric_limits<double>::digits>(d.rng);
                                draws[(size_t) d.i_batch * bk + q] = u; d.predrawn.push_back(u);
                            }
                            rowinfo[2 * d.i_batch] |= bk << 8;
                        }
                        sreq.draws = draws.data(); sreq.stride = bk;
                    }
                    if (!decode_batch(*ctx, *state, b_tok.data(), b_pos.data(), b_seq.data(), b_want.data(), (int) b_tok.size(), dev_samp ? &sreq : nullptr)) {
                        logf(LOG_ERROR, "%s: failed to decode\n", __func__); return -9;
                    }
                    if (params.abort_callback && params.abort_callback(params.abort_callback_user_data)) return -9;
                    if (!state->samp_out.empty()) {
                        for (int j = 0; j < n_cur; ++j) {
                            Decoder & d = state->decoders[j];
                            if (d.failed || d.completed) continue;
                            if (dev_beam) {
                                d.pending_k.clear();
                                for (int q = 0; q < bk; ++q) d.pending_k.push_back(from_samp(state->samp_out[(size_t) d.i_batch * state->samp_stride + q]));
                                d.have_pending_k = true; d.predrawn.clear();
                            } else { d.pending = from_samp(state->samp_out[(size_t) d.i_batch * state->samp_stride]); d.have_pending = true; }
                        }
                        continue;
                    }
                    const int64_t ts1 = time_us();
                    std::atomic<int> j_cur(0);
                    auto work = [&]() {
                        for (;;) {
                            const int j = j_cur.fetch_add(1);
                            if (j >= n_cur) break;
                            Decoder & d = state->decoders[j];
                            if (d.failed || d.completed) continue;
                            process_logits(*ctx, *state, d, params, t_cur);
                        }
                    };
                    run_parallel(std::min(params.n_threads, n_cur), work);
                    state->t_sample_us += time_us() - ts1;
                }
            }

            { // rank the sequences (whisper.cpp:7549-7583)
                double best_score = -INFINITY;
                for (int j = 0; j < n_cur; ++j) {
                    Decoder & d = state->decoders[j];
                    if (d.failed) continue;
                    d.sequence.tokens.resize(d.sequence.result_len);
                    sequence_score(params, d.sequence);
                    if (d.sequence.result_len > 32 && d.sequence.entropy < params.entropy_thold) { d.failed = true; state->n_fail_h++; continue; }
                    if (best_score < d.sequence.score) { best_score = d.sequence.score; best_decoder_id = j; }
                }
            }
            bool success = true;
            if (it != (int) temperatures.size() - 1) {
                const Decoder & d = state->decoders[best_decoder_id];
                if (d.failed || (d.sequence.avg_logprobs < params.logprob_thold && state->no_speech_prob < params.no_speech_thold)) { success = false; state->n_fail_p++; }
            }
            if (success) break;
        }

        { // emit segments (whisper.cpp:7612-7784)
            const size_t n_segments_before = result_all.size();
            const Decoder & best = state->decoders[best_decoder_id];
            int seek_delta = best.seek_delta;
            const int result_len = best.sequence.result_len;
            const auto & cur = best.sequence.tokens;
            const bool is_no_speech = state->no_speech_prob > params.no_speech_thold && best.sequence.avg_logprobs < params.logprob_thold;

            past1.clear();
            if (!params.carry_initial_prompt && !prompt.empty() && prompt.front() == vocab.token_prev)
                past1.insert(past1.end(), prompt.begin() + 1, prompt.end() - prompt_init.size());
            if (!is_no_speech) for (int i = 0; i < result_len; ++i) past1.push_back(cur[i].id);

            if (!cur.empty() && ctx->model.n_loaded > 0 && !is_no_speech) {
                int i0 = 0;
                int64_t t0 = seek + 2 * (cur.front().tid - vocab.token_beg);
                std::string text; bool speaker_turn_next = false;
                auto push_segment = [&](int64_t a, int64_t b, int from, int to_incl) {
                    if (params.print_realtime) {
                        if (params.print_timestamps) printf("[%s --> %s]  %s\n", to_timestamp(a).c_str(), to_timestamp(b).c_str(), text.c_str());
                        else printf("%s", text.c_str());
                        fflush(stdout);
                    }
                    Segment sg; sg.t0 = a; sg.t1 = b; sg.text = text; sg.no_speech_prob = state->no_speech_prob; sg.speaker_turn_next = speaker_turn_next;
                    for (int j = from; j <= to_incl; ++j) sg.tokens.push_back(cur[j]);
                    result_all.push_back(std::move(sg));
                    int n_new = 1;
                    if (params.token_timestamps) {               // whisper.cpp:7688-7695
                        token_level_timestamps(*ctx, *state, (int) result_all.size() - 1, params.thold_pt, params.thold_ptsum);
                        if (params.max_len > 0) n_new = wrap_segment(*ctx, *state, params.max_len, params.split_on_word);
                    }
                    if (params.new_segment_callback && !ctx->params.dtw_token_timestamps) params.new_segment_callback(ctx, state, n_new, params.new_segment_callback_user_data);
                };
                for (int i = 0; i < (int) cur.size(); ++i) {
                    if (params.print_special || cur[i].id < vocab.token_eot) text += whisper_token_to_str(ctx, cur[i].id);
                    if (params.tdrz_enable && cur[i].id == vocab.token_solm) speaker_turn_next = true;
                    if (cur[i].id > vocab.token_beg && !params.single_segment) {
                        const int64_t t1 = seek + 2 * (cur[i].tid - vocab.token_beg);
                        if (!text.empty()) push_segment(t0, t1, i0, i);
                        text.clear();
                        t0 = t1;
                        while (i + 1 < (int) cur.size() && cur[i + 1].id > vocab.token_beg) {
                            ++i;
                            if (params.print_special) text += whisper_token_to_str(ctx, cur[i].id);
                            t0 = seek + 2 * (cur[i].tid - vocab.token_beg);
                        }
                        i0 = i + 1;
                        speaker_turn_next = false;
                    }
                }
                if (!text.empty()) push_segment(t0, seek + seek_delta, i0, (int) cur.size() - 1);
            }

            // DTW token timestamps for the segments of this window (whisper.cpp:7750-7765, 9009-9160)
            if (ctx->params.dtw_token_timestamps && result_all.size() > n_segments_before) {
                const int n_segments = (int) (result_all.size() - n_segments_before);
                const int n_frames = std::min(std::min(WB_CHUNK_SIZE * 100, seek_delta), seek_end - seek);
                if (!dtw_window(*ctx, *state, params, (int) n_segments_before, n_segments, seek, n_frames)) { logf(LOG_ERROR, "%s: DTW pass failed: %s\n", __func__, last_error()); return -8; }
                if (params.new_segment_callback)                      // same (peculiar) range as the reference
                    for (int seg = (int) result_all.size() - n_segments; seg < n_segments; seg++) params.new_segment_callback(ctx, state, seg, params.new_segment_callback_user_data);
            }

            const bool max_tokens_ts_ending = params.max_tokens > 0 && !params.single_segment && cur.size() > (size_t) params.max_tokens;
            const bool single_ts_ending = cur.size() > 1 && !max_tokens_ts_ending &&
                cur[cur.size() - 2].id < vocab.token_beg && cur[cur.size() - 1].id > vocab.token_beg;
            if (single_ts_ending) seek_delta = std::min(seek_end - seek, WB_CHUNK_SIZE * 100);
            seek += seek_delta;
        }
    }
    return 0;
}

} // extern "C"

// params.vad: run the detector on the whole clip and keep only the speech (whisper_vad, src/whisper.cpp:6669-6829).  The
// network runs on the context's GPU; cutting the PCM is a host copy because the C ABI hands the samples over in host memory.
static bool vad_filter(whisper_context * ctx, whisper_state * st, const whisper_full_params & params, const float * samples, int n_samples,
                       std::vector<float> & filtered) {
    st->vad.table.clear(); st->vad.has_segments = false;
    if (!st->vad_context) {
        whisper_vad_context_params vp = whisper_vad_default_context_params();
        vp.gpu_device = ctx->params.gpu_device;
        whisper_vad_context * v = nullptr;
        if (ctx->scripted) {                                                            // engine-less test context: host-only VAD context
            std::ifstream fin(params.vad_model_path ? params.vad_model_path : "", std::ios::binary);
            whisper_model_loader loader = {};
            loader.context = &fin;
            loader.read  = [](void * c, void * out, size_t n) -> size_t { auto * f = (std::ifstream *) c; f->read((char *) out, (std::streamsize) n); return (size_t) f->gcount(); };
            loader.eof   = [](void * c) -> bool { return ((std::ifstream *) c)->eof(); };
            loader.close = [](void *) {};
            if (fin) v = vad_load(&loader, -1);
        } else
        v = whisper_vad_init_from_file_with_params(params.vad_model_path, vp);
        if (!v) { logf(LOG_ERROR, "%s: failed to initialize VAD context\n", __func__); return false; }
        st->vad_context.reset(v);
    }
    whisper_vad_segments * segs = whisper_vad_segments_from_samples(st->vad_context.get(), params.vad_params, samples, n_samples);
    if (!segs) return false;
    if (!segs->data.empty()) {
        logf(LOG_INFO, "%s: detected %d speech segments\n", __func__, (int) segs->data.size());
        try { vad_cut_samples(segs->data, params.vad_params, samples, n_samples, filtered, st->vad); }
        catch (...) { whisper_vad_free_segments(segs); logf(LOG_ERROR, "%s: failed to allocate memory for filtered samples\n", __func__); return false; }
    }
    whisper_vad_free_segments(segs);
    return true;
}

extern "C" {

WB_EXPORT int whisper_full(struct whisper_context * ctx, struct whisper_full_params params, const float * samples, int n_samples) {
    if (!ctx || !ctx->state) return -1;
    std::vector<float> speech;
    if (params.vad) {                                                                      // whisper.cpp:7796-7809
        logf(LOG_INFO, "%s: VAD is enabled, processing speech segments only\n", __func__);
        if (!vad_filter(ctx, ctx->state, params, samples, n_samples, speech)) { logf(LOG_ERROR, "%s: failed to compute VAD\n", __func__); return -1; }
        if (speech.empty()) { ctx->state->result_all.clear(); return 0; }
        samples = speech.data(); n_samples = (int) speech.size();
    }
    return whisper_full_with_state(ctx, ctx->state, params, samples, n_samples);
}

WB_EXPORT int whisper_full_parallel(struct whisper_context * ctx, struct whisper_full_params params, const float * samples, int n_samples, int n_processors) {
    if (n_processors <= 1) return whisper_full(ctx, params, samples, n_samples);          // whisper.cpp:7813-7941
    if (!ctx || !ctx->state) return -1;
    std::vector<float> speech;
    if (params.vad) {                                                                      // whisper.cpp:7824-7836
        logf(LOG_INFO, "%s: VAD is enabled, processing speech segments only\n", __func__);
        if (!vad_filter(ctx, ctx->state, params, samples, n_samples, speech)) { logf(LOG_ERROR, "%s: failed to compute VAD\n", __func__); return -1; }
        if (speech.empty()) return 0;
        samples = speech.data(); n_samples = (int) speech.size();
    }
    int ret = 0;
    std::vector<whisper_state *> states;
    const int offset_samples = (WB_SAMPLE_RATE * params.offset_ms) / 1000;
    const int per = (n_samples - offset_samples) / n_processors;
    std::vector<std::thread> workers(n_processors - 1);
    std::vector<int> rets(n_processors - 1, 0);
    for (int i = 0; i < n_processors - 1; ++i) {                                          // whisper.cpp:7848-7852: one new state per extra processor
        states.push_back(whisper_init_state(ctx));
        if (!states.back()) { states.pop_back(); for (whisper_state * s : states) whisper_free_state(s); return -7; }
    }
    // The states of one context advance in lock-step (wb_state.h).  All of them join the rendezvous BEFORE the first thread starts, so the
    // very first pass already carries every processor's window; each one leaves as soon as its own slice is done.
    whisper_state * main_state = ctx->state;
    if (main_state->group) main_state->group->enter(main_state);
    for (whisper_state * s : states) if (s->group) s->group->enter(s);
    for (int i = 0; i < n_processors - 1; ++i) {
        const int start = offset_samples + (i + 1) * per;
        const int n_cur = (i == n_processors - 2) ? n_samples - start : per;
        whisper_full_params pc = params;
        pc.offset_ms = 0; pc.print_progress = false; pc.print_realtime = false;
        pc.new_segment_callback = nullptr; pc.new_segment_callback_user_data = nullptr;
        pc.progress_callback = nullptr; pc.progress_callback_user_data = nullptr;
        whisper_state * s = states[i]; int * r = &rets[i];
        workers[i] = std::thread([ctx, s, pc, samples, start, n_cur, r]() {
            *r = whisper_full_with_state(ctx, s, pc, samples + start, n_cur);
            if (s->group) s->group->leave(s);
        });
    }
    {
        whisper_full_params pc = params; pc.print_realtime = false;
        ret = whisper_full_with_state(ctx, ctx->state, pc, samples, offset_samples + per);
        if (main_state->group) main_state->group->leave(main_state);
    }
    for (auto & w : workers) w.join();
    const int64_t offset_t = (int64_t) (params.offset_ms / 10.0);
    whisper_state * main = ctx->state;
    for (int i = 0; i < n_processors - 1; ++i) {
        for (auto & r : states[i]->result_all) {
            const int64_t shift = 100 * ((int64_t) (i + 1) * per) / WB_SAMPLE_RATE + offset_t;
            r.t0 += shift; r.t1 += shift;
            if (!main->result_all.empty()) r.t0 = std::max(r.t0, main->result_all.back().t1);
            main->result_all.push_back(std::move(r));
            if (params.new_segment_callback) params.new_segment_callback(ctx, main, 1, params.new_segment_callback_user_data);
        }
        main->t_mel_us += states[i]->t_mel_us; main->t_sample_us += states[i]->t_sample_us; main->t_encode_us += states[i]->t_encode_us;
        main->t_decode_us += states[i]->t_decode_us; main->t_batchd_us += states[i]->t_batchd_us; main->t_prompt_us += states[i]->t_prompt_us;
        main->n_sample += states[i]->n_sample; main->n_encode += states[i]->n_encode; main->n_decode += states[i]->n_decode;
        main->n_batchd += states[i]->n_batchd; main->n_prompt += states[i]->n_prompt;
        if (rets[i] != 0 && ret == 0) ret = rets[i];
        whisper_free_state(states[i]);
    }
    main->t_mel_us /= n_processors; main->t_sample_us /= n_processors; main->t_encode_us /= n_processors; main->t_decode_us /= n_processors;
    logf(LOG_WARN, "\n%s: the audio has been split into %d chunks at the following times:\n", __func__, n_processors);
    for (int i = 0; i < n_processors - 1; ++i)
        logf(LOG_WARN, "%s: split %d - %s\n", __func__, i + 1, to_timestamp(100 * ((int64_t) (i + 1) * per) / WB_SAMPLE_RATE + offset_t).c_str());
    logf(LOG_WARN, "%s: the transcription quality may be degraded near these boundaries\n", __func__);
    return ret;
}

// Convenience driver on top of the context's pool: independent PCM buffers, a queue of chunks served by up to 64 pool states that
// call whisper_full_with_state concurrently (the same lock-step passes any concurrent whisper.h callers get).  Chunk i's
// segments are returned in states_out[i] (result-only states; free with whisper_free_state).  Chunk semantics are those
// of whisper_full_with_state.  flags bit 0: `samples[i]` are DEVICE pointers (PCM already resident in HBM).
WB_EXPORT int wb200_full_batch_ex(struct whisper_context * ctx, struct whisper_full_params params, const float * const * samples,
                                  const int * n_samples, int n_chunks, struct whisper_state ** states_out, int flags) {
    if (!ctx || !samples || !n_samples || !states_out || n_chunks <= 0) return -1;
    if ((flags & 1) && !ctx->replicas.empty()) { set_error("wb200_full_batch: device-pointer input needs a single-GPU context (WB200_DEVICES is set)"); logf(LOG_ERROR, "%s: %s\n", __func__, last_error()); return -1; }
    if (params.vad) { set_error("wb200_full_batch: params.vad is not applied to pre-cut chunks; run whisper_vad_* first"); logf(LOG_ERROR, "%s: %s\n", __func__, last_error()); return -1; }
    int S = ctx->model.dec_tm ? 64 : 8;          // concurrent sequences: one row each in the decode pass (64 rows per launch of the persistent kernel)
    if (const char * e = getenv("WB200_BATCH_MEMBERS")) S = std::max(1, std::min(64, atoi(e)));
    S = std::min(S, n_chunks);
    // the members are ordinary states of the context's pool (whisper_init_state): slots and front ends are recycled, so this is cheap
    std::vector<whisper_state *> members;
    for (int i = 0; i < S; ++i) {
        whisper_state * st = whisper_init_state(ctx);
        if (!st) { for (whisper_state * m : members) whisper_free_state(m); return -7; }
        members.push_back(st);
    }
    for (whisper_state * st : members) if (st->group) st->group->enter(st);      // all of them before the first request (see whisper_full_parallel)
    std::atomic<int> next(0); std::atomic<int> rc(0);
    whisper_full_params pc = params;
    pc.print_progress = false; pc.print_realtime = false;
    std::vector<std::thread> th;
    for (int mi = 0; mi < S; ++mi) {
        th.emplace_back([&, mi]() {
            whisper_state * st = members[mi];
            for (;;) {
                const int i = next.fetch_add(1);
                if (i >= n_chunks) break;
                // a chunk starts from what a fresh state would hold
                st->decoders[0].rng = std::mt19937(0);
                st->prompt_past0.clear(); st->prompt_past1.clear();
                st->t_beg = st->t_last = 0; st->tid_last = 0; st->energy.clear(); st->no_speech_prob = 0.0f;
                st->logits.clear(); st->lrows.clear(); st->row0_is_copy = false; st->lang_id = 0;
                st->t_sample_us = st->t_encode_us = st->t_decode_us = st->t_batchd_us = st->t_prompt_us = st->t_mel_us = 0;
                st->n_sample = st->n_encode = st->n_decode = st->n_batchd = st->n_prompt = st->n_fail_p = st->n_fail_h = 0;
                wb::tls_pcm_is_device() = (flags & 1) != 0;
                const int r = whisper_full_with_state(ctx, st, pc, samples[i], n_samples[i]);
                wb::tls_pcm_is_device() = false;
                if (r != 0) rc.store(r);
                whisper_state * out = new whisper_state();          // result-only
                out->result_all = std::move(st->result_all); st->result_all.clear();
                out->lang_id = st->lang_id;
                out->t_sample_us = st->t_sample_us; out->t_encode_us = st->t_encode_us; out->t_decode_us = st->t_decode_us;
                out->t_batchd_us = st->t_batchd_us; out->t_prompt_us = st->t_prompt_us; out->t_mel_us = st->t_mel_us;
                out->n_sample = st->n_sample; out->n_encode = st->n_encode; out->n_decode = st->n_decode; out->n_batchd = st->n_batchd; out->n_prompt = st->n_prompt;
                states_out[i] = out;
            }
            if (st->group) st->group->leave(st);
        });
    }
    for (auto & t : th) t.join();
    for (whisper_state * m : members) whisper_free_state(m);
    return rc.load();
}
// Host-only test hook (no CUDA): the logits filter + greedy pick of this library on injected logits, with the vocabulary of
// `model_path`.  Same contract as the oracle's wref_process_logits (oracle/ref_harness.cpp), so the two can be compared bit for
// bit on a CPU-only box.  history: ids already in the decoder's sequence.  Returns 0, or -1 when the file cannot be parsed.
static whisper_context * dbg_vocab_ctx(const char * model_path) {       // header + vocabulary of a model file, no CUDA
    static std::mutex mu; static std::map<std::string, std::unique_ptr<whisper_context>> cache;
    std::lock_guard<std::mutex> lk(mu);
    auto & slot = cache[model_path];
    if (!slot) {
        std::ifstream fin(model_path, std::ios::binary);
        if (!fin) return nullptr;
        whisper_model_loader loader = {};
        loader.context = &fin;
        loader.read  = [](void * c, void * out, size_t n) -> size_t { auto * f = (std::ifstream *) c; f->read((char *) out, (std::streamsize) n); return (size_t) f->gcount(); };
        loader.eof   = [](void * c) -> bool { return ((std::ifstream *) c)->eof(); };
        loader.close = [](void * c) { ((std::ifstream *) c)->close(); };
        std::unique_ptr<whisper_context> c(new whisper_context());
        if (!wb::model_load(&loader, c->model, c->vocab, -1)) return nullptr;
        slot = std::move(c);
    }
    return slot.get();
}

// Host-only: a context that holds only the header + vocabulary of a model file (no CUDA, no weights, no state).  Valid for the
// vocabulary / tokenizer / special-token / model-shape getters of whisper.h; owned by the library.
WB_EXPORT struct whisper_context * wb200_dbg_vocab_context(const char * model_path) { return model_path ? dbg_vocab_ctx(model_path) : nullptr; }

// Host-only: an ENGINE-LESS context + state for tests/test_full_scripted_cpu.py.  whisper_full* run their complete control flow on it (seek
// loop, prompts, temperature fallback, beam search, segment emission, token timestamps, whisper_full_parallel) but every decode leaves zero
// logits: the transcript is scripted by the caller's logits_filter_callback, exactly as it can be scripted on the reference.  The caller
// owns the context (whisper_free).  Not reachable from whisper.h.
WB_EXPORT struct whisper_context * wb200_dbg_scripted_context(const char * model_path) {
    if (!model_path) return nullptr;
    std::ifstream fin(model_path, std::ios::binary);
    if (!fin) return nullptr;
    whisper_model_loader loader = {};
    loader.context = &fin;
    loader.read  = [](void * c, void * out, size_t n) -> size_t { auto * f = (std::ifstream *) c; f->read((char *) out, (std::streamsize) n); return (size_t) f->gcount(); };
    loader.eof   = [](void * c) -> bool { return ((std::ifstream *) c)->eof(); };
    loader.close = [](void * c) { ((std::ifstream *) c)->close(); };
    std::unique_ptr<whisper_context> c(new whisper_context());
    if (!wb::model_load(&loader, c->model, c->vocab, -1)) return nullptr;
    c->params = whisper_context_default_params();
    c->scripted = true;
    c->model.n_loaded = 1;                       // "has weights" as far as the segment emission of whisper_full is concerned (whisper.cpp:7635)
    c->state = whisper_init_state(c.get());
    return c->state ? c.release() : nullptr;
}

// The ON-DEVICE logits filter + greedy pick (k_greedy_sample) on injected logits: same inputs as wb200_dbg_process_logits at
// temperature 0; fills `sampled`.  Needs a CUDA device.
WB_EXPORT int wb200_dbg_greedy_sample(const char * model_path, const struct whisper_full_params * params, const whisper_token * history,
                                      int n_history, int has_ts, int seek_delta, const float * logits_in, whisper_token_data * sampled) {
    if (!model_path || !params || !logits_in || !sampled) return -1;
    whisper_context * pc = dbg_vocab_ctx(model_path);
    if (!pc) return -1;
    whisper_context & ctx = *pc;
    const int n = ctx.vocab.n_vocab;
    Decoder dec;
    for (int i = 0; i < n_history; ++i) { whisper_token_data td = blank_token(); td.id = history[i]; dec.sequence.tokens.push_back(td); }
    dec.has_ts = has_ts != 0; dec.seek_delta = seek_delta;
    std::vector<uint32_t> bits; uint64_t key = 0;
    build_static_mask(ctx, *params, bits, key);
    SampCfg cfg; make_samp_cfg(ctx, *params, cfg);
    int rowinfo[2]; samp_rowinfo(ctx.vocab, *params, dec, rowinfo);
    DevBuf<float> dl; DevBuf<uint32_t> dm; DevBuf<int> dr; DevBuf<SampOut> dout;
    if (!dl.alloc(n) || !dm.alloc(bits.size()) || !dr.alloc(2) || !dout.alloc(1)) return -2;
    SampOut o;
    if (cudaMemcpy(dl.p, logits_in, (size_t) n * 4, cudaMemcpyHostToDevice) != cudaSuccess || cudaMemcpy(dm.p, bits.data(), bits.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(dr.p, rowinfo, sizeof(rowinfo), cudaMemcpyHostToDevice) != cudaSuccess) return -2;
    cfg.mask = dm.p;
    greedy_sample(dl.p, n, 1, dr.p, cfg, dout.p, nullptr);
    if (cudaMemcpy(&o, dout.p, sizeof(o), cudaMemcpyDeviceToHost) != cudaSuccess) return -2;
    *sampled = from_samp(o);
    return 0;
}

WB_EXPORT int wb200_dbg_process_logits(const char * model_path, const struct whisper_full_params * params, const whisper_token * history,
                                       int n_history, int has_ts, int seek_delta, float temperature, const float * logits_in,
                                       float * logits_out, float * logprobs_out, float * probs_out, whisper_token_data * sampled) {
    if (!model_path || !params || !logits_in) return -1;
    whisper_context * pc = dbg_vocab_ctx(model_path);
    if (!pc) return -1;
    whisper_context & ctx = *pc;
    const int n = ctx.vocab.n_vocab;
    whisper_state st;
    Decoder & dec = st.decoders[0];
    for (int i = 0; i < n_history; ++i) { whisper_token_data td = blank_token(); td.id = history[i]; dec.sequence.tokens.push_back(td); }
    dec.has_ts = has_ts != 0; dec.seek_delta = seek_delta; dec.i_batch = 0;
    st.logits.assign(logits_in, logits_in + n);
    process_logits(ctx, st, dec, *params, temperature);
    if (logits_out)   memcpy(logits_out,   dec.logits.data(),   (size_t) n * sizeof(float));
    if (logprobs_out) memcpy(logprobs_out, dec.logprobs.data(), (size_t) n * sizeof(float));
    if (probs_out)    memcpy(probs_out,    dec.probs.data(),    (size_t) n * sizeof(float));
    if (sampled)      *sampled = sample_token(ctx, dec, true);
    return 0;
}

// Host-only: experimental token-level timestamps + max_len wrapping on an injected segment (same contract as the oracle's
// wref_token_timestamps) and the signal-energy envelope they use
WB_EXPORT int wb200_dbg_token_timestamps(const char * model_path, const int * ids, const int * tids, const float * pt, const float * ptsum, int n,
                                         int64_t seg_t0, int64_t seg_t1, const float * energy, int n_energy, float thold_pt, float thold_ptsum,
                                         int max_len, int split_on_word, int64_t * carry, int64_t * tok_out, float * vlen_out,
                                         int64_t * piece_out, int max_pieces) {
    whisper_context * pc = model_path ? dbg_vocab_ctx(model_path) : nullptr;
    if (!pc || !ids || !tids || !pt || !ptsum || !energy || !carry || !tok_out || !vlen_out || !piece_out) return -1;
    whisper_state st;
    st.energy.assign(energy, energy + n_energy);
    st.t_beg = carry[0]; st.t_last = carry[1]; st.tid_last = (whisper_token) carry[2];
    Segment seg; seg.t0 = seg_t0; seg.t1 = seg_t1;
    for (int i = 0; i < n; ++i) { whisper_token_data td = blank_token(); td.id = ids[i]; td.tid = tids[i]; td.pt = pt[i]; td.ptsum = ptsum[i]; seg.tokens.push_back(td); }
    st.result_all.push_back(seg);
    token_level_timestamps(*pc, st, 0, thold_pt, thold_ptsum);
    for (int i = 0; i < n; ++i) { tok_out[2 * i] = st.result_all[0].tokens[i].t0; tok_out[2 * i + 1] = st.result_all[0].tokens[i].t1; vlen_out[i] = st.result_all[0].tokens[i].vlen; }
    int pieces = 1;
    if (max_len > 0) pieces = wrap_segment(*pc, st, max_len, split_on_word != 0);
    for (int i = 0; i < (int) st.result_all.size() && i < max_pieces; ++i) {
        piece_out[3 * i] = st.result_all[i].t0; piece_out[3 * i + 1] = st.result_all[i].t1; piece_out[3 * i + 2] = (int64_t) st.result_all[i].tokens.size();
    }
    carry[0] = st.t_beg; carry[1] = st.t_last; carry[2] = st.tid_last;
    return pieces;
}
WB_EXPORT int wb200_dbg_signal_energy(const float * pcm, int n, int hw, float * out) {
    if (!pcm || !out || n < 0) return -1;
    const auto e = signal_energy(pcm, n, hw);
    memcpy(out, e.data(), (size_t) n * sizeof(float));
    return 0;
}

// Host-only: logits filter with a grammar; the parse state is built from params->grammar_rules and advanced over `accepted` first
// (same contract as the oracle's wref_process_logits_grammar)
WB_EXPORT int wb200_dbg_process_logits_grammar(const char * model_path, const struct whisper_full_params * params, const whisper_token * history,
                                               int n_history, int has_ts, int seek_delta, float temperature, const whisper_token * accepted, int n_accepted,
                                               const float * logits_in, float * logits_out, float * logprobs_out, float * probs_out,
                                               whisper_token_data * sampled, int * n_stacks_out) {
    if (!model_path || !params || !logits_in) return -1;
    whisper_context * pc = dbg_vocab_ctx(model_path);
    if (!pc) return -1;
    whisper_context & ctx = *pc;
    const int n = ctx.vocab.n_vocab;
    whisper_state st;
    Decoder & dec = st.decoders[0];
    for (int i = 0; i < n_history; ++i) { whisper_token_data td = blank_token(); td.id = history[i]; dec.sequence.tokens.push_back(td); }
    dec.has_ts = has_ts != 0; dec.seek_delta = seek_delta; dec.i_batch = 0;
    dec.grammar = grammar_init(params->grammar_rules, params->n_grammar_rules, params->i_start_rule);
    for (int i = 0; i < n_accepted; ++i) grammar_accept_token(ctx.vocab, dec.grammar, accepted[i]);
    if (n_stacks_out) *n_stacks_out = (int) dec.grammar.stacks.size();
    st.logits.assign(logits_in, logits_in + n);
    process_logits(ctx, st, dec, *params, temperature);
    if (logits_out)   memcpy(logits_out,   dec.logits.data(),   (size_t) n * sizeof(float));
    if (logprobs_out) memcpy(logprobs_out, dec.logprobs.data(), (size_t) n * sizeof(float));
    if (probs_out)    memcpy(probs_out,    dec.probs.data(),    (size_t) n * sizeof(float));
    if (sampled)      *sampled = sample_token(ctx, dec, true);
    return 0;
}

// Host-only: the k beam-search candidates (sample_token_topk) for the same inputs, decoder.rng = std::mt19937(seed)
WB_EXPORT int wb200_dbg_sample_topk(const char * model_path, const struct whisper_full_params * params, const whisper_token * history,
                                    int n_history, int has_ts, int seek_delta, float temperature, const float * logits_in, int k_in, int seed,
                                    whisper_token_data * out) {
    const int k = k_in < 0 ? -k_in : k_in;                                    // k < 0: uniforms drawn first, then sample_token_topk_u
    if (!model_path || !params || !logits_in || !out || k <= 0) return -1;
    whisper_context * pc = dbg_vocab_ctx(model_path);
    if (!pc) return -1;
    whisper_context & ctx = *pc;
    whisper_state st;
    Decoder & dec = st.decoders[0];
    for (int i = 0; i < n_history; ++i) { whisper_token_data td = blank_token(); td.id = history[i]; dec.sequence.tokens.push_back(td); }
    dec.has_ts = has_ts != 0; dec.seek_delta = seek_delta; dec.i_batch = 0;
    st.logits.assign(logits_in, logits_in + ctx.vocab.n_vocab);
    process_logits(ctx, st, dec, *params, temperature);
    dec.rng = std::mt19937(seed);
    if (k_in < 0) {                                                           // the path whisper_full takes when the uniforms were drawn ahead of the decode
        std::vector<double> u((size_t) k);
        for (double & v : u) v = std::generate_canonical<double, std::numeric_limits<double>::digits>(dec.rng);
        const auto r = sample_token_topk_u(ctx, dec, k, u.data());
        for (int i = 0; i < k; ++i) out[i] = r[i];
        return 0;
    }
    const auto r = sample_token_topk(ctx, dec, k);
    for (int i = 0; i < k; ++i) out[i] = r[i];
    return 0;
}

// The ON-DEVICE filter + k categorical draws (k_greedy_sample with draws) on injected logits, uniforms from std::mt19937(seed) as in
// whisper_full's beam search.  Needs a CUDA device.
WB_EXPORT int wb200_dbg_draw_sample(const char * model_path, const struct whisper_full_params * params, const whisper_token * history,
                                    int n_history, int has_ts, int seek_delta, const float * logits_in, int k, int seed, whisper_token_data * out) {
    if (!model_path || !params || !logits_in || !out || k <= 0 || k > SAMP_MAX_DRAWS) return -1;
    whisper_context * pc = dbg_vocab_ctx(model_path);
    if (!pc) return -1;
    whisper_context & ctx = *pc;
    const int n = ctx.vocab.n_vocab;
    Decoder dec;
    for (int i = 0; i < n_history; ++i) { whisper_token_data td = blank_token(); td.id = history[i]; dec.sequence.tokens.push_back(td); }
    dec.has_ts = has_ts != 0; dec.seek_delta = seek_delta;
    std::vector<uint32_t> bits; uint64_t key = 0;
    build_static_mask(ctx, *params, bits, key);
    SampCfg cfg; make_samp_cfg(ctx, *params, cfg);
    int rowinfo[2]; samp_rowinfo(ctx.vocab, *params, dec, rowinfo);
    rowinfo[0] |= k << 8;
    std::mt19937 rng(seed);
    std::vector<double> u((size_t) k);
    for (double & v : u) v = std::generate_canonical<double, std::numeric_limits<double>::digits>(rng);
    DevBuf<float> dl; DevBuf<uint32_t> dm; DevBuf<int> dr; DevBuf<SampOut> dout; DevBuf<double> du;
    if (!dl.alloc(n) || !dm.alloc(bits.size()) || !dr.alloc(2) || !dout.alloc(k) || !du.alloc(k)) return -2;
    std::vector<SampOut> o((size_t) k);
    if (cudaMemcpy(dl.p, logits_in, (size_t) n * 4, cudaMemcpyHostToDevice) != cudaSuccess || cudaMemcpy(dm.p, bits.data(), bits.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(dr.p, rowinfo, sizeof(rowinfo), cudaMemcpyHostToDevice) != cudaSuccess || cudaMemcpy(du.p, u.data(), (size_t) k * 8, cudaMemcpyHostToDevice) != cudaSuccess) return -2;
    cfg.mask = dm.p;
    greedy_sample(dl.p, n, 1, dr.p, cfg, dout.p, nullptr, du.p, k);
    if (cudaMemcpy(o.data(), dout.p, (size_t) k * sizeof(SampOut), cudaMemcpyDeviceToHost) != cudaSuccess) return -2;
    for (int i = 0; i < k; ++i) out[i] = from_samp(o[i]);
    return 0;
}

WB_EXPORT int wb200_full_batch(struct whisper_context * ctx, struct whisper_full_params params, const float * const * samples,
                               const int * n_samples, int n_chunks, struct whisper_state ** states_out) {
    return wb200_full_batch_ex(ctx, params, samples, n_samples, n_chunks, states_out, 0);
}

} // extern "C"

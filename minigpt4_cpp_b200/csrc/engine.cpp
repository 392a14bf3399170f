// engine.cpp — see engine.h.
#include "engine.h"
#include "../../include/minigpt4.h"
#include <stddef.h>
#include <string.h>
#include <algorithm>
#include <cmath>
#include <exception>

namespace mg4 {

TPConfig g_tp_config;

// where a constraint's pairs start in its device table (in ints): after the n_states + 2 offsets, at an 8-byte boundary
static size_t constraint_pairs_at(const Constraint &c) { return (c.off.size() + 1) / 2 * 2; }

Engine::~Engine() {
    llm_.reset();
    vis_lanes_.reset();   // (lanes borrow the first lane's weights)
    vis_.reset();
    tp.destroy();
}

Error Engine::init(const std::string &path, const std::string &llm_path, int verbosity, int seed, int n_ctx, int n_batch, bool /*numa: CPU-only notion*/) {
    g_verbosity = verbosity;
    n_batch_ = n_batch > 0 ? n_batch : 512;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        // No CPU fallback exists: the hot path is CUDA only.  Reported at every verbosity - a caller must never mistake this for a slow success.
        cudaGetLastError();
        fprintf(stderr, "[minigpt4-b200][error] no CUDA device available; this engine has no CPU path\n");
        return ErrLoadLanguageModel;
    }
    Error where = ErrLoadLanguageModel;
    try {
        LoadScope loading;   // failed checks below throw LoadFailure instead of aborting the host process (common.h)
        if (g_tp_config.set && g_tp_config.world > 1) tp.init(g_tp_config.rank, g_tp_config.world, g_tp_config.id);
        {
            const double t0 = now_ms();
            LlamaFile lf;
            if (!lf.load(llm_path)) { MG4_ERR("failed to read language model %s", llm_path.c_str()); return ErrLoadLanguageModel; }
            tok_->init(lf.vocab);
            llm_.reset(new LlamaDevice());
            if (!llm_->load(lf, n_ctx > 0 ? n_ctx : 2048, tp.world > 1 ? &tp : nullptr)) return ErrLoadLanguageModel;
            MG4_INFO("Load language model took %.0f ms", now_ms() - t0);
        }
        if (!path.empty()) {
            where = ErrLoadModelFileHeader;
            const double t0 = now_ms();
            vfile_.reset(new VisionFile());   // (kept mapped: further encode lanes are built from it on demand)
            VisionFile &vf = *vfile_;
            if (Error e = vf.load(path)) return e;
            vis_.reset(new VisionDevice());
            if (Error e = vis_->load(vf)) return e;
            if (vis_->dims().n_embd_llm != llm_->dims().n_embd)
                MG4_ERR("warning: llama_proj width %d != language model n_embd %d", vis_->dims().n_embd_llm, llm_->dims().n_embd);
            MG4_INFO("Load model from file took %.0f ms", now_ms() - t0);
        }
    } catch (const LoadFailure &f) {
        fprintf(stderr, "[minigpt4-b200][error] %s\n", f.msg);
        return where;
    } catch (const std::exception &e) {   // (host memory exhausted while reading a file, ...)
        fprintf(stderr, "[minigpt4-b200][error] %s\n", e.what());
        return where;
    }
    sampler_.reset(new Sampler(seed));
    logits_.resize((size_t)llm_->dims().n_vocab);
    return ErrNone;
}

Error Engine::init_session(const Engine &parent, int seed) {
    if (parent.tp.world > 1) { MG4_ERR("sessions of a tensor-parallel context are not supported"); return ErrLoadLanguageModel; }
    vfile_ = parent.vfile_; vis_ = parent.vis_; vis_lanes_ = parent.vis_lanes_; tok_ = parent.tok_;
    n_batch_ = parent.n_batch_;
    try {
        LoadScope loading;   // device memory exhausted -> an error code, not an abort
        llm_.reset(new LlamaDevice());
        if (!llm_->load_session(*parent.llm_)) return ErrLoadLanguageModel;
    } catch (const LoadFailure &f) {
        fprintf(stderr, "[minigpt4-b200][error] session: %s\n", f.msg);
        return ErrLoadLanguageModel;
    } catch (const std::exception &e) {
        fprintf(stderr, "[minigpt4-b200][error] session: %s\n", e.what());
        return ErrLoadLanguageModel;
    }
    sampler_.reset(new Sampler(seed));
    logits_.resize((size_t)llm_->dims().n_vocab);
    return ErrNone;
}

// Batched decode (extension): every check happens before anything runs, so a refused batch leaves every context as it was.
bool Engine::group_valid(Engine *const *e, int n, const char *what) {
    if (!e || n < 1 || n > LlamaDevice::kMaxBatch) { MG4_ERR("%s: %d contexts (1 .. %d)", what, n, LlamaDevice::kMaxBatch); return false; }
    for (int i = 0; i < n; ++i) {
        if (!e[i]) { MG4_ERR("%s: context %d is NULL", what, i); return false; }
        for (int j = 0; j < i; ++j) if (e[j] == e[i]) { MG4_ERR("%s: context %d appears twice", what, i); return false; }
        if (e[i]->llm_->group() != e[0]->llm_->group()) { MG4_ERR("%s: context %d serves another model", what, i); return false; }
    }
    return true;
}
bool Engine::batch_valid(Engine *const *e, int n, const int32_t *ids) {
    if (!group_valid(e, n, "decode_batch")) return false;
    for (int i = 0; i < n; ++i) {
        const LlamaDims &d = e[i]->llm_->dims();
        if (e[i]->n_past_ + 1 > d.n_ctx) { MG4_ERR("decode_batch: context %d is full (n_ctx %d)", i, d.n_ctx); return false; }
        if (ids && ids[i] >= d.n_vocab) { MG4_ERR("decode_batch: token id %d out of range", ids[i]); return false; }
    }
    return true;
}
Error Engine::decode_batch(Engine *const *e, int n, const int32_t *ids, int32_t *ids_out) {
    if (!ids || !ids_out || !batch_valid(e, n, ids)) return ErrFailedToAddString;
    if (!flush_group(e, n)) return ErrFailedToAddString;   // queued prompt rows of all n contexts in shared passes
    if (n == 1) {   // one context: its own decode graph or megakernel, exactly as add_tokens' single-token step
        Engine &c = *e[0];
        if (!c.llm_->decode_step(ids[0], c.n_past_)) return ErrFailedToAddString;
        ids_out[0] = c.llm_->argmax();
    } else {
        LlamaDevice *L[LlamaDevice::kMaxBatch]; int np[LlamaDevice::kMaxBatch];
        for (int i = 0; i < n; ++i) { L[i] = e[i]->llm_.get(); np[i] = e[i]->n_past_; }
        LlamaDevice::decode_batch(L, n, ids, np, ids_out);
    }
    for (int i = 0; i < n; ++i) e[i]->n_past_ += 1;
    return ErrNone;
}
Error Engine::end_chat_batch(Engine *const *e, int n, const char **tokens, const SamplingArgs &p) {
    if (!tokens || !batch_valid(e, n, nullptr)) return ErrFailedToAddString;   // (before any sampler draws)
    if ((p.mirostat == 1 || p.mirostat == 2) && any_constrained(e, n)) { MG4_ERR("end_chat_batch: mirostat on a constrained context"); return ErrFailedToAddString; }
    if (!flush_group(e, n)) return ErrFailedToAddString;   // so that each sample_token finds its queue empty
    int32_t ids[LlamaDevice::kMaxBatch], out[LlamaDevice::kMaxBatch];
    for (int i = 0; i < n; ++i) { ids[i] = e[i]->sample_token(p); tokens[i] = e[i]->id_to_token(ids[i]); }
    const Error err = decode_batch(e, n, ids, out);
    for (int i = 0; i < n; ++i) e[i]->reply_take_id(ids[i]);
    return err;
}
// a sampler's generator and mirostat μ, to and from the device sampler's form
static void sampler_state(const Sampler &s, uint32_t rng[625], MirostatState &mu) {
    bool init[2];
    s.get_rng(rng);
    s.get_mu(mu.mu, init);
    mu.init[0] = init[0]; mu.init[1] = init[1];
}
static void set_sampler_state(Sampler &s, const SamplingArgs &p, const uint32_t rng[625], const MirostatState &mu) {
    if (p.temp <= 0.f) return;   // greedy: neither was touched
    s.set_rng(rng);
    const bool init[2] = {mu.init[0] != 0, mu.init[1] != 0};
    if (p.mirostat) s.set_mu(mu.mu, init);
}

bool Engine::any_constrained(Engine *const *e, int n) {
    for (int i = 0; i < n; ++i) if (e[i]->cons_) return true;
    return false;
}
template <class Call>
float Engine::device_sampling(Engine *const *e, int n, const SamplingArgs *p, const int32_t *fed, const int32_t *ids_out, Call call) {
    LlamaDevice *L[LlamaDevice::kMaxBatch]; int np[LlamaDevice::kMaxBatch]; MirostatState mu[LlamaDevice::kMaxBatch]; SampleConstraint cons[LlamaDevice::kMaxBatch];
    std::vector<uint32_t> rng_words((size_t)n * 625);   // (625 words a generator: 160 KB at kMaxBatch, off the stack)
    uint32_t (*rng)[625] = reinterpret_cast<uint32_t (*)[625]>(rng_words.data());
    for (int i = 0; i < n; ++i) {
        L[i] = e[i]->llm_.get(); np[i] = e[i]->n_past_; sampler_state(*e[i]->sampler_, rng[i], mu[i]);
        cons[i] = SampleConstraint{};
        if (const Constraint *c = e[i]->cons_.get()) {
            const int *off = (const int *)c->dev->dev;
            cons[i] = SampleConstraint{off, (const int2 *)(off + constraint_pairs_at(*c)), e[i]->cons_state_};
        }
    }
    const float ms = call(L, np, rng, mu, cons);
    for (int i = 0; i < n; ++i) {
        set_sampler_state(*e[i]->sampler_, p[i], rng[i], mu[i]);
        e[i]->n_past_ += fed[i];
        for (int t = 0; t < fed[i]; ++t) e[i]->reply_take_id(ids_out[(size_t)t * n + i]);
    }
    return ms;
}

Error Engine::sample_steps(Engine *const *e, int n, int steps, const SamplingArgs &p, int32_t *ids_out, float *ms_out) {
    if (!ids_out || !group_valid(e, n, "sample_steps")) return ErrFailedToAddString;
    if (steps < 1) { MG4_ERR("sample_steps: %d steps", steps); return ErrFailedToAddString; }
    if (p.mirostat && any_constrained(e, n)) { MG4_ERR("sample_steps: mirostat on a constrained context"); return ErrFailedToAddString; }
    for (int i = 0; i < n; ++i) {
        if (e[i]->tp.world > 1) { MG4_ERR("sample_steps: context %d is tensor-parallel", i); return ErrFailedToAddString; }
        const int n_ctx = e[i]->llm_->dims().n_ctx;
        if (e[i]->n_past_ + steps > n_ctx) { MG4_ERR("sample_steps: context %d: %d + %d > n_ctx %d", i, e[i]->n_past_, steps, n_ctx); return ErrFailedToAddString; }
    }
    if (!flush_group(e, n)) return ErrFailedToAddString;
    SamplingArgs ps[LlamaDevice::kMaxBatch];
    int32_t fed[LlamaDevice::kMaxBatch];
    std::fill(ps, ps + n, p);
    std::fill(fed, fed + n, steps);
    const float ms = device_sampling(e, n, ps, fed, ids_out, [&](LlamaDevice *const *L, const int *np, uint32_t (*rng)[625], MirostatState *mu,
                                                                 const SampleConstraint *cons) {
        return LlamaDevice::sample_steps(L, n, steps, np, p, rng, mu, ids_out, cons);
    });
    if (ms_out) *ms_out = ms;
    return ErrNone;
}
Error Engine::sample_until(Engine *const *e, int n, const UntilArgs *u, int32_t *ids_out, int32_t *n_out, int32_t *stopped, float *ms_out,
                           const LogprobRequest *rec, const char *what) {
    if (rec) {   // (arguments first: none of these reads a context)
        if (!rec->logprob) { MG4_ERR("%s: NULL logprob_out", what); return ErrFailedToAddString; }
        if (rec->top_n < 0 || rec->top_n > LlamaDevice::kLogprobTop) { MG4_ERR("%s: top_n %d (0 .. %d)", what, rec->top_n, LlamaDevice::kLogprobTop); return ErrFailedToAddString; }
        if (rec->top_n > 0 && !rec->top_ids) { MG4_ERR("%s: NULL top_ids_out with top_n %d", what, rec->top_n); return ErrFailedToAddString; }
    }
    if (!u) { MG4_ERR("%s: NULL params", what); return ErrFailedToAddString; }
    if (!ids_out || !n_out || !group_valid(e, n, what)) return ErrFailedToAddString;
    const int n_vocab = e[0]->llm_->dims().n_vocab;
    for (int i = 0; i < n; ++i) {   // each context's own settings, as the single calls check them
        const UntilArgs &g = u[i];
        if (e[i]->tp.world > 1) { MG4_ERR("%s: context %d is tensor-parallel", what, i); return ErrFailedToAddString; }
        if (g.max_steps < 1) { MG4_ERR("%s: context %d: %d steps", what, i, g.max_steps); return ErrFailedToAddString; }
        if (g.stop.size() > (size_t)LlamaDevice::kStopMax) {
            MG4_ERR("%s: context %d: stop text of %zu bytes (at most %d)", what, i, g.stop.size(), LlamaDevice::kStopMax); return ErrFailedToAddString;
        }
        if (!penalty_valid(g.q, g.p.mirostat, what) || !history_valid(g.last_ids, g.n_last, n_vocab, what)) return ErrFailedToAddString;
        if (g.p.mirostat && e[i]->cons_) { MG4_ERR("%s: mirostat on constrained context %d", what, i); return ErrFailedToAddString; }
        if (rec && e[i]->n_past_ == 0) { MG4_ERR("%s: context %d: the conversation is empty", what, i); return ErrFailedToAddString; }
        const int n_ctx = e[i]->llm_->dims().n_ctx;
        if (e[i]->n_past_ + g.max_steps > n_ctx) { MG4_ERR("%s: context %d: %d + %d > n_ctx %d", what, i, e[i]->n_past_, g.max_steps, n_ctx); return ErrFailedToAddString; }
    }
    if (!flush_group(e, n)) return ErrFailedToAddString;
    e[0]->ensure_token_table();
    SamplingArgs p[LlamaDevice::kMaxBatch];
    std::string tail[LlamaDevice::kMaxBatch];
    for (int i = 0; i < n; ++i) { p[i] = u[i].p; tail[i] = e[i]->reply_; }
    const float ms = device_sampling(e, n, p, n_out, ids_out, [&](LlamaDevice *const *L, const int *np, uint32_t (*rng)[625], MirostatState *mu,
                                                                  const SampleConstraint *cons) {
        return LlamaDevice::sample_until(L, n, u, np, rng, mu, tail, ids_out, n_out, stopped, cons, rec);
    });
    if (ms_out) *ms_out = ms;
    return ErrNone;
}
bool Engine::penalty_valid(const PenaltyParams &q, int mirostat, const char *what) {
    if (mirostat < 0 || mirostat > 2) { MG4_ERR("%s: mirostat %d (0 .. 2)", what, mirostat); return false; }
    if (q.repeat_last_n < 0) { MG4_ERR("%s: repeat_last_n %d", what, q.repeat_last_n); return false; }
    if (!std::isfinite(q.repeat_penalty) || q.repeat_penalty <= 0.f) { MG4_ERR("%s: repeat_penalty %g (finite, > 0)", what, q.repeat_penalty); return false; }
    if (!std::isfinite(q.alpha_presence) || !std::isfinite(q.alpha_frequency)) { MG4_ERR("%s: an alpha is not finite", what); return false; }
    if (q.penalize_nl != 0 && q.penalize_nl != 1) { MG4_ERR("%s: penalize_nl %d (0 or 1)", what, q.penalize_nl); return false; }
    return true;
}
bool Engine::history_valid(const int32_t *ids, int n, int n_vocab, const char *what) {
    if (n < 0) { MG4_ERR("%s: a history of %d ids", what, n); return false; }
    if (n > 0 && !ids) { MG4_ERR("%s: NULL last_ids for a history of %d ids", what, n); return false; }
    for (int j = 0; j < n; ++j) if (ids[j] < 0 || ids[j] >= n_vocab) { MG4_ERR("%s: history id %d out of range", what, ids[j]); return false; }
    return true;
}
Error Engine::end_chat_penalized(const SamplingArgs &p, const PenaltyParams &q, const int32_t *last_ids, int n_last, const char **token,
                                 int32_t *id_out) {
    if (!token || !penalty_valid(q, p.mirostat, "end_chat_penalized")) return ErrFailedToAddString;
    const int V = llm_->dims().n_vocab;
    if (!history_valid(last_ids, n_last, V, "end_chat_penalized")) return ErrFailedToAddString;
    if (cons_ && (p.mirostat == 1 || p.mirostat == 2)) { MG4_ERR("end_chat_penalized: mirostat on a constrained context"); return ErrFailedToAddString; }
    int32_t id;
    if (q.neutral()) id = sample_token(p);   // no logit changes: minigpt4_end_chat itself
    else {
        flush();
        llm_->logits_to_host(logits_.data());
        const int w = std::min(q.repeat_last_n, n_last);
        Sampler::penalize(logits_.data(), V, last_ids + (n_last - w), w, q.repeat_penalty, q.alpha_presence, q.alpha_frequency, q.penalize_nl);
        if (cons_) {   // (as sample_token: the chain over the allowed ids, greedy their first arg-max)
            const int m = cons_->row_size(cons_state_);
            const int32_t *row = cons_->row(cons_state_);
            std::vector<int32_t> ids((size_t)m);
            for (int j = 0; j < m; ++j) ids[(size_t)j] = row[2 * j];
            id = sampler_->sample_allowed(logits_.data(), ids.data(), m, p);
        } else id = sampler_->sample(logits_.data(), V, p);
    }
    *token = id_to_token(id);
    if (id_out) *id_out = id;
    add_tokens({id});   // (minigpt4_end_chat ignores this return value too)
    reply_take_id(id);
    return ErrNone;
}
Error Engine::beam_search(Engine *const *e, int n, int max_steps, const char *stop, float length_penalty, int n_hyp, int32_t *ids_out,
                          int32_t *n_out, float *score_out, float *logprob_out, int32_t *stopped, float *ms_out) {
    if (!e || !ids_out || !n_out || !score_out) { MG4_ERR("beam_search: NULL contexts or outputs"); return ErrFailedToAddString; }
    if (n < 1 || n > LlamaDevice::kMaxBeams) { MG4_ERR("beam_search: %d beams (1 .. %d)", n, LlamaDevice::kMaxBeams); return ErrFailedToAddString; }
    if (!group_valid(e, n, "beam_search")) return ErrFailedToAddString;
    if (max_steps < 1) { MG4_ERR("beam_search: %d steps", max_steps); return ErrFailedToAddString; }
    if (n_hyp < 1 || n_hyp > n) { MG4_ERR("beam_search: %d hypotheses (1 .. %d)", n_hyp, n); return ErrFailedToAddString; }
    const std::string st = stop ? stop : "###";   // the reference's EOS_SUFFIX
    if (st.size() > (size_t)LlamaDevice::kStopMax) { MG4_ERR("beam_search: stop text of %zu bytes (at most %d)", st.size(), LlamaDevice::kStopMax); return ErrFailedToAddString; }
    if (!std::isfinite(length_penalty)) { MG4_ERR("beam_search: length_penalty is not finite"); return ErrFailedToAddString; }
    for (int i = 0; i < n; ++i) {
        if (e[i]->tp.world > 1) { MG4_ERR("beam_search: context %d is tensor-parallel", i); return ErrFailedToAddString; }
        if (e[i]->cons_) { MG4_ERR("beam_search: context %d is constrained", i); return ErrFailedToAddString; }
    }
    Engine &c0 = *e[0];
    const int n0 = c0.n_past_, n_ctx = c0.llm_->dims().n_ctx;
    if (n0 == 0) { MG4_ERR("beam_search: the conversation is empty"); return ErrFailedToAddString; }
    if (n0 + max_steps > n_ctx) { MG4_ERR("beam_search: %d + %d > n_ctx %d", n0, max_steps, n_ctx); return ErrFailedToAddString; }
    if (!c0.flush()) return ErrFailedToAddString;
    c0.ensure_token_table();
    LlamaDevice *L[LlamaDevice::kMaxBeams];
    for (int i = 0; i < n; ++i) L[i] = e[i]->llm_.get();
    std::vector<LlamaDevice::BeamHyp> hyps;
    const float ms = LlamaDevice::beam_search(L, n, max_steps, n0, st, c0.reply_, length_penalty, hyps);
    for (int h = 0; h < n_hyp; ++h) {
        const bool has = h < (int)hyps.size();
        const int len = has ? (int)hyps[(size_t)h].ids.size() : 0;
        for (int j = 0; j < max_steps; ++j) ids_out[(size_t)h * max_steps + j] = j < len ? hyps[(size_t)h].ids[(size_t)j] : -1;
        n_out[h] = len;
        score_out[h] = has ? hyps[(size_t)h].score : -INFINITY;
        if (logprob_out) logprob_out[h] = has ? hyps[(size_t)h].logprob : -INFINITY;
        if (stopped) stopped[h] = has ? hyps[(size_t)h].stopped : 0;
    }
    // the other contexts: the conversation as it was (as session_copy leaves a destination); e[0]: the best reply fed, as sample_until
    // leaves a context that fed those ids.  One beam fed them with its own decode steps; with more, e[0]'s rows from n0 belong to
    // several beams, and the best reply is evaluated again by the prompt pass (the bits of the decode steps)
    const std::string tail = c0.reply_;
    for (int i = 1; i < n; ++i) { e[i]->n_past_ = n0; e[i]->pend_ids_.clear(); e[i]->pend_emb_.clear(); e[i]->reply_ = tail; e[i]->cons_state_ = 0; }
    const std::vector<int32_t> &best = hyps[0].ids;
    if (n >= 2 && !c0.llm_->eval_rows(best.data(), (int)best.size(), nullptr, 0, n0)) return ErrFailedToAddString;
    c0.n_past_ = n0 + (int)best.size();
    for (int32_t id : best) c0.reply_take_id(id);
    if (ms_out) *ms_out = ms;
    return ErrNone;
}
Error Engine::reply_stop(const int32_t *ids, int n, const char *stop, const char *tail, int32_t *stop_at) {
    const std::string st = stop ? stop : "###";
    if (!stop_at || n < 0 || (n > 0 && !ids) || st.size() > (size_t)LlamaDevice::kStopMax) return ErrFailedToAddString;
    for (int i = 0; i < n; ++i) if (ids[i] < 0 || ids[i] >= llm_->dims().n_vocab) { MG4_ERR("reply_stop: token id %d out of range", ids[i]); return ErrFailedToAddString; }
    ensure_token_table();
    *stop_at = llm_->test_reply_stop(ids, n, st, tail ? tail : "");
    return ErrNone;
}
void Engine::ensure_token_table() {
    if (llm_->has_token_table()) return;
    const int V = llm_->dims().n_vocab;
    std::vector<int> off((size_t)V + 1, 0);
    std::string bytes;
    for (int id = 0; id < V; ++id) { bytes += id_to_token(id); off[(size_t)id + 1] = (int)bytes.size(); }
    llm_->set_token_table(off, bytes);
}
void Engine::reply_take(const char *text) {
    reply_ += text;
    if (reply_.size() > (size_t)LlamaDevice::kStopMax) reply_.erase(0, reply_.size() - LlamaDevice::kStopMax);
}
Error Engine::flush_batch(Engine *const *e, int n) {
    if (!group_valid(e, n, "flush_batch")) return ErrFailedToAddString;
    return flush_group(e, n) ? ErrNone : ErrFailedToAddString;
}
Error Engine::score_tokens(Engine *const *e, int n, const int32_t *ids, const int32_t *n_ids, int keep, float *logprob, int32_t *rank, float *logits) {
    if (!ids || !n_ids || !logprob || !group_valid(e, n, "score_tokens")) return ErrFailedToAddString;
    if (keep != 0 && keep != 1) { MG4_ERR("score_tokens: keep %d (0 or 1)", keep); return ErrFailedToAddString; }
    const int n_vocab = e[0]->llm_->dims().n_vocab;
    size_t off[LlamaDevice::kMaxBatch];
    size_t total = 0;
    for (int i = 0; i < n; ++i) {
        if (e[i]->tp.world > 1) { MG4_ERR("score_tokens: context %d is tensor-parallel", i); return ErrFailedToAddString; }
        const int n_ctx = e[i]->llm_->dims().n_ctx;
        if (n_ids[i] < 1) { MG4_ERR("score_tokens: context %d: %d ids", i, n_ids[i]); return ErrFailedToAddString; }
        if (n_ids[i] > n_ctx - e[i]->n_past_) { MG4_ERR("score_tokens: context %d: %d + %d > n_ctx %d", i, e[i]->n_past_, n_ids[i], n_ctx); return ErrFailedToAddString; }
        off[i] = total;
        total += (size_t)n_ids[i];
    }
    for (size_t t = 0; t < total; ++t)
        if (ids[t] < 0 || ids[t] >= n_vocab) { MG4_ERR("score_tokens: token id %d out of range", ids[t]); return ErrFailedToAddString; }
    if (!flush_group(e, n)) return ErrFailedToAddString;
    LlamaDevice *L[LlamaDevice::kMaxBatch]; const int32_t *id[LlamaDevice::kMaxBatch]; int np[LlamaDevice::kMaxBatch];
    float *lp[LlamaDevice::kMaxBatch], *lg[LlamaDevice::kMaxBatch]; int32_t *rk[LlamaDevice::kMaxBatch];
    for (int i = 0; i < n; ++i) {
        L[i] = e[i]->llm_.get(); id[i] = ids + off[i]; np[i] = e[i]->n_past_; lp[i] = logprob + off[i];
        rk[i] = rank ? rank + off[i] : nullptr; lg[i] = logits ? logits + off[i] * (size_t)n_vocab : nullptr;
    }
    LlamaDevice::score_rows(L, n, id, n_ids, np, keep == 1, lp, rank ? rk : nullptr, logits ? lg : nullptr);
    if (keep)
        for (int i = 0; i < n; ++i) { e[i]->n_past_ += n_ids[i]; e[i]->reply_clear(); }
    return ErrNone;
}
Error Engine::session_copy(Engine *src, Engine *const *dsts, int n, float *kernel_ms) {
    if (!src || !dsts) { MG4_ERR("session_copy: NULL source or destinations"); return ErrFailedToAddString; }
    if (n < 1 || n > LlamaDevice::kMaxBatch) { MG4_ERR("session_copy: %d destinations (1 .. %d)", n, LlamaDevice::kMaxBatch); return ErrFailedToAddString; }
    if (src->tp.world > 1) { MG4_ERR("session_copy: the source is tensor-parallel"); return ErrFailedToAddString; }
    for (int i = 0; i < n; ++i) {
        if (!dsts[i]) { MG4_ERR("session_copy: destination %d is NULL", i); return ErrFailedToAddString; }
        if (dsts[i] == src) { MG4_ERR("session_copy: destination %d is the source", i); return ErrFailedToAddString; }
        for (int j = 0; j < i; ++j) if (dsts[j] == dsts[i]) { MG4_ERR("session_copy: destination %d appears twice", i); return ErrFailedToAddString; }
        if (dsts[i]->llm_->group() != src->llm_->group()) { MG4_ERR("session_copy: destination %d serves another model", i); return ErrFailedToAddString; }
        if (dsts[i]->tp.world > 1) { MG4_ERR("session_copy: destination %d is tensor-parallel", i); return ErrFailedToAddString; }
    }
    if (!src->flush()) return ErrFailedToAddString;
    LlamaDevice *L[LlamaDevice::kMaxBatch];
    for (int i = 0; i < n; ++i) L[i] = dsts[i]->llm_.get();
    const float ms = LlamaDevice::copy_state(*src->llm_, L, n, src->n_past_);
    for (int i = 0; i < n; ++i) {
        Engine &d = *dsts[i];
        d.n_past_ = src->n_past_; d.pend_ids_.clear(); d.pend_emb_.clear(); d.reply_ = src->reply_;
        d.cons_state_ = d.cons_ && d.cons_ == src->cons_ ? src->cons_state_ : 0;   // the source's state means nothing to another constraint
    }
    if (kernel_ms) *kernel_ms = ms;
    return ErrNone;
}

// The saved conversation (minigpt4_b200_state_save): this header, n_vocab F32 logits, then K[n_layer][n_past][n_embd] and V[...] as F16.
// Little-endian, as the engine's x86-64 / aarch64 hosts store it; every field sits at its natural alignment, so the struct is the layout.
namespace {
constexpr char kStateMagic[8] = {'M', 'G', '4', 'S', 'T', 'A', 'T', 'E'};
constexpr uint32_t kStateVersion = 1;
struct StateHeader {
    char magic[8];
    uint32_t version;
    int32_t n_vocab, n_embd, n_head, n_layer, n_ff;
    uint64_t fingerprint;
    int32_t n_past;
    int32_t reply_len;
    char reply[LlamaDevice::kStopMax];
    DeviceState state;
};
static_assert(sizeof(DeviceState) == 64 && sizeof(StateHeader) == 144 && offsetof(StateHeader, state) == 80, "the documented blob layout");
long long state_bytes(const LlamaDims &d, long long n_past) { return (long long)sizeof(StateHeader) + 4LL * d.n_vocab + 4LL * d.n_layer * n_past * d.n_embd; }
}  // namespace

long long Engine::state_size() const { return tp.world > 1 ? -1 : state_bytes(llm_->dims(), n_past_); }

Error Engine::state_save(void *buf, long long cap, long long *written) {
    if (!buf || tp.world > 1) { MG4_ERR("state_save: NULL buffer or a tensor-parallel context"); return ErrFailedToAddString; }
    const long long need = state_size();
    if (cap < need) { MG4_ERR("state_save: %lld bytes of room for a %lld-byte state", cap, need); return ErrFailedToAddString; }
    if (!flush()) return ErrFailedToAddString;
    const LlamaDims &d = llm_->dims();
    StateHeader h;
    memset(&h, 0, sizeof h);
    memcpy(h.magic, kStateMagic, 8); h.version = kStateVersion;
    h.n_vocab = d.n_vocab; h.n_embd = d.n_embd; h.n_head = d.n_head; h.n_layer = d.n_layer; h.n_ff = d.n_ff;
    h.fingerprint = llm_->fingerprint(); h.n_past = n_past_;
    h.reply_len = (int32_t)reply_.size(); memcpy(h.reply, reply_.data(), reply_.size());
    unsigned char *out = (unsigned char *)buf;
    float *logits = (float *)(out + sizeof h);
    llm_->state_to_host(n_past_, &h.state, logits, out + sizeof h + 4 * (size_t)d.n_vocab);
    h.state.n_past = n_past_;   // (minigpt4_reset_chat rewinds the conversation, not the device state, which the next evaluation sets)
    memcpy(out, &h, sizeof h);
    if (written) *written = need;
    return ErrNone;
}

Error Engine::state_load(const void *buf, long long size) {
    if (!buf || tp.world > 1) { MG4_ERR("state_load: NULL buffer or a tensor-parallel context"); return ErrFailedToAddString; }
    if (size < (long long)sizeof(StateHeader)) { MG4_ERR("state_load: %lld bytes, shorter than the header", size); return ErrFailedToAddString; }
    StateHeader h;
    memcpy(&h, buf, sizeof h);
    const LlamaDims &d = llm_->dims();
    if (memcmp(h.magic, kStateMagic, 8) != 0 || h.version != kStateVersion) { MG4_ERR("state_load: not a version %u state", kStateVersion); return ErrFailedToAddString; }
    if (h.n_vocab != d.n_vocab || h.n_embd != d.n_embd || h.n_head != d.n_head || h.n_layer != d.n_layer || h.n_ff != d.n_ff) {
        MG4_ERR("state_load: the state was saved by a model of other dimensions"); return ErrFailedToAddString;
    }
    if (h.fingerprint != llm_->fingerprint()) { MG4_ERR("state_load: the state was saved by another model"); return ErrFailedToAddString; }
    if (h.n_past < 0 || h.n_past > d.n_ctx) { MG4_ERR("state_load: n_past %d outside 0 .. n_ctx %d", h.n_past, d.n_ctx); return ErrFailedToAddString; }
    if (size != state_bytes(d, h.n_past)) { MG4_ERR("state_load: %lld bytes, the header implies %lld", size, state_bytes(d, h.n_past)); return ErrFailedToAddString; }
    if (h.state.n_past != h.n_past) { MG4_ERR("state_load: device state at %d, header at %d", h.state.n_past, h.n_past); return ErrFailedToAddString; }
    if (h.reply_len < 0 || h.reply_len > LlamaDevice::kStopMax) { MG4_ERR("state_load: reply tail of %d bytes", h.reply_len); return ErrFailedToAddString; }
    const unsigned char *in = (const unsigned char *)buf;
    llm_->state_from_host(h.n_past, h.state, (const float *)(in + sizeof h), in + sizeof h + 4 * (size_t)d.n_vocab);
    n_past_ = h.n_past; pend_ids_.clear(); pend_emb_.clear(); reply_.assign(h.reply, (size_t)h.reply_len);
    cons_state_ = 0;   // (the blob carries no constraint state)
    return ErrNone;
}

// the queues of a validated batch: one context with queued rows is its own flush(), several share the passes of eval_rows_batch
bool Engine::flush_group(Engine *const *e, int n) {
    Engine *q[LlamaDevice::kMaxBatch]; int m = 0;
    for (int i = 0; i < n; ++i) if (!e[i]->pend_ids_.empty()) q[m++] = e[i];
    if (m <= 1) return m == 0 || q[0]->flush();
    LlamaDevice *L[LlamaDevice::kMaxBatch]; const int32_t *ids[LlamaDevice::kMaxBatch]; const float *emb[LlamaDevice::kMaxBatch];
    int rows[LlamaDevice::kMaxBatch], base[LlamaDevice::kMaxBatch];
    for (int i = 0; i < m; ++i) {
        L[i] = q[i]->llm_.get(); ids[i] = q[i]->pend_ids_.data(); emb[i] = q[i]->pend_emb_.data();
        rows[i] = (int)q[i]->pend_ids_.size(); base[i] = q[i]->pend_base_;
    }
    LlamaDevice::eval_rows_batch(L, m, ids, rows, emb, base);
    for (int i = 0; i < m; ++i) { q[i]->pend_ids_.clear(); q[i]->pend_emb_.clear(); }
    return true;
}

// input validation = reference minigpt4.cpp:2130-2138
Error Engine::encode_image(const ::MiniGPT4Image *image, ::MiniGPT4Embedding *out) {
    if (!vis_) MG4_PANIC("encode_image on a context loaded without a vision model");
    if ((long)image->width * image->height * image->channels != 224L * 224 * 3) return ErrImageNot224_244_3;
    if (image->format != MINIGPT4_IMAGE_FORMAT_F32) return ErrImageNotF32;
    const size_t n = (size_t)32 * vis_->dims().n_embd_llm;
    out->elements = n;
    out->data = new float[n];
    last_encode_ms = vis_->encode((const float *)image->data, out->data);
    MG4_INFO("Encoding image took %.3f ms on device", last_encode_ms);
    return ErrNone;
}

// Batched encode (extension; the reference encodes one image per call, minigpt4.cpp:2094): up to kEncodeLanes images are in flight at once, each on
// its own lane = its own activations, CUDA graph and stream over the SHARED weights.  One image's graph leaves most SMs idle most of the time
// (its GEMMs are 44-144 CTAs, its attention 144, the Q-Former a handful), so concurrent graphs interleave on the machine; every image goes
// through exactly the single-image graph, so each embedding is bit-identical to minigpt4_encode_image's.
Error Engine::encode_images(const ::MiniGPT4Image *images, size_t n, ::MiniGPT4Embedding *out, float *total_ms) {
    if (!vis_) MG4_PANIC("encode_images on a context loaded without a vision model");
    for (size_t i = 0; i < n; ++i) {
        if ((long)images[i].width * images[i].height * images[i].channels != 224L * 224 * 3) return ErrImageNot224_244_3;
        if (images[i].format != MINIGPT4_IMAGE_FORMAT_F32) return ErrImageNotF32;
    }
    const size_t lanes = std::min<size_t>(n, (size_t)kEncodeLanes);
    while (vis_lanes_->size() + 1 < lanes) {
        std::unique_ptr<VisionDevice> l(new VisionDevice());
        try {
            LoadScope loading;   // (a lane that does not fit in device memory is an error code, not an abort)
            if (Error e = l->load(*vfile_, vis_.get())) return e;
        } catch (const LoadFailure &f) {
            fprintf(stderr, "[minigpt4-b200][error] encode lane %zu: %s\n", vis_lanes_->size() + 1, f.msg);
            return ErrLoadModelFileHeader;
        }
        vis_lanes_->push_back(std::move(l));
    }
    auto lane = [&](size_t k) { return k == 0 ? vis_.get() : (*vis_lanes_)[k - 1].get(); };
    const size_t ne = (size_t)32 * vis_->dims().n_embd_llm;
    const double t0 = now_ms();
    for (size_t base = 0; base < n; base += lanes) {
        const size_t c = std::min(lanes, n - base);
        for (size_t k = 0; k < c; ++k) lane(k)->encode_begin((const float *)images[base + k].data);
        for (size_t k = 0; k < c; ++k) {
            out[base + k].elements = ne; out[base + k].data = new float[ne];
            last_encode_ms = lane(k)->encode_end(out[base + k].data);
        }
    }
    if (total_ms) *total_ms = (float)(now_ms() - t0);
    return ErrNone;
}

// add_tokens (minigpt4.cpp:2365-2382) / add_embedding (:2399-2415).  The reference evaluates every piece of a chat turn separately
// (system prompt, "Human: <Img>", the 32 image rows, "</Img> ", the question, "### Assistant:" = six passes over the weights).  Results are
// batch invariant (every row is quantised and reduced on its own), so the pieces are only QUEUED here and evaluated together - one pass over
// the weights per LlamaDevice::kPrefillMax rows - when something needs the model state (sampling, logits, a decode step, the hidden state).
// Validation happens at queue time, so the error codes of the reference's call sites are unchanged.  A single token on an empty queue is
// the decode loop: it goes straight through the captured decode graph.
Error Engine::add_tokens(const std::vector<int32_t> &tokens) {
    if (tokens.empty()) return ErrNone;
    const int n = (int)tokens.size(), n_vocab = llm_->dims().n_vocab;
    bool ok = n_past_ + n <= llm_->dims().n_ctx;
    if (!ok) MG4_ERR("context overflow: %d + %d > n_ctx %d", n_past_, n, llm_->dims().n_ctx);
    for (int i = 0; ok && i < n; ++i) if (tokens[(size_t)i] < 0 || tokens[(size_t)i] >= n_vocab) { MG4_ERR("token id %d out of range", tokens[(size_t)i]); ok = false; }
    if (ok) {
        if (n == 1 && pend_ids_.empty()) ok = llm_->decode_step(tokens[0], n_past_);   // asynchronous: the next sample / flush synchronises
        else {
            for (int i = 0; ok && i < n; i += kMaxPending) {   // a queue never exceeds kMaxPending rows
                const int c = std::min(kMaxPending, n - i);
                if ((int)pend_ids_.size() + c > kMaxPending) ok = flush();
                if (pend_ids_.empty()) pend_base_ = n_past_ + i;
                pend_ids_.insert(pend_ids_.end(), tokens.begin() + i, tokens.begin() + i + c);
            }
        }
    }
    if (!ok) { MG4_ERR("Failed to add string"); return ErrFailedToAddString; }
    n_past_ += n;
    return ErrNone;
}
// add_strings (minigpt4.cpp:2384-2397): add_bos is ALWAYS true
Error Engine::add_strings(const char *s) { return add_tokens(tok_->encode(s ? s : "", true)); }

Error Engine::add_embedding(const float *rows, int n_rows) {
    if (n_rows <= 0) return ErrNone;
    const size_t E = (size_t)llm_->dims().n_embd;
    bool ok = n_rows <= kMaxPending && n_past_ + n_rows <= llm_->dims().n_ctx;
    if (ok && (int)pend_ids_.size() + n_rows > kMaxPending) ok = flush();
    if (ok) {
        if (pend_ids_.empty()) pend_base_ = n_past_;
        const int k0 = (int)(pend_emb_.size() / E);
        for (int i = 0; i < n_rows; ++i) pend_ids_.push_back(-1 - (k0 + i));
        pend_emb_.insert(pend_emb_.end(), rows, rows + (size_t)n_rows * E);
    }
    if (!ok) { MG4_ERR("Failed to add embedding"); return ErrFailedToAddEmbedding; }
    n_past_ += n_rows;
    return ErrNone;
}
// evaluate the queued rows (no-op when the queue is empty)
bool Engine::flush() {
    if (pend_ids_.empty()) return true;
    const bool ok = llm_->eval_rows(pend_ids_.data(), (int)pend_ids_.size(), pend_emb_.data(), (int)(pend_emb_.size() / (size_t)llm_->dims().n_embd), pend_base_);
    pend_ids_.clear(); pend_emb_.clear();
    if (!ok) MG4_ERR("deferred evaluation of the queued prompt rows failed");
    return ok;
}

int32_t Engine::sample_token(const SamplingArgs &p) {
    flush();
    if (cons_) {   // the chain over the allowed ids (greedy too: the arg-max among them, not the device's over every id)
        llm_->logits_to_host(logits_.data());
        const int m = cons_->row_size(cons_state_);
        const int32_t *row = cons_->row(cons_state_);
        std::vector<int32_t> ids((size_t)m);
        for (int j = 0; j < m; ++j) ids[(size_t)j] = row[2 * j];
        return sampler_->sample_allowed(logits_.data(), ids.data(), m, p);
    }
    if (p.temp <= 0) return llm_->argmax();  // greedy: arg-max was computed on device with the logits
    llm_->logits_to_host(logits_.data());
    return sampler_->sample(logits_.data(), (int)logits_.size(), p);
}

std::vector<std::string> Engine::token_texts() const {
    std::vector<std::string> t((size_t)llm_->dims().n_vocab);
    for (size_t id = 0; id < t.size(); ++id) t[id] = id_to_token((int32_t)id);
    return t;
}
std::shared_ptr<Constraint> Engine::make_constraint(int n_states, const int32_t *next, const uint8_t *accept) {
    if (tp.world > 1) { MG4_ERR("constraint_create: a tensor-parallel context"); return nullptr; }
    std::shared_ptr<Constraint> c = std::make_shared<Constraint>();
    std::string why;
    try {
        if (!compile_constraint(token_texts(), n_states, next, accept, *c, &why)) { MG4_ERR("constraint_create: %s", why.c_str()); return nullptr; }
        // on the device: off, then the pairs from an 8-byte boundary
        const size_t at = constraint_pairs_at(*c);
        std::vector<int32_t> buf(at + c->pairs.size(), 0);
        std::copy(c->off.begin(), c->off.end(), buf.begin());
        std::copy(c->pairs.begin(), c->pairs.end(), buf.begin() + (ptrdiff_t)at);
        c->dev = llm_->upload_table(buf.data(), buf.size() * 4);
    } catch (const std::exception &ex) {   // (host memory exhausted by a huge table)
        MG4_ERR("constraint_create: %s", ex.what());
        return nullptr;
    }
    if (!c->dev) { MG4_ERR("constraint_create: device memory exhausted"); return nullptr; }
    c->group = llm_->group();
    return c;
}
bool Engine::constraint_attach(const std::shared_ptr<Constraint> &c) {
    if (c && c->group != llm_->group()) { MG4_ERR("constraint_attach: the constraint was compiled for another model"); return false; }
    cons_ = c;
    cons_state_ = 0;
    return true;
}
const char *Engine::id_to_token(int32_t id) const {  // minigpt4.cpp:2485-2497
    if (id == 2) return "</s>";
    return tok_->piece(id);
}

}  // namespace mg4

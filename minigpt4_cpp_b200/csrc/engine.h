// engine.h — the engine object behind the C ABI: mirrors the reference's `class MiniGPT4`
// (minigpt4.cpp:1740-2522: init, encode_image, add_tokens, add_strings, add_embedding, sample_token,
// id_to_token, reset) with a device-resident vision graph and LLaMA step instead of ggml/llama.cpp.
#pragma once
#include "constraint.h"
#include "llama.h"
#include "text.h"
#include "tp.h"
#include "vision.h"
#include <memory>

struct MiniGPT4Image;
struct MiniGPT4Embedding;

namespace mg4 {

struct TPConfig { bool set = false; int rank = 0, world = 1; unsigned char id[128]; };
extern TPConfig g_tp_config;

class Engine {
public:
    ~Engine();
    // path may be empty (language model only, extension entry point)
    Error init(const std::string &path, const std::string &llm_path, int verbosity, int seed, int n_ctx, int n_batch, bool numa);
    // a session: a new conversation over the model of `parent` (language and vision weights, encode lanes, tokenizer shared; own KV
    // cache, prompt queue, logits, state and a sampler seeded with `seed`)
    Error init_session(const Engine &parent, int seed);
    // one decode step of n (1..64, LlamaDevice::kMaxBatch) distinct contexts of one group, weights streamed once (see minigpt4_b200_decode_batch); all or nothing
    static Error decode_batch(Engine *const *e, int n, const int32_t *ids, int32_t *ids_out);
    // minigpt4_end_chat on each context (own logits, own sampler), then one decode_batch of the sampled ids
    static Error end_chat_batch(Engine *const *e, int n, const char **tokens, const SamplingArgs &p);
    // `steps` decode steps of n (1..64, LlamaDevice::kMaxBatch) distinct contexts of one group, each fed the id the device sampler draws from its logits with its
    // own generator and mirostat μ (see minigpt4_b200_sample_steps / _mirostat); ids_out[s * n + i]; all or nothing
    static Error sample_steps(Engine *const *e, int n, int steps, const SamplingArgs &p, int32_t *ids_out, float *ms_out);
    // sample_steps that stops each context where the reference's chat loop stops its reply, each with its own settings u[i]: sampling
    // arguments, budget, stop text and penalties (see minigpt4_b200_generate_batch; the uniform calls minigpt4_b200_sample_until,
    // _mirostat, _penalized and _logprobs pass the same settings for every context); ids_out[s * n + i], s < max u[i].max_steps.  All or
    // nothing: every context's settings are checked before any device work.  what: the caller's name in the messages
    // rec (may be null): also each fed id's record (see minigpt4_b200_sample_until_logprobs), with its further refusals
    static Error sample_until(Engine *const *e, int n, const UntilArgs *u, int32_t *ids_out, int32_t *n_out, int32_t *stopped, float *ms_out,
                              const LogprobRequest *rec = nullptr, const char *what = "sample_until");
    // minigpt4_end_chat with the context's host sampler over the penalised copy of its logits (see minigpt4_b200_end_chat_penalized)
    Error end_chat_penalized(const SamplingArgs &p, const PenaltyParams &q, const int32_t *last_ids, int n_last, const char **token, int32_t *id_out);
    // the penalty arguments that need no context (mirostat 0..2 too: the penalised calls take all three modes); what: the caller's name
    static bool penalty_valid(const PenaltyParams &q, int mirostat, const char *what);
    // the n_hyp best replies of e[0]'s conversation by beam search over n (1..16) contexts of its group (see minigpt4_b200_beam_search);
    // all or nothing
    static Error beam_search(Engine *const *e, int n, int max_steps, const char *stop, float length_penalty, int n_hyp, int32_t *ids_out,
                             int32_t *n_out, float *score_out, float *logprob_out, int32_t *stopped, float *ms_out);
    // sample_until's text check over ids from the reply `tail` (see minigpt4_b200_op_reply_stop); -1: no id ends the reply
    Error reply_stop(const int32_t *ids, int n, const char *stop, const char *tail, int32_t *stop_at);
    // the queued prompt rows of n (1..64, LlamaDevice::kMaxBatch) distinct contexts of one group in shared passes over the weights (see minigpt4_b200_flush_batch)
    static Error flush_batch(Engine *const *e, int n);
    // log-probability, rank and (logits non-NULL) logits of every id of a known continuation of n (1..64, LlamaDevice::kMaxBatch) distinct
    // contexts of one group, in shared passes over the weights (see minigpt4_b200_score_tokens); keep: the ids stay evaluated, as
    // b200_eval_tokens + flush leaves them; otherwise every context is left as it was.  All or nothing
    static Error score_tokens(Engine *const *e, int n, const int32_t *ids, const int32_t *n_ids, int keep, float *logprob, int32_t *rank, float *logits);
    // src's conversation into n (1..64, LlamaDevice::kMaxBatch) distinct other contexts of its group (see minigpt4_b200_session_copy):
    // src's queue is evaluated first; each destination gets n_past, K / V rows, logits, greedy id, device state and reply tail, loses its
    // queue and keeps its sampler.  kernel_ms (may be null): the copy kernel's CUDA-event time.  All or nothing
    static Error session_copy(Engine *src, Engine *const *dsts, int n, float *kernel_ms);
    // save / restore the conversation through host memory (see minigpt4_b200_state_save); state_size: -1 for a tensor-parallel context
    long long state_size() const;
    Error state_save(void *buf, long long cap, long long *written);
    Error state_load(const void *buf, long long size);
    Error encode_image(const ::MiniGPT4Image *image, ::MiniGPT4Embedding *out);
    static constexpr int kEncodeLanes = 8;
    Error encode_images(const ::MiniGPT4Image *images, size_t n, ::MiniGPT4Embedding *out, float *total_ms);   // batched: concurrent lanes
    Error add_tokens(const std::vector<int32_t> &tokens);
    Error add_strings(const char *s);
    Error add_embedding(const float *rows, int n_rows);
    int32_t sample_token(const SamplingArgs &p);
    const char *id_to_token(int32_t id) const;
    void reset() { n_past_ = 0; pend_ids_.clear(); pend_emb_.clear(); reply_clear(); }
    // the current reply's last LlamaDevice::kStopMax bytes (the reference's `chat` of a turn): a new turn or prompt clears it, every
    // fed id's text extends it, so a reply streamed over several sample_until calls stops where one call would.  The attached
    // constraint's state restarts and advances with it.
    void reply_clear() { reply_.clear(); cons_state_ = 0; }
    void reply_take(const char *text);
    void reply_take_id(int32_t id) { reply_take(id_to_token(id)); if (cons_) cons_state_ = cons_->next(cons_state_, id); }

    // constrained replies (minigpt4_b200_constraint_*): compile an automaton against this context's vocabulary, its tables on the device
    // counted in the group's shared bytes; null (and the reason logged) on bad input, a tensor-parallel context or exhausted device memory
    std::shared_ptr<Constraint> make_constraint(int n_states, const int32_t *next, const uint8_t *accept);
    // attach c (null: detach) with its state at the start; false for a constraint of another group
    bool constraint_attach(const std::shared_ptr<Constraint> &c);
    const Constraint *constraint() const { return cons_.get(); }
    int constraint_state() const { return cons_state_; }
    // the texts of every id, as minigpt4_end_chat returns them (the constraint compiler's vocabulary)
    std::vector<std::string> token_texts() const;
    bool flush();                     // evaluate the queued prompt rows (see add_tokens)
    static constexpr int kMaxPending = LlamaDevice::kPrefillMax;

    bool has_vision() const { return (bool)vis_; }
    VisionDevice *vision() { return vis_.get(); }
    LlamaDevice &llm() { return *llm_; }
    Tokenizer &tokenizer() { return *tok_; }
    int n_past() const { return n_past_; }
    void advance(int n) { n_past_ += n; }
    int n_embd_llm() const { return llm_->dims().n_embd; }
    float last_encode_ms = 0.f;
    TPLink tp;

private:
    static bool group_valid(Engine *const *e, int n, const char *what);   // 1..LlamaDevice::kMaxBatch distinct non-NULL contexts of one group
    static bool batch_valid(Engine *const *e, int n, const int32_t *ids);
    static bool flush_group(Engine *const *e, int n);
    static bool any_constrained(Engine *const *e, int n);
    // the handoff around a device sampling call: each context's device twin, position, generator, μ and constraint go to call, which
    // returns the device ms; afterwards context i's sampler takes back its generator and μ (settings p[i]), and its position and reply move
    // on by its fed[i] ids in ids_out[s * n + i] (fed is read after the call)
    // (call(L, n_past, rng, mu, cons): LlamaDevice's call over the arrays of the contexts' device twins and their state)
    template <class Call>
    static float device_sampling(Engine *const *e, int n, const SamplingArgs *p, const int32_t *fed, const int32_t *ids_out, Call call);
    // a history of n ids for the penalties: n >= 0, ids non-null if n > 0, every id in 0 .. n_vocab - 1
    static bool history_valid(const int32_t *ids, int n, int n_vocab, const char *what);
    // shared by the sessions of one model (the last context of the group frees them, lanes before lane 0)
    std::shared_ptr<VisionFile> vfile_;
    std::shared_ptr<VisionDevice> vis_;
    std::shared_ptr<std::vector<std::unique_ptr<VisionDevice>>> vis_lanes_ = std::make_shared<std::vector<std::unique_ptr<VisionDevice>>>();   // lanes 1.. of the batched encode (lane 0 = vis_)
    std::shared_ptr<Tokenizer> tok_ = std::make_shared<Tokenizer>();
    std::unique_ptr<LlamaDevice> llm_;
    std::unique_ptr<Sampler> sampler_;
    std::vector<float> logits_;
    int n_past_ = 0;
    std::vector<int32_t> pend_ids_;   // queued rows: token id, or -1 - k for row k of pend_emb_
    std::vector<float> pend_emb_;
    int pend_base_ = 0;               // position of the first queued row
    std::string reply_;
    std::shared_ptr<Constraint> cons_;   // the attached constraint (shared with the handle and other contexts) and its state here
    int cons_state_ = 0;
    void ensure_token_table();          // the group's device table of id_to_token (sample_until's stop rule)
    int n_batch_ = 512;
};

}  // namespace mg4

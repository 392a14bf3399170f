// text.h — host-side text logic of the language path: tokenizer and samplers.
// Semantics follow llama.cpp@master-31cfbb1 (llama_tokenizer, llama_sample_*), which the reference
// calls at minigpt4.cpp:2389 (llama_tokenize) and :2452-2477 (sampler chain).  Written fresh for this
// engine; the arithmetic-heavy part (logits) comes from the CUDA path, sampling stays on the host
// except greedy, which is an on-device arg-max.
#pragma once
#include "formats.h"
#include <random>
#include <unordered_map>

namespace mg4 {

class Tokenizer {
public:
    void init(const std::vector<LlamaVocabEntry> &vocab);
    // SentencePiece-style: UTF-8 characters merged greedily by best bigram score; unknown bytes -> id byte+3.
    // Empty text yields no tokens at all (not even BOS), like llama_tokenize.
    std::vector<int32_t> encode(const std::string &text, bool add_bos) const;
    const char *piece(int32_t id) const { return vocab_[(size_t)id].text.c_str(); }
    size_t size() const { return vocab_.size(); }
private:
    std::vector<LlamaVocabEntry> vocab_;
    std::unordered_map<std::string, int32_t> index_;
};

struct Candidate { int32_t id; float logit; float p; };

class Sampler {
public:
    explicit Sampler(int seed);
    // Mirrors MiniGPT4::sample_token (reference minigpt4.cpp:2425-2483).  Repeat/presence/frequency penalties
    // and penalize_nl are accepted by the ABI but never applied by the reference; same here (penalize() applies them on request:
    // minigpt4_b200_end_chat_penalized / sample_until_penalized).
    int32_t sample(const float *logits, int n_vocab, const SamplingArgs &p);
    // llama.cpp's repetition penalty, then its frequency and presence penalties, then main.cpp's penalize_nl, in place over the window
    // ids[0, n) (the caller's last repeat_last_n ids), as include/minigpt4_b200.h states them: for each id v with c >= 1 copies in the
    // window, z1 = repeat_penalty == 1 ? z : z <= 0 ? z * repeat_penalty : z / repeat_penalty, then z1 - (c * alpha_frequency +
    // alpha_presence) unless both alphas are 0; penalize_nl 0 with n_vocab > 13 leaves id 13 as it was.  Every operation rounds to float.
    static void penalize(float *logits, int n_vocab, const int32_t *ids, int n, float repeat_penalty, float alpha_presence, float alpha_frequency,
                         int penalize_nl);
    static int32_t greedy(const float *logits, int n_vocab);  // first arg-max
    // sample over the candidates ids[0, n) only (ascending ids: a constraint's allowed ids), in that order: the chain of sample() with
    // top_k <= 0 as n; temp <= 0: the first arg-max among them.  No mirostat.
    int32_t sample_allowed(const float *logits, const int32_t *ids, int n, const SamplingArgs &p);
    // individual stages (exposed for unit tests)
    static void top_k(std::vector<Candidate> &c, bool &sorted, int k, size_t min_keep);
    static void softmax(std::vector<Candidate> &c, bool &sorted);
    static void top_p(std::vector<Candidate> &c, bool &sorted, float p, size_t min_keep);
    static void tail_free(std::vector<Candidate> &c, bool &sorted, float z, size_t min_keep);
    static void typical(std::vector<Candidate> &c, bool &sorted, float p, size_t min_keep);
    static void temperature(std::vector<Candidate> &c, float t);
    int32_t draw(std::vector<Candidate> &c, bool &sorted);
    // the non-mirostat chain over the unsorted candidates c: top_k (k) -> tail_free -> typical -> top_p -> temperature -> draw
    int32_t chain(std::vector<Candidate> &c, int k, const SamplingArgs &p);
    // the generator's state through its textual representation (operator<< / >>): the 624 words, then the position in them
    void get_rng(uint32_t state[625]) const;
    void set_rng(const uint32_t state[625]);
    // mirostat's μ of v1 / v2, and whether each has been set by its mode's first use
    void get_mu(float mu[2], bool init[2]) const;
    void set_mu(const float mu[2], const bool init[2]);
private:
    std::mt19937 rng_;
    float mu_v1_ = 0, mu_v2_ = 0; bool mu_v1_init_ = false, mu_v2_init_ = false;
};

}  // namespace mg4

// text.cpp — tokenizer + samplers (see text.h).
#include "text.h"
#include <algorithm>
#include <math.h>
#include <numeric>
#include <queue>
#include <sstream>
#include <time.h>

namespace mg4 {

void Tokenizer::init(const std::vector<LlamaVocabEntry> &vocab) {
    vocab_ = vocab;
    index_.clear();
    index_.reserve(vocab.size() * 2);
    for (size_t i = 0; i < vocab.size(); ++i) index_[vocab[i].text] = (int32_t)i;  // later ids win, as in the loader loop
}

namespace {
struct Sym { int prev, next; size_t off, len; };
struct Bigram { int left, right; float score; size_t size; };
struct BigramLess {  // max-heap on score; equal score -> smaller left index first
    bool operator()(const Bigram &a, const Bigram &b) const { return a.score < b.score || (a.score == b.score && a.left > b.left); }
};
inline size_t utf8_len(unsigned char c) {
    static const unsigned char t[16] = {1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 2, 2, 3, 4};
    return t[c >> 4];
}
}  // namespace

std::vector<int32_t> Tokenizer::encode(const std::string &text, bool add_bos) const {
    std::vector<int32_t> out;
    if (text.empty()) return out;
    if (add_bos) out.push_back(1);
    std::vector<Sym> syms;
    for (size_t off = 0; off < text.size();) {
        size_t n = std::min(text.size() - off, utf8_len((unsigned char)text[off]));
        Sym s; s.off = off; s.len = n; s.prev = (int)syms.size() - 1; off += n;
        s.next = off == text.size() ? -1 : (int)syms.size() + 1;
        syms.push_back(s);
    }
    std::priority_queue<Bigram, std::vector<Bigram>, BigramLess> work;
    auto consider = [&](int l, int r) {
        if (l < 0 || r < 0) return;
        std::string piece = text.substr(syms[l].off, syms[l].len + syms[r].len);
        auto it = index_.find(piece);
        if (it == index_.end()) return;
        work.push(Bigram{l, r, vocab_[(size_t)it->second].score, piece.size()});
    };
    for (int i = 1; i < (int)syms.size(); ++i) consider(i - 1, i);
    while (!work.empty()) {
        Bigram b = work.top(); work.pop();
        Sym &L = syms[b.left], &R = syms[b.right];
        if (L.len == 0 || R.len == 0 || L.len + R.len != b.size) continue;  // stale entry
        L.len += R.len; R.len = 0;
        L.next = R.next;
        if (R.next >= 0) syms[R.next].prev = b.left;
        consider(L.prev, b.left);
        consider(b.left, L.next);
    }
    for (int i = 0; i != -1; i = syms[i].next) {
        const Sym &s = syms[i];
        auto it = index_.find(text.substr(s.off, s.len));
        if (it == index_.end()) { for (size_t j = 0; j < s.len; ++j) out.push_back((int32_t)(unsigned char)text[s.off + j] + 3); }
        else out.push_back(it->second);
    }
    return out;
}

// ------------------------------------------------------------------------------------------------
Sampler::Sampler(int seed) : rng_((uint32_t)(seed < 0 ? (int)time(nullptr) : seed)) {}

int32_t Sampler::greedy(const float *logits, int n) {
    int best = 0;
    for (int i = 1; i < n; ++i) if (logits[i] > logits[best]) best = i;
    return best;
}
static bool by_logit_desc(const Candidate &a, const Candidate &b) { return a.logit > b.logit; }

void Sampler::top_k(std::vector<Candidate> &c, bool &sorted, int k, size_t min_keep) {
    k = std::max(k, (int)min_keep);
    k = std::min(k, (int)c.size());
    if (!sorted) {
        if (k == (int)c.size()) std::sort(c.begin(), c.end(), by_logit_desc);
        else std::partial_sort(c.begin(), c.begin() + k, c.end(), by_logit_desc);
        sorted = true;
    }
    c.resize((size_t)k);
}
void Sampler::softmax(std::vector<Candidate> &c, bool &sorted) {
    if (!sorted) { std::sort(c.begin(), c.end(), by_logit_desc); sorted = true; }
    const float mx = c[0].logit; float sum = 0.f;
    for (auto &x : c) { x.p = expf(x.logit - mx); sum += x.p; }
    for (auto &x : c) x.p /= sum;
}
void Sampler::top_p(std::vector<Candidate> &c, bool &sorted, float p, size_t min_keep) {
    if (p >= 1.0f) return;
    softmax(c, sorted);
    float cum = 0.f; size_t last = c.size();
    for (size_t i = 0; i < c.size(); ++i) { cum += c[i].p; if (cum >= p && i + 1 >= min_keep) { last = i + 1; break; } }
    c.resize(last);
}
void Sampler::tail_free(std::vector<Candidate> &c, bool &sorted, float z, size_t min_keep) {
    if (z >= 1.0f || c.size() <= 2) return;
    softmax(c, sorted);
    std::vector<float> d1(c.size() - 1), d2(c.size() - 2);
    for (size_t i = 0; i < d1.size(); ++i) d1[i] = c[i].p - c[i + 1].p;
    for (size_t i = 0; i < d2.size(); ++i) d2[i] = fabsf(d1[i] - d1[i + 1]);
    float s = std::accumulate(d2.begin(), d2.end(), 0.0f);
    for (float &v : d2) v /= s;
    float cum = 0.f; size_t last = c.size();
    for (size_t i = 0; i < d2.size(); ++i) { cum += d2[i]; if (cum > z && i >= min_keep) { last = i; break; } }
    c.resize(last);
}
void Sampler::typical(std::vector<Candidate> &c, bool &sorted, float p, size_t min_keep) {
    if (p >= 1.0f) return;
    softmax(c, sorted);
    float entropy = 0.f;
    for (auto &x : c) entropy += -x.p * logf(x.p);
    std::vector<float> shifted(c.size());
    for (size_t i = 0; i < c.size(); ++i) shifted[i] = fabsf(-logf(c[i].p) - entropy);
    std::vector<size_t> idx(c.size());
    std::iota(idx.begin(), idx.end(), 0);
    std::sort(idx.begin(), idx.end(), [&](size_t a, size_t b) { return shifted[a] < shifted[b]; });
    float cum = 0.f; size_t last = idx.size();
    for (size_t i = 0; i < idx.size(); ++i) { cum += c[idx[i]].p; if (cum > p && i >= min_keep - 1) { last = i + 1; break; } }
    std::vector<Candidate> kept; kept.reserve(last);
    for (size_t i = 0; i < last; ++i) kept.push_back(c[idx[i]]);
    c.swap(kept);
    sorted = false;
}
void Sampler::temperature(std::vector<Candidate> &c, float t) { for (auto &x : c) x.logit /= t; }

int32_t Sampler::draw(std::vector<Candidate> &c, bool &sorted) {
    softmax(c, sorted);
    std::vector<float> probs; probs.reserve(c.size());
    for (auto &x : c) probs.push_back(x.p);
    std::discrete_distribution<> dist(probs.begin(), probs.end());
    return c[(size_t)dist(rng_)].id;
}

void Sampler::get_rng(uint32_t state[625]) const {
    std::stringstream ss;
    ss << rng_;
    for (int i = 0; i < 625; ++i) ss >> state[i];
}
void Sampler::set_rng(const uint32_t state[625]) {
    std::stringstream ss;
    for (int i = 0; i < 625; ++i) ss << state[i] << ' ';
    ss >> rng_;
}
void Sampler::get_mu(float mu[2], bool init[2]) const { mu[0] = mu_v1_; mu[1] = mu_v2_; init[0] = mu_v1_init_; init[1] = mu_v2_init_; }
void Sampler::set_mu(const float mu[2], const bool init[2]) { mu_v1_ = mu[0]; mu_v2_ = mu[1]; mu_v1_init_ = init[0]; mu_v2_init_ = init[1]; }

int32_t Sampler::sample(const float *logits, int n_vocab, const SamplingArgs &sp) {
    if (sp.temp <= 0) return greedy(logits, n_vocab);
    std::vector<Candidate> c((size_t)n_vocab);
    for (int i = 0; i < n_vocab; ++i) c[(size_t)i] = Candidate{i, logits[i], 0.f};
    bool sorted = false;
    const int k = sp.top_k <= 0 ? n_vocab : sp.top_k;
    auto surprise_of = [&](int32_t id) { for (auto &x : c) if (x.id == id) return -log2f(x.p); return 0.f; };
    if (sp.mirostat == 1) {
        if (!mu_v1_init_) { mu_v1_ = 2.0f * sp.mirostat_tau; mu_v1_init_ = true; }  // function-local static in the reference (:2458)
        temperature(c, sp.temp);
        softmax(c, sorted);
        const int m = 100; float s_tb = 0.f, s_tt = 0.f;
        for (size_t i = 0; i < (size_t)(m - 1) && i + 1 < c.size(); ++i) {
            float t = logf((float)(i + 2) / (float)(i + 1)), b = logf(c[i].p / c[i + 1].p);
            s_tb += t * b; s_tt += t * t;
        }
        float s_hat = s_tb / s_tt, eps = s_hat - 1;
        float kf = powf((eps * powf(2, mu_v1_)) / (1 - powf((float)n_vocab, -eps)), 1 / s_hat);
        top_k(c, sorted, (int)kf, 1);
        int32_t id = draw(c, sorted);
        mu_v1_ -= sp.mirostat_eta * (surprise_of(id) - sp.mirostat_tau);
        return id;
    }
    if (sp.mirostat == 2) {
        if (!mu_v2_init_) { mu_v2_ = 2.0f * sp.mirostat_tau; mu_v2_init_ = true; }
        temperature(c, sp.temp);
        softmax(c, sorted);
        size_t keep = 0;
        while (keep < c.size() && -log2f(c[keep].p) <= mu_v2_) ++keep;
        c.resize(std::max<size_t>(keep, 1));
        int32_t id = draw(c, sorted);
        mu_v2_ -= sp.mirostat_eta * (surprise_of(id) - sp.mirostat_tau);
        return id;
    }
    return chain(c, k, sp);
}

void Sampler::penalize(float *logits, int n_vocab, const int32_t *ids, int n, float repeat_penalty, float alpha_presence, float alpha_frequency,
                       int penalize_nl) {
    std::vector<int> count((size_t)n_vocab, 0);
    for (int j = 0; j < n; ++j) ++count[(size_t)ids[j]];
    const bool keep_nl = !penalize_nl && n_vocab > 13;
    for (int j = 0; j < n; ++j) {
        const int v = ids[j];
        const int c = count[(size_t)v];
        if (c == 0 || (keep_nl && v == 13)) continue;   // (an id seen before in the window is done)
        count[(size_t)v] = 0;
        const float z = logits[v];
        const float z1 = repeat_penalty == 1.0f ? z : (z <= 0 ? z * repeat_penalty : z / repeat_penalty);
        logits[v] = (alpha_frequency == 0 && alpha_presence == 0) ? z1 : z1 - ((float)c * alpha_frequency + alpha_presence);
    }
}

int32_t Sampler::chain(std::vector<Candidate> &c, int k, const SamplingArgs &sp) {
    bool sorted = false;
    top_k(c, sorted, k, 1);
    tail_free(c, sorted, sp.tfs_z, 1);
    typical(c, sorted, sp.typical_p, 1);
    top_p(c, sorted, sp.top_p, 1);
    temperature(c, sp.temp);
    return draw(c, sorted);
}

int32_t Sampler::sample_allowed(const float *logits, const int32_t *ids, int n, const SamplingArgs &sp) {
    if (sp.temp <= 0) {   // the first arg-max over the allowed ids, which are ascending: the lower id on ties
        int best = 0;
        for (int j = 1; j < n; ++j) if (logits[ids[j]] > logits[ids[best]]) best = j;
        return ids[best];
    }
    std::vector<Candidate> c((size_t)n);
    for (int j = 0; j < n; ++j) c[(size_t)j] = Candidate{ids[j], logits[ids[j]], 0.f};
    return chain(c, sp.top_k <= 0 ? n : sp.top_k, sp);
}

}  // namespace mg4

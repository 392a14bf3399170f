// api.cpp — the C ABI of libminigpt4.so: the reference's 18 entry points (include/minigpt4.h, mirroring reference
// minigpt4.cpp:2543-2987) plus the extensions (include/minigpt4_b200.h).
#include "../../include/minigpt4_b200.h"
#include "engine.h"
#include "image.h"
#include <stddef.h>
#include <string.h>
#include <sys/stat.h>
#include <exception>
#include <math.h>
#include <algorithm>
#include <thread>
#include <string>

using namespace mg4;

namespace {
Engine *E(struct MiniGPT4Context *c) { return reinterpret_cast<Engine *>(c); }
bool path_exists(const char *p) { struct stat st; return p && stat(p, &st) == 0; }
// prompt constants: reference minigpt4.cpp:139-141
const char *kSystemPrompt = "Give the following image: <Img>ImageContent</Img>. You will be able to see the image once I provide it to you. Please answer my questions.###";
const char *kEosTokenSuffix = "##";
const char *kEosSuffix = "###";

// allowed(state) as the ABI reports it: the finished state's index as -1
int allowed_of(const Constraint &c, int state, int32_t *ids, int32_t *next_states, int cap) {
    if (state < 0 || state >= c.n_states) return -1;
    const int m = c.row_size(state);
    if (m == 0) return -1;   // a state that is not live
    if (cap < m) return -m;
    const int32_t *r = c.row(state);
    for (int j = 0; j < m; ++j) {
        if (ids) ids[j] = r[2 * j];
        if (next_states) next_states[j] = r[2 * j + 1] == c.finished() ? -1 : r[2 * j + 1];
    }
    return m;
}
}  // namespace

// a constraint handle: one reference to the compiled tables (constraint.h); each attached context holds another
struct MiniGPT4B200Constraint { std::shared_ptr<Constraint> c; };

extern "C" {

struct MiniGPT4Context *minigpt4_model_load(const char *path, const char *llm_model, int verbosity, int seed, int n_ctx, int n_batch, bool numa) {
    g_verbosity = verbosity;
    const double t0 = now_ms();
    if (!path_exists(path)) { MG4_ERR("%s does not exist", path ? path : "(null)"); return nullptr; }
    if (!path_exists(llm_model)) { MG4_ERR("%s does not exist", llm_model ? llm_model : "(null)"); return nullptr; }
    Engine *e = new Engine();
    if (Error err = e->init(path, llm_model, verbosity, seed, n_ctx, n_batch, numa)) {
        MG4_ERR("Failed to initialize MiniGPT4: %s", error_name(err));
        delete e;
        return nullptr;
    }
    MG4_INFO("Load model from file took %.0f ms", now_ms() - t0);
    return reinterpret_cast<struct MiniGPT4Context *>(e);
}

// Image file -> 8-bit RGB (reference minigpt4.cpp:2576-2596: cv::imread(IMREAD_COLOR) + BGR2RGB, compiled only with OpenCV - its default build
// returns OpenCVNotLinked).  Decoded here without third-party code: PNG, JPEG and binary PPM / PGM (csrc/image.cpp, csrc/jpeg.cpp); anything else is OpenImage.
// Pixel buffers of MiniGPT4Image are float-array allocations whatever they hold, because minigpt4_free_image releases them as such (:2790-2798).
int minigpt4_image_load_from_file(struct MiniGPT4Context *, const char *path, struct MiniGPT4Image *image, int) {
    if (!image) return ErrOpenImage;
    try {
        RgbImage im; std::string err;
        if (!decode_image_file(path, im, err)) { MG4_ERR("%s: %s", path ? path : "(null)", err.c_str()); return ErrOpenImage; }
        const size_t bytes = im.px.size();
        float *buf = new float[(bytes + 3) / 4];
        memcpy(buf, im.px.data(), bytes);
        image->data = buf; image->width = im.w; image->height = im.h; image->channels = 3; image->format = MINIGPT4_IMAGE_FORMAT_U8;
        return ErrNone;
    } catch (const std::exception &e) {   // (an image that does not fit in host memory must not unwind through the C ABI)
        MG4_ERR("%s: %s", path ? path : "(null)", e.what());
        return ErrOpenImage;
    }
}

// 8-bit RGB of any size -> the encoder's input (reference :2598-2651): Pillow-bicubic resize to 224 x 224, / 255, CLIP mean / std, planar CHW.
// The reference describes the result as a 1 x 150528 single-channel image (it reports the shape of its concatenated planes, :2639-2641);
// minigpt4_encode_image only checks the element count (:2130), and the same description is returned here.
int minigpt4_preprocess_image(struct MiniGPT4Context *, const struct MiniGPT4Image *image, struct MiniGPT4Image *preprocessed_image, int) {
    if (!image || !preprocessed_image || !image->data) return ErrOpenImage;
    if (image->channels != 3) { MG4_ERR("Image must have 3 channels"); return ErrImageChannelsExpectedRGB; }
    if (image->format != MINIGPT4_IMAGE_FORMAT_U8) { MG4_ERR("Image must be in U8 format"); return ErrImageFormatExpectedU8; }
    if (image->width <= 0 || image->height <= 0 || image->width > 32768 || image->height > 32768) return ErrImageSize;
    float *out = nullptr;
    try {
        std::vector<uint8_t> small((size_t)224 * 224 * 3);
        resize_bicubic_u8((const uint8_t *)image->data, image->width, image->height, small.data(), 224, 224);
        out = new float[(size_t)3 * 224 * 224];
        normalize_to_chw(small.data(), 224, 224, out);
    } catch (const std::exception &e) {
        MG4_ERR("preprocess: %s", e.what());
        delete[] out;
        return ErrImageSize;
    }
    preprocessed_image->data = out; preprocessed_image->width = 1; preprocessed_image->height = 3 * 224 * 224; preprocessed_image->channels = 1;
    preprocessed_image->format = MINIGPT4_IMAGE_FORMAT_F32;
    return ErrNone;
}

int minigpt4_encode_image(struct MiniGPT4Context *ctx, struct MiniGPT4Image *image, struct MiniGPT4Embedding *embedding, size_t /*n_threads: CPU notion, ignored*/) {
    return E(ctx)->encode_image(image, embedding);
}

int minigpt4_begin_chat_image(struct MiniGPT4Context *ctx, struct MiniGPT4Embedding *image_embedding, const char *s, size_t) {
    Engine *e = E(ctx);
    e->reply_clear();
    if (Error err = e->add_strings("Human: <Img>")) return err;
    if (image_embedding->elements != 32u * 5120u && image_embedding->elements != 32u * 4096u) {
        MG4_ERR("LLAMA projection image embedding size not valid: %zu", image_embedding->elements);
        return ErrLLamaProjectionEmbeddingInvalidSize;
    }
    if (Error err = e->add_embedding(image_embedding->data, 32)) { MG4_ERR("Failed to add image embedding: %s", error_name(err)); return err; }
    if (Error err = e->add_strings("</Img> ")) return err;
    if (Error err = e->add_strings(s)) return err;
    if (Error err = e->add_strings("### Assistant:")) return err;
    return ErrNone;
}

int minigpt4_end_chat_image(struct MiniGPT4Context *ctx, const char **token, size_t, float temp, int32_t top_k, float top_p, float tfs_z, float typical_p,
                            int32_t /*repeat_last_n*/, float /*repeat_penalty*/, float /*alpha_presence*/, float /*alpha_frequency*/, int mirostat,
                            float mirostat_tau, float mirostat_eta, int /*penalize_nl*/) {
    Engine *e = E(ctx);
    if (e->constraint() && (mirostat == 1 || mirostat == 2)) { MG4_ERR("end_chat: mirostat on a constrained context"); return ErrFailedToAddString; }
    SamplingArgs sp{temp, top_k, top_p, tfs_z, typical_p, mirostat, mirostat_tau, mirostat_eta};
    const int32_t id = e->sample_token(sp);
    *token = e->id_to_token(id);
    e->add_tokens({id});  // the reference ignores this return value too (minigpt4.cpp:2715)
    e->reply_take_id(id);
    return ErrNone;
}

int minigpt4_system_prompt(struct MiniGPT4Context *ctx, size_t) { E(ctx)->reply_clear(); return E(ctx)->add_strings(kSystemPrompt); }

int minigpt4_begin_chat(struct MiniGPT4Context *ctx, const char *s, size_t) {
    Engine *e = E(ctx);
    e->reply_clear();
    if (Error err = e->add_strings("Human: ")) return err;
    if (Error err = e->add_strings(s)) return err;
    if (Error err = e->add_strings("### Assistant:")) return err;
    return ErrNone;
}

int minigpt4_end_chat(struct MiniGPT4Context *ctx, const char **token, size_t n_threads, float temp, int32_t top_k, float top_p, float tfs_z, float typical_p,
                      int32_t repeat_last_n, float repeat_penalty, float alpha_presence, float alpha_frequency, int mirostat, float mirostat_tau,
                      float mirostat_eta, int penalize_nl) {
    return minigpt4_end_chat_image(ctx, token, n_threads, temp, top_k, top_p, tfs_z, typical_p, repeat_last_n, repeat_penalty, alpha_presence, alpha_frequency,
                                   mirostat, mirostat_tau, mirostat_eta, penalize_nl);
}

int minigpt4_reset_chat(struct MiniGPT4Context *ctx) { E(ctx)->reset(); return ErrNone; }

// (the reference dereferences a null argument in the next five entry points; here a null is simply "nothing to do")
int minigpt4_contains_eos_token(const char *s) { return (s && strcmp(s, kEosTokenSuffix) == 0) ? ErrEosToken : ErrNone; }
int minigpt4_is_eos(const char *s) {
    if (!s) return ErrNone;
    const size_t n = strlen(s), m = strlen(kEosSuffix);
    return (n >= m && memcmp(s + n - m, kEosSuffix, m) == 0) ? ErrEos : ErrNone;
}

int minigpt4_free(struct MiniGPT4Context *ctx) { delete E(ctx); return ErrNone; }
int minigpt4_free_image(struct MiniGPT4Image *image) {
    if (image && image->data) { delete[] (float *)image->data; image->data = nullptr; }
    return ErrNone;
}
int minigpt4_free_embedding(struct MiniGPT4Embedding *embedding) {
    if (embedding && embedding->data) { delete[] embedding->data; embedding->data = nullptr; }
    return ErrNone;
}
const char *minigpt4_error_code_to_string(int error_code) { return error_name(error_code); }
void minigpt4_set_verbosity(int verbosity) { g_verbosity = verbosity; }

// quantize.cpp
int mg4_quantize_container(const char *in_path, const char *out_path, int data_type);
int minigpt4_quantize_model(const char *in_path, const char *out_path, int data_type) {
    if (!in_path || !out_path || !path_exists(in_path)) return ErrPathDoesNotExist;
    return mg4_quantize_container(in_path, out_path, data_type);
}

// ------------------------------------------------------------------------------------------------
// extensions (include/minigpt4_b200.h)
// ------------------------------------------------------------------------------------------------
int minigpt4_b200_device_count(void) { int n = 0; return cudaGetDeviceCount(&n) == cudaSuccess ? n : 0; }
int minigpt4_b200_set_device(int device) { return cudaSetDevice(device) == cudaSuccess ? 0 : 1; }
int minigpt4_b200_tp_unique_id(void *out128) { return TPLink::unique_id(out128) ? 0 : 1; }
int minigpt4_b200_tp_configure(int rank, int world, const void *id128) {
    g_tp_config.set = world > 1; g_tp_config.rank = rank; g_tp_config.world = world;
    if (id128) memcpy(g_tp_config.id, id128, 128);
    return 0;
}
struct MiniGPT4Context *minigpt4_b200_llm_load(const char *llm_model, int n_ctx, int seed, int verbosity) {
    g_verbosity = verbosity;
    if (!path_exists(llm_model)) { MG4_ERR("%s does not exist", llm_model ? llm_model : "(null)"); return nullptr; }
    Engine *e = new Engine();
    if (Error err = e->init("", llm_model, verbosity, seed, n_ctx, 512, false)) { MG4_ERR("Failed to initialize: %s", error_name(err)); delete e; return nullptr; }
    return reinterpret_cast<struct MiniGPT4Context *>(e);
}
int minigpt4_b200_n_vocab(struct MiniGPT4Context *ctx) { return E(ctx)->llm().dims().n_vocab; }
int minigpt4_b200_n_embd(struct MiniGPT4Context *ctx) { return E(ctx)->llm().dims().n_embd; }
int minigpt4_b200_n_past(struct MiniGPT4Context *ctx) { return E(ctx)->n_past(); }
int minigpt4_b200_tokenize(struct MiniGPT4Context *ctx, const char *text, int add_bos, int32_t *out, int max_tokens) {
    std::vector<int32_t> t = E(ctx)->tokenizer().encode(text ? text : "", add_bos != 0);
    if ((int)t.size() > max_tokens) return -(int)t.size();  // llama_tokenize convention
    memcpy(out, t.data(), t.size() * sizeof(int32_t));
    return (int)t.size();
}
int minigpt4_b200_eval_tokens(struct MiniGPT4Context *ctx, const int32_t *ids, int n) {
    E(ctx)->reply_clear();
    return n <= 0 ? 0 : E(ctx)->add_tokens(std::vector<int32_t>(ids, ids + n));
}
int minigpt4_b200_eval_embd(struct MiniGPT4Context *ctx, const float *rows, int n) { E(ctx)->reply_clear(); return E(ctx)->add_embedding(rows, n); }
int minigpt4_b200_flush(struct MiniGPT4Context *ctx) { return E(ctx)->flush() ? 0 : ErrFailedToAddString; }
int minigpt4_b200_get_logits(struct MiniGPT4Context *ctx, float *out) { E(ctx)->flush(); E(ctx)->llm().logits_to_host(out); return 0; }
int minigpt4_b200_greedy_id(struct MiniGPT4Context *ctx) { E(ctx)->flush(); return E(ctx)->llm().argmax(); }
int minigpt4_b200_get_hidden(struct MiniGPT4Context *ctx, float *out, int n_rows) { E(ctx)->flush(); E(ctx)->llm().hidden_to_host(out, n_rows); return 0; }
const char *minigpt4_b200_token_text(struct MiniGPT4Context *ctx, int32_t id) { return E(ctx)->id_to_token(id); }
int minigpt4_b200_decode_chain(struct MiniGPT4Context *ctx, int steps, int32_t *ids_out, float *ms_out) {
    Engine *e = E(ctx);
    if (e->constraint()) { MG4_ERR("decode_chain: a constrained context"); return ErrFailedToAddString; }
    if (!e->flush()) return ErrFailedToAddString;
    const float ms = e->llm().decode_chain(steps, e->n_past(), ids_out);
    if (ms < 0) return ErrFailedToAddString;
    e->advance(steps);
    if (ms_out) *ms_out = ms;
    return 0;
}
struct MiniGPT4Context *minigpt4_b200_session_create(struct MiniGPT4Context *ctx, int seed) {
    if (!ctx) return nullptr;
    Engine *e = new Engine();
    if (Error err = e->init_session(*E(ctx), seed)) { MG4_ERR("Failed to create a session: %s", error_name(err)); delete e; return nullptr; }
    return reinterpret_cast<struct MiniGPT4Context *>(e);
}
int minigpt4_b200_session_info(struct MiniGPT4Context *ctx, int *n_contexts, double *owned_bytes, double *shared_bytes) {
    if (!ctx) return ErrLoadLanguageModel;
    const LlamaDevice &l = E(ctx)->llm();
    if (n_contexts) *n_contexts = l.group_size();
    if (owned_bytes) *owned_bytes = (double)l.owned_bytes();
    if (shared_bytes) *shared_bytes = (double)l.shared_bytes();
    return 0;
}
int minigpt4_b200_decode_batch(struct MiniGPT4Context **ctxs, int n, const int32_t *ids, int32_t *ids_out) {
    for (int i = 0; ctxs && i < n && i < LlamaDevice::kMaxBatch; ++i)
        if (ctxs[i] && E(ctxs[i])->constraint()) { MG4_ERR("decode_batch: context %d is constrained", i); return ErrFailedToAddString; }
    return Engine::decode_batch(reinterpret_cast<Engine *const *>(ctxs), n, ids, ids_out);
}
int minigpt4_b200_flush_batch(struct MiniGPT4Context **ctxs, int n) { return Engine::flush_batch(reinterpret_cast<Engine *const *>(ctxs), n); }
int minigpt4_b200_score_tokens(struct MiniGPT4Context **ctxs, int n, const int32_t *ids, const int32_t *n_ids, int keep, float *logprob_out,
                               int32_t *rank_out, float *logits_out) {
    return Engine::score_tokens(reinterpret_cast<Engine *const *>(ctxs), n, ids, n_ids, keep, logprob_out, rank_out, logits_out);
}
int minigpt4_b200_session_copy(struct MiniGPT4Context *src, struct MiniGPT4Context **dsts, int n) {
    return minigpt4_b200_session_copy_timed(src, dsts, n, nullptr);
}
int minigpt4_b200_session_copy_timed(struct MiniGPT4Context *src, struct MiniGPT4Context **dsts, int n, float *kernel_ms) {
    return Engine::session_copy(E(src), reinterpret_cast<Engine *const *>(dsts), n, kernel_ms);
}
long long minigpt4_b200_state_size(struct MiniGPT4Context *ctx) { return ctx ? E(ctx)->state_size() : -1; }
int minigpt4_b200_state_save(struct MiniGPT4Context *ctx, void *buf, long long cap, long long *written) {
    return ctx ? E(ctx)->state_save(buf, cap, written) : ErrFailedToAddString;
}
int minigpt4_b200_state_load(struct MiniGPT4Context *ctx, const void *buf, long long size) {
    return ctx ? E(ctx)->state_load(buf, size) : ErrFailedToAddString;
}
int minigpt4_b200_end_chat_batch(struct MiniGPT4Context **ctxs, int n, const char **tokens, float temp, int32_t top_k, float top_p, float tfs_z,
                                 float typical_p, int32_t /*repeat_last_n*/, float /*repeat_penalty*/, float /*alpha_presence*/,
                                 float /*alpha_frequency*/, int mirostat, float mirostat_tau, float mirostat_eta, int /*penalize_nl*/) {
    SamplingArgs sp{temp, top_k, top_p, tfs_z, typical_p, mirostat, mirostat_tau, mirostat_eta};
    return Engine::end_chat_batch(reinterpret_cast<Engine *const *>(ctxs), n, tokens, sp);
}
int minigpt4_b200_sample_steps(struct MiniGPT4Context **ctxs, int n, int steps, float temp, int32_t top_k, float top_p, float tfs_z, float typical_p,
                               int32_t *ids_out, float *ms_out) {
    if (!ctxs) return ErrFailedToAddString;
    return Engine::sample_steps(reinterpret_cast<Engine *const *>(ctxs), n, steps, SamplingArgs{temp, top_k, top_p, tfs_z, typical_p}, ids_out, ms_out);
}
// the settings of one context of a uniform reply call: the same for every context (n clamped: Engine::sample_until refuses n outside
// 1 .. kMaxBatch before it reads them), neutral penalties unless set afterwards
static std::vector<UntilArgs> uniform_until(int n, int max_steps, const char *stop, const SamplingArgs &p) {
    const UntilArgs u{p, max_steps, stop ? stop : "###", PenaltyParams{0, 1.f, 0.f, 0.f, 1}, nullptr, 0};   // (NULL stop: the reference's EOS_SUFFIX)
    return std::vector<UntilArgs>((size_t)std::max(1, std::min(n, LlamaDevice::kMaxBatch)), u);
}
int minigpt4_b200_sample_until(struct MiniGPT4Context **ctxs, int n, int max_steps, const char *stop, float temp, int32_t top_k, float top_p,
                               float tfs_z, float typical_p, int32_t *ids_out, int32_t *n_out, int32_t *stopped, float *ms_out) {
    if (!ctxs) return ErrFailedToAddString;
    const std::vector<UntilArgs> u = uniform_until(n, max_steps, stop, SamplingArgs{temp, top_k, top_p, tfs_z, typical_p});
    return Engine::sample_until(reinterpret_cast<Engine *const *>(ctxs), n, u.data(), ids_out, n_out, stopped, ms_out);
}
int minigpt4_b200_beam_search(struct MiniGPT4Context **ctxs, int n_beams, int max_steps, const char *stop, float length_penalty, int n_hyp,
                              int32_t *ids_out, int32_t *n_out, float *score_out, float *logprob_out, int32_t *stopped, float *ms_out) {
    return Engine::beam_search(reinterpret_cast<Engine *const *>(ctxs), n_beams, max_steps, stop, length_penalty, n_hyp, ids_out, n_out, score_out,
                               logprob_out, stopped, ms_out);
}
int minigpt4_b200_op_beam_rank(const float *logits, int n_live, const float *S, int n_beams, int n_vocab, int32_t *parent_out, int32_t *id_out,
                               float *c_out) {
    if (!logits || !S || !parent_out || !id_out || !c_out || n_beams < 1 || n_beams > LlamaDevice::kMaxBeams || n_live < 1 || n_live > n_beams ||
        n_vocab < 1)
        return ErrFailedToAddString;
    return LlamaDevice::test_beam_rank(logits, n_live, S, n_beams, n_vocab, parent_out, id_out, c_out) >= 0 ? 0 : ErrFailedToAddString;
}
int minigpt4_b200_sample_steps_mirostat(struct MiniGPT4Context **ctxs, int n, int steps, float temp, int mirostat, float mirostat_tau,
                                        float mirostat_eta, int32_t *ids_out, float *ms_out) {
    if (!ctxs || (mirostat != 1 && mirostat != 2)) return ErrFailedToAddString;
    return Engine::sample_steps(reinterpret_cast<Engine *const *>(ctxs), n, steps, sampling_args(temp, 0, 1.f, 1.f, 1.f, mirostat, mirostat_tau, mirostat_eta),
                                ids_out, ms_out);
}
int minigpt4_b200_sample_until_mirostat(struct MiniGPT4Context **ctxs, int n, int max_steps, const char *stop, float temp, int mirostat,
                                        float mirostat_tau, float mirostat_eta, int32_t *ids_out, int32_t *n_out, int32_t *stopped, float *ms_out) {
    if (!ctxs || (mirostat != 1 && mirostat != 2)) return ErrFailedToAddString;
    const std::vector<UntilArgs> u = uniform_until(n, max_steps, stop, sampling_args(temp, 0, 1.f, 1.f, 1.f, mirostat, mirostat_tau, mirostat_eta));
    return Engine::sample_until(reinterpret_cast<Engine *const *>(ctxs), n, u.data(), ids_out, n_out, stopped, ms_out);
}
int minigpt4_b200_sample_until_logprobs(struct MiniGPT4Context **ctxs, int n, int max_steps, const char *stop, float temp, int32_t top_k,
                                        float top_p, float tfs_z, float typical_p, int mirostat, float mirostat_tau, float mirostat_eta, int top_n,
                                        int32_t *ids_out, int32_t *n_out, int32_t *stopped, float *logprob_out, int32_t *rank_out,
                                        int32_t *top_ids_out, float *top_logprob_out, float *ms_out) {
    if (!ctxs) return ErrFailedToAddString;
    // the sampling arguments of the call this one stands for
    const SamplingArgs p = sampling_args(temp, top_k, top_p, tfs_z, typical_p, mirostat, mirostat_tau, mirostat_eta);
    const LogprobRequest rec{top_n, logprob_out, rank_out, top_ids_out, top_logprob_out};
    const std::vector<UntilArgs> u = uniform_until(n, max_steps, stop, p);
    return Engine::sample_until(reinterpret_cast<Engine *const *>(ctxs), n, u.data(), ids_out, n_out, stopped, ms_out, &rec, "sample_until_logprobs");
}
int minigpt4_b200_op_logprobs(const float *logits, int rows, int n_vocab, const int32_t *ids, int top_n, float *logprob_out, int32_t *rank_out,
                              int32_t *top_ids_out, float *top_logprob_out, float *kernel_ms) {
    if (!logits || !ids || !logprob_out || rows < 1 || rows > LlamaDevice::kMaxBatch || n_vocab < 1 || top_n < 0 ||
        top_n > LlamaDevice::kLogprobTop || (top_n > 0 && !top_ids_out))
        return ErrFailedToAddString;
    for (int r = 0; r < rows; ++r) if (ids[r] < 0 || ids[r] >= n_vocab) return ErrFailedToAddString;
    LlamaDevice::test_logprobs(logits, rows, n_vocab, ids, LogprobRequest{top_n, logprob_out, rank_out, top_ids_out, top_logprob_out}, kernel_ms);
    return 0;
}
int minigpt4_b200_sample_until_penalized(struct MiniGPT4Context **ctxs, int n, int max_steps, const char *stop, float temp, int32_t top_k,
                                         float top_p, float tfs_z, float typical_p, int mirostat, float mirostat_tau, float mirostat_eta,
                                         int32_t repeat_last_n, float repeat_penalty, float alpha_presence, float alpha_frequency, int penalize_nl,
                                         const int32_t *last_ids, const int32_t *n_last, int32_t *ids_out, int32_t *n_out, int32_t *stopped,
                                         float *ms_out) {
    if (!ctxs) return ErrFailedToAddString;
    // the sampling arguments of the call this one stands for
    const SamplingArgs p = sampling_args(temp, top_k, top_p, tfs_z, typical_p, mirostat, mirostat_tau, mirostat_eta);
    std::vector<UntilArgs> u = uniform_until(n, max_steps, stop, p);
    size_t at = 0;   // context i's history: its n_last[i] ids after those of contexts 0 .. i-1
    for (int i = 0; i < (int)u.size() && i < n; ++i) {
        u[(size_t)i].q = PenaltyParams{repeat_last_n, repeat_penalty, alpha_presence, alpha_frequency, penalize_nl};
        u[(size_t)i].n_last = n_last ? n_last[i] : 0;
        u[(size_t)i].last_ids = last_ids ? last_ids + at : nullptr;
        at += (size_t)std::max(0, u[(size_t)i].n_last);
    }
    return Engine::sample_until(reinterpret_cast<Engine *const *>(ctxs), n, u.data(), ids_out, n_out, stopped, ms_out, nullptr, "sample_until_penalized");
}
static_assert(sizeof(MiniGPT4B200GenParams) == 80 && offsetof(MiniGPT4B200GenParams, stop) == 8 && offsetof(MiniGPT4B200GenParams, penalize_nl) == 64 &&
                  offsetof(MiniGPT4B200GenParams, last_ids) == 72, "the layout include/minigpt4_b200.h states");
int minigpt4_b200_generate_batch(struct MiniGPT4Context **ctxs, int n, const struct MiniGPT4B200GenParams *params, int top_n, int32_t *ids_out,
                                 int32_t *n_out, int32_t *stopped, float *logprob_out, int32_t *rank_out, int32_t *top_ids_out, float *top_logprob_out,
                                 float *ms_out) {
    if (!ctxs || !params) { MG4_ERR("generate_batch: NULL contexts or params"); return ErrFailedToAddString; }
    if (n < 1 || n > LlamaDevice::kMaxBatch) { MG4_ERR("generate_batch: %d contexts (1 .. %d)", n, LlamaDevice::kMaxBatch); return ErrFailedToAddString; }
    if (!logprob_out && top_n != 0) { MG4_ERR("generate_batch: top_n %d without records", top_n); return ErrFailedToAddString; }
    std::vector<UntilArgs> u((size_t)n);
    for (int i = 0; i < n; ++i) {
        const MiniGPT4B200GenParams &g = params[i];
        if (g.size != (int32_t)sizeof(MiniGPT4B200GenParams)) {
            MG4_ERR("generate_batch: params[%d].size %d (%zu)", i, g.size, sizeof(MiniGPT4B200GenParams)); return ErrFailedToAddString;
        }
        // mirostat 1 / 2 ignores top_k .. typical_p, as sample_until_mirostat does
        const SamplingArgs p = sampling_args(g.temp, g.top_k, g.top_p, g.tfs_z, g.typical_p, g.mirostat, g.mirostat_tau, g.mirostat_eta);
        u[(size_t)i] = UntilArgs{p, g.max_steps, g.stop ? g.stop : "###",
                                 PenaltyParams{g.repeat_last_n, g.repeat_penalty, g.alpha_presence, g.alpha_frequency, g.penalize_nl}, g.last_ids, g.n_last};
    }
    const LogprobRequest rec{top_n, logprob_out, rank_out, top_ids_out, top_logprob_out};
    return Engine::sample_until(reinterpret_cast<Engine *const *>(ctxs), n, u.data(), ids_out, n_out, stopped, ms_out, logprob_out ? &rec : nullptr,
                                "generate_batch");
}
int minigpt4_b200_end_chat_penalized(struct MiniGPT4Context *ctx, const char **token, float temp, int32_t top_k, float top_p, float tfs_z,
                                     float typical_p, int32_t repeat_last_n, float repeat_penalty, float alpha_presence, float alpha_frequency,
                                     int penalize_nl, int mirostat, float mirostat_tau, float mirostat_eta, const int32_t *last_ids, int n_last,
                                     int32_t *id_out) {
    if (!ctx) return ErrFailedToAddString;
    const SamplingArgs sp{temp, top_k, top_p, tfs_z, typical_p, mirostat, mirostat_tau, mirostat_eta};
    return E(ctx)->end_chat_penalized(sp, PenaltyParams{repeat_last_n, repeat_penalty, alpha_presence, alpha_frequency, penalize_nl}, last_ids, n_last,
                                      token, id_out);
}
int minigpt4_b200_op_penalize(const float *logits, int rows, int n_vocab, const int32_t *last_ids, const int32_t *n_last, int32_t repeat_last_n,
                              float repeat_penalty, float alpha_presence, float alpha_frequency, int penalize_nl, int on_device, float *out,
                              float *kernel_ms) {
    const PenaltyParams q{repeat_last_n, repeat_penalty, alpha_presence, alpha_frequency, penalize_nl};
    if (!logits || !out || rows < 1 || rows > LlamaDevice::kMaxBatch || n_vocab < 1 || (on_device != 0 && on_device != 1) ||
        !Engine::penalty_valid(q, 0, "op_penalize"))
        return ErrFailedToAddString;
    std::vector<int32_t> none((size_t)rows, 0);
    if (!n_last) n_last = none.data();
    size_t at = 0;
    for (int r = 0; r < rows; ++r) {
        if (n_last[r] < 0 || (n_last[r] > 0 && !last_ids)) return ErrFailedToAddString;
        for (int j = 0; j < n_last[r]; ++j) if (last_ids[at + j] < 0 || last_ids[at + j] >= n_vocab) return ErrFailedToAddString;
        at += (size_t)n_last[r];
    }
    if (on_device) {
        LlamaDevice::test_penalize(logits, rows, n_vocab, last_ids, n_last, q, out, kernel_ms);
        return 0;
    }
    memcpy(out, logits, (size_t)rows * n_vocab * 4);
    at = 0;
    for (int r = 0; r < rows; ++r) {
        const int w = std::min(repeat_last_n, n_last[r]);
        Sampler::penalize(out + (size_t)r * n_vocab, n_vocab, last_ids + at + (n_last[r] - w), w, repeat_penalty, alpha_presence, alpha_frequency,
                          penalize_nl);
        at += (size_t)n_last[r];
    }
    if (kernel_ms) *kernel_ms = 0.f;
    return 0;
}
struct MiniGPT4B200Constraint *minigpt4_b200_constraint_create(struct MiniGPT4Context *ctx, int n_states, const int32_t *next, const uint8_t *accept) {
    if (!ctx) return nullptr;
    std::shared_ptr<Constraint> c = E(ctx)->make_constraint(n_states, next, accept);
    return c ? new MiniGPT4B200Constraint{c} : nullptr;
}
void minigpt4_b200_constraint_free(struct MiniGPT4B200Constraint *c) { delete c; }
int minigpt4_b200_constraint_attach(struct MiniGPT4Context *ctx, struct MiniGPT4B200Constraint *c) {
    if (!ctx) return ErrFailedToAddString;
    return E(ctx)->constraint_attach(c ? c->c : nullptr) ? 0 : ErrFailedToAddString;
}
int minigpt4_b200_constraint_state(struct MiniGPT4Context *ctx, int *state, int *finished) {
    if (!ctx || !E(ctx)->constraint()) return ErrFailedToAddString;
    const Engine &e = *E(ctx);
    const bool fin = e.constraint_state() == e.constraint()->finished();
    if (state) *state = fin ? -1 : e.constraint_state();
    if (finished) *finished = fin ? 1 : 0;
    return 0;
}
int minigpt4_b200_constraint_allowed(struct MiniGPT4B200Constraint *c, int state, int32_t *ids, int32_t *next_states, int cap) {
    return c ? allowed_of(*c->c, state, ids, next_states, cap) : -1;
}
int minigpt4_b200_host_constraint_allowed(const char *llm_model, int n_states, const int32_t *next, const uint8_t *accept, int state, int32_t *ids,
                                          int32_t *next_states, int cap) {
    LlamaFile f;
    if (!f.load(llm_model)) return -1000000;
    std::vector<std::string> texts(f.vocab.size());
    for (size_t id = 0; id < texts.size(); ++id) texts[id] = id == 2 ? "</s>" : f.vocab[id].text.c_str();   // (Engine::id_to_token)
    Constraint c;
    std::string why;
    if (!compile_constraint(texts, n_states, next, accept, c, &why)) return -1000000;
    return allowed_of(c, state, ids, next_states, cap);
}
int minigpt4_b200_encode_images(struct MiniGPT4Context *ctx, struct MiniGPT4Images *images, struct MiniGPT4Embeddings *embeddings) {
    if (embeddings->n_embeddings < images->n_images) return ErrImageSize;
    return E(ctx)->encode_images(images->images, images->n_images, embeddings->embeddings, nullptr);
}
int minigpt4_b200_stats(struct MiniGPT4Context *ctx, struct MiniGPT4B200Stats *out) {
    Engine *e = E(ctx);
    memset(out, 0, sizeof(*out));
    const LlamaDims &d = e->llm().dims();
    out->llm_weight_bytes_per_token = (double)e->llm().weight_bytes_per_token();
    out->kernel_launches = e->llm().kernel_launches();
    if (e->has_vision()) {
        out->vision_flops_per_image = e->vision()->flops_per_image();
        out->vision_weight_bytes = (double)e->vision()->weight_bytes();
        out->kernel_launches += e->vision()->kernel_launches();
    }
    out->last_encode_ms = e->last_encode_ms;
    out->n_layer = d.n_layer; out->n_embd = d.n_embd; out->n_ff = d.n_ff; out->n_vocab = d.n_vocab; out->n_ctx = d.n_ctx;
    out->tp_rank = e->tp.rank; out->tp_world = e->tp.world; out->sm_count = e->llm().sm_count();
    out->decode_megakernel = e->llm().mega_generation();
    out->prefill_gemm = e->llm().uses_prefill_gemm() ? 1 : 0;
    return 0;
}
int minigpt4_b200_time_matvec(struct MiniGPT4Context *ctx, int kind, int reps, float *avg_ms, double *bytes_per_launch) {
    *avg_ms = E(ctx)->llm().time_matvec(kind, reps, bytes_per_launch); return 0;
}
int minigpt4_b200_tp_time_allreduce(struct MiniGPT4Context *ctx, int reps, float *us_out, int *peer_path) {
    E(ctx)->flush();
    *us_out = E(ctx)->llm().time_allreduce(reps);
    if (peer_path) *peer_path = E(ctx)->llm().tp_peer_path() ? 1 : 0;
    return 0;
}
int minigpt4_b200_mega_trace(struct MiniGPT4Context *ctx, long long *out, int max_values) { E(ctx)->flush(); return E(ctx)->llm().mega_trace(out, max_values); }
int minigpt4_b200_op_matvec(int ggml_type, int rows, int cols, const void *w_blocks, const float *x, int n, float *y) {
    LlamaDevice::test_matvec(ggml_type, rows, cols, w_blocks, x, n, y); return 0;
}
int minigpt4_b200_op_gemm_f16(int M, int T, int K, const void *w_f16, const void *x_f16, const float *bias, int epi, const float *aux, float qscale,
                              int qscale_rows, int ksplit, int tsplit, int in_place, void *out, int32_t *plan_out) {
    return VisionDevice::test_gemm(M, T, K, w_f16, x_f16, bias, epi, aux, qscale, qscale_rows, ksplit, tsplit, in_place, out, plan_out);
}
int minigpt4_b200_op_layernorm(const float *x, int rows, int n, const float *w, const float *b, float *out32, void *out16) {
    return VisionDevice::test_layernorm(x, rows, n, w, b, out32, out16);
}
int minigpt4_b200_op_layernorm_fold(float *x, int rows, int n, const float *w, const float *b, const float *parts, int n_parts, long long part_stride,
                                    void *out16) {
    return VisionDevice::test_layernorm_fold(x, rows, n, w, b, parts, n_parts, part_stride, out16);
}
int minigpt4_b200_op_attention(const float *buf, long long n_buf, long long q_off, int ldq, long long k_off, long long v_off, int ldkv, int nq, int nk,
                               int heads, int dh, float score_div, int q_per_cta, int ld_out, float *out) {
    return VisionDevice::test_attention(buf, n_buf, q_off, ldq, k_off, v_off, ldkv, nq, nk, heads, dh, score_div, q_per_cta, ld_out, out);
}
int minigpt4_b200_encode_taps(struct MiniGPT4Context *ctx, const float *image, float *embed, float *vit_blocks, float *ln_vision, float *qformer, float *out) {
    if (!ctx || !image || !E(ctx)->has_vision()) return ErrFailedToAddString;
    E(ctx)->vision()->encode_taps(image, embed, vit_blocks, ln_vision, qformer, out);
    return 0;
}

int minigpt4_b200_op_llama_attention(const float *q, const void *k_f16, const void *v_f16, int n_head, int n_ctx, int rows, const int32_t *pos, int path,
                                     float *out) {
    if (!q || !k_f16 || !v_f16 || !pos || !out) return ErrFailedToAddString;
    return LlamaDevice::test_attention(q, (const uint16_t *)k_f16, (const uint16_t *)v_f16, n_head, n_ctx, rows, pos, path, out) ? 0 : ErrFailedToAddString;
}

int minigpt4_b200_op_dequant_f16(int ggml_type, const void *raw, long n, void *out_f16) { return VisionDevice::test_dequant(ggml_type, raw, n, out_f16); }
extern "C" long mg4_quantize_row(int gg_type, const float *x, long n, unsigned char *out);
long minigpt4_b200_host_quantize_row(int ggml_type, const float *x, long n, void *out_blocks) { return mg4_quantize_row(ggml_type, x, n, (unsigned char *)out_blocks); }

int minigpt4_b200_host_tokenize(const char *llm_model, const char *text, int add_bos, int32_t *out, int max_tokens) {
    LlamaFile f;
    if (!f.load(llm_model)) return -1000000;
    Tokenizer t; t.init(f.vocab);
    std::vector<int32_t> ids = t.encode(text ? text : "", add_bos != 0);
    if ((int)ids.size() > max_tokens) return -(int)ids.size();
    memcpy(out, ids.data(), ids.size() * sizeof(int32_t));
    return (int)ids.size();
}
int minigpt4_b200_host_sample(const float *logits, int n_vocab, int seed, float temp, int32_t top_k, float top_p, float tfs_z, float typical_p,
                              int mirostat, float mirostat_tau, float mirostat_eta, int n_draws, int32_t *out_ids) {
    Sampler s(seed);
    SamplingArgs sp{temp, top_k, top_p, tfs_z, typical_p, mirostat, mirostat_tau, mirostat_eta};
    for (int i = 0; i < n_draws; ++i) out_ids[i] = s.sample(logits, n_vocab, sp);
    return 0;
}
int minigpt4_b200_op_sample(const float *logits, int n_vocab, int seed, float temp, int32_t top_k, float top_p, float tfs_z, float typical_p,
                            int n_draws, int32_t *out_ids) {
    return minigpt4_b200_op_sample_timed(logits, n_vocab, seed, temp, top_k, top_p, tfs_z, typical_p, n_draws, out_ids, nullptr);
}
int minigpt4_b200_op_sample_timed(const float *logits, int n_vocab, int seed, float temp, int32_t top_k, float top_p, float tfs_z, float typical_p,
                                  int n_draws, int32_t *out_ids, float *kernel_ms) {
    if (!logits || !out_ids || n_vocab < 1 || n_draws < 1 || !(temp > 0.f)) return ErrFailedToAddString;
    uint32_t rng[625];
    Sampler(seed).get_rng(rng);
    LlamaDevice::test_sample(logits, n_vocab, SamplingArgs{temp, top_k, top_p, tfs_z, typical_p}, rng, n_draws, out_ids, kernel_ms);
    return 0;
}
int minigpt4_b200_op_sample_mirostat(const float *logits, int n_vocab, int seed, float temp, int mirostat, float mirostat_tau, float mirostat_eta,
                                     int n_draws, int on_device, int32_t *ids_out, float *mu_out, float *kernel_ms) {
    if (!logits || !ids_out || !mu_out || n_vocab < 1 || n_draws < 1 || (mirostat != 1 && mirostat != 2) || (on_device != 0 && on_device != 1))
        return ErrFailedToAddString;
    if (!on_device) {
        Sampler s(seed);
        const SamplingArgs sp = sampling_args(temp, 0, 1.f, 1.f, 1.f, mirostat, mirostat_tau, mirostat_eta);
        for (int d = 0; d < n_draws; ++d) {
            ids_out[d] = s.sample(logits, n_vocab, sp);
            float mu[2]; bool init[2];
            s.get_mu(mu, init);
            mu_out[d] = mu[mirostat - 1];
        }
        if (kernel_ms) *kernel_ms = 0.f;
        return 0;
    }
    if (!(temp > 0.f)) return ErrFailedToAddString;   // greedy: not the sampler
    uint32_t rng[625];
    Sampler(seed).get_rng(rng);
    LlamaDevice::test_sample(logits, n_vocab, sampling_args(temp, 0, 1.f, 1.f, 1.f, mirostat, mirostat_tau, mirostat_eta), rng, n_draws, ids_out, kernel_ms,
                             mu_out);
    return 0;
}
int minigpt4_b200_op_reply_stop(struct MiniGPT4Context *ctx, const int32_t *ids, int n, const char *stop, const char *tail, int32_t *stop_at) {
    if (!ctx) return ErrFailedToAddString;
    return E(ctx)->reply_stop(ids, n, stop, tail, stop_at);
}
// the device libm twin fn (LlamaDevice::test_libm) against the host's libm over the float bit patterns lo_bits .. hi_bits, bit for bit
static int check_libm(int fn, float x, uint32_t lo_bits, uint32_t hi_bits, long long *mismatches) {
    if (hi_bits < lo_bits || !mismatches) return ErrFailedToAddString;
    const uint64_t total = (uint64_t)hi_bits - lo_bits + 1, chunk = (uint64_t)1 << 26;
    std::vector<float> dev((size_t)std::min(total, chunk));
    const unsigned nt = std::max(1u, std::min(64u, std::thread::hardware_concurrency()));
    long long bad = 0;
    for (uint64_t base = 0; base < total; base += chunk) {
        const uint32_t lo = (uint32_t)(lo_bits + base), c = (uint32_t)std::min(chunk, total - base);
        LlamaDevice::test_libm(fn, lo, c, dev.data(), x);
        std::vector<long long> part(nt, 0);
        std::vector<std::thread> th;
        for (unsigned t = 0; t < nt; ++t) th.emplace_back([&, t] {
            long long m = 0;
            for (uint32_t i = (uint32_t)((uint64_t)c * t / nt); i < (uint32_t)((uint64_t)c * (t + 1) / nt); ++i) {
                float v; const uint32_t u = lo + i; memcpy(&v, &u, 4);
                const float h = fn == 0 ? expf(v) : fn == 1 ? logf(v) : fn == 2 ? log2f(v) : powf(x, v);
                if (memcmp(&h, &dev[i], 4) != 0) ++m;
            }
            part[t] = m;
        });
        for (auto &x : th) x.join();
        for (long long m : part) bad += m;
    }
    *mismatches = bad;
    return 0;
}
int minigpt4_b200_op_check_libm(int fn, uint32_t lo_bits, uint32_t hi_bits, long long *mismatches) {
    if (fn != 0 && fn != 1) return ErrFailedToAddString;
    return check_libm(fn, 0.f, lo_bits, hi_bits, mismatches);
}
int minigpt4_b200_op_check_log2f(uint32_t lo_bits, uint32_t hi_bits, long long *mismatches) { return check_libm(2, 0.f, lo_bits, hi_bits, mismatches); }
int minigpt4_b200_op_check_powf(float x, uint32_t lo_bits, uint32_t hi_bits, long long *mismatches) { return check_libm(3, x, lo_bits, hi_bits, mismatches); }
int minigpt4_b200_host_inspect_container(const char *path, int *n_models, int *n_tensors, int *n_embd_llm) {
    VisionFile f;
    if (Error e = f.load(path)) return e;
    int nt = 0; for (auto &m : f.models) nt += (int)m.second.size();
    if (n_models) *n_models = (int)f.models.size();
    if (n_tensors) *n_tensors = nt;
    if (n_embd_llm) { const HostTensor *t = f.find("llama_proj", "weight"); *n_embd_llm = t ? (int)t->ne[1] : 0; }
    return 0;
}
int minigpt4_b200_host_inspect_ggjt(const char *path, int *n_vocab, int *n_embd, int *n_layer, int *n_tensors) {
    LlamaFile f;
    if (!f.load(path)) return ErrLoadLanguageModel;
    if (n_vocab) *n_vocab = (int)f.n_vocab;
    if (n_embd) *n_embd = (int)f.n_embd;
    if (n_layer) *n_layer = (int)f.n_layer;
    if (n_tensors) *n_tensors = (int)f.tensors.size();
    return 0;
}

}  // extern "C"

// llama.h — device-resident LLaMA/Vicuna step (the path behind llama_eval / llama_eval_embd,
// called by the reference at minigpt4.cpp:2373 and :2412).
//
// Data layout in HBM (owned by this engine; algorithmic bytes == file bytes):
//   * every quantised matrix is repacked at load into SoA planes so that each warp-level access is a
//     128-bit aligned vector (Q4_1/Q4_0: row-packed [nb x 16 B nibbles][nb x half2{d,m} | half d] so a run of rows is ONE contiguous range for cp.async.bulk;
//     Q5_K: row-packed [nsb x 128 B qs][nsb x 32 B qh][nsb x 16 B {scales[12],d,dmin}]; Q6_K: ql 128 B + qh 64 B + scales 16 B + half d)
//   * wq|wk|wv are concatenated row-wise (one launch), w1/w3 are row-interleaved (gate r, up r adjacent)
//   * KV cache: F16 [layer][n_ctx][n_embd_local] for K and V (token-major; values as in ggml's cache)
//   * activations between kernels are F32 vectors; each consumer re-quantises them to the weight type's
//     vec_dot type (Q8_0/Q8_1/Q8_K/F16) in its prologue — the integer-dot formulation ggml uses (SURVEY §A.3)
#pragma once
#include "formats.h"
#include <memory>

namespace mg4 {

struct TPLink;  // tensor-parallel communicator (tp.h)
namespace pf { struct PrefillArgs; }   // llama_prefill.cuh
namespace k { struct MatvecArgs; }    // llama_kernels.cuh

struct QMat {          // one repacked weight matrix (or a fused group of matrices of one type)
    int type = -1;     // GGType
    int rows = 0, cols = 0;
    void *p0 = nullptr, *p1 = nullptr, *p2 = nullptr, *p3 = nullptr;
    size_t bytes = 0;  // algorithmic bytes (rows * row_bytes)
    int row_bytes = 0; // row-packed layouts (p0 holds rows of row_bytes each): Q4_0 / Q4_1 [nb x 16 B nibbles][nb x scales]; Q5_K [nsb x 128 B qs][nsb x 32 B qh][nsb x 16 B {scales, d, dmin}]
};

struct PQMat {         // prefill operand cache of one Q4_0 / Q4_1 matrix (llama_prefill.cuh): int8, class-major, + {d, m} in the same order
    int rows = 0, rows_pad = 0, cols = 0, nb = 0, S = 0; bool q41 = false;
    signed char *q = nullptr; void *sc = nullptr;
    alignas(64) unsigned char tm[128];  // CUtensorMap over q
};

struct LlamaDims { int n_vocab, n_embd, n_head, n_layer, n_ff, n_ctx, head_dim; };

struct DeviceState {   // lives in device memory; kernels read positions/tokens from here so graphs are position independent
    int n_past;
    int n_tok;
    int tokens[8];
    unsigned long long argmax_key;
    int argmax_id;
    int pad[3];
};

struct SessionSlot {   // one column of a batched decode step (device table of the group, refreshed by one copy per step)
    int n_past;        // the context's position: its token is evaluated there
    int id;            // token to feed; < 0: the context's on-device greedy id (DeviceState::tokens[0])
    __half *kcache, *vcache;   // the context's caches (layer 0)
    float *logits;
    DeviceState *state;
};

// Sampler::sample's arguments: the non-mirostat chain, or mirostat 1 / 2 (which ignores top_k .. typical_p); mirostat 0: the chain
struct SamplingArgs { float temp; int top_k; float top_p, tfs_z, typical_p; int mirostat; float mirostat_tau, mirostat_eta; };
struct MirostatState { float mu[2]; int init[2]; };   // a context's mirostat μ of v1 / v2 and whether each is set (Sampler::get_mu)
struct SamplerScratch; // a context's device sampler: mt19937 state, candidate scratch, the ids of a call (llama.cu, llama_sample.cuh)
struct ReplyScratch;   // a context's stop state in sample_until: reply tail, stop text, done flag, snapshot (llama.cu, llama_sample.cuh)
namespace smp { template <int N> struct SampleArgsN; }

struct LlamaGroup;     // what the contexts of one model share besides the weights: the batch workspace and its graphs (llama.cu)
struct ScoreCall;      // the outputs of a score_rows call, which eval_rows_batch's passes fill (llama.cu)

class LlamaDevice {
public:
    LlamaDevice();
    ~LlamaDevice();
    bool load(const LlamaFile &f, int n_ctx, TPLink *tp);
    // A new context over the weights of `parent` (the repacked matrices, the prefill operand cache, token embeddings, RoPE table,
    // LUTs and the prefill scratch, which is only used synchronously): own KV cache of the parent's n_ctx, activations, state,
    // stream and decode graph / megakernel.  The weights go with the last context of the group.  Single GPU only.
    bool load_session(const LlamaDevice &parent);
    const LlamaGroup *group() const { return group_.get(); }
    int group_size() const { return (int)group_.use_count(); }
    size_t owned_bytes() const { return owned_bytes_; }   // device bytes of this context: KV cache + per-context scratch
    size_t shared_bytes() const;                          // device bytes shared by the group: weights, operand cache, tables, prefill scratch, batch workspace
    // the most contexts one batched call takes: two 32-token tiles of the prefill GEMM (pf::kTok), and about the 7B sessions at n_ctx 2048
    // that fit on an 80 GB card
    static constexpr int kMaxBatch = 64;
    // One decode step of n (2..kMaxBatch) distinct contexts of one group; the weights stream once.  Column i is fed ids[i] (< 0: the context's
    // on-device greedy id) at position n_past[i]; afterwards each context holds what its own decode_step would have left (logits,
    // arg-max, DeviceState) and ids_out[i] = its new arg-max.  Synchronous.  The caller validates (distinct, one group, ranges).
    // n <= 8: per-op matvecs at NT = n; more: the layers in 8-column matvec chunks, or from kWideGemmMin (llama.cu) columns on a
    // pf_ready_ model the tensor-core pass of eval_rows_batch with one row per column.
    static void decode_batch(LlamaDevice *const *ctx, int n, const int32_t *ids, const int *n_past, int32_t *ids_out);
    // The queued prompt rows of n (1..kMaxBatch) distinct contexts of one group in shared passes over the weights, kPrefillMax rows per pass:
    // context i has n_rows[i] (1..kPrefillMax) rows starting at position n_past[i], ids[i][j] >= 0 a token, < 0 row -1 - ids[i][j] of
    // emb[i] (n_embd floats per row, in order of first use).  Afterwards each context holds what its own eval_rows would have left
    // (KV cache, logits, arg-max, DeviceState) and the first rows of its hidden state are its rows of the pass that evaluated its
    // last row.  Synchronous.  The caller validates (distinct, one group, rows checked when they were queued).
    // score (score_rows): every row's logits go to the group's scoring scratch and its entries are scored; without score->keep the
    // contexts' logits, DeviceState, arg-max and hidden rows are left as they were.
    static void eval_rows_batch(LlamaDevice *const *ctx, int n, const int32_t *const *ids, const int *n_rows, const float *const *emb, const int *n_past,
                                const ScoreCall *score = nullptr);
    // Score known ids against n (1..kMaxBatch) distinct contexts of one group: context i's n_ids[i] (>= 1) token ids are evaluated at
    // positions n_past[i] .. in the shared passes of eval_rows_batch, and every row's logits are computed (llama_score.cuh).  Entry j of
    // context i: logprob[i][j] = log p(ids[i][j]) under the logits before row j (j = 0: the context's current logits; NaN and rank -1 when
    // n_past[i] = 0), rank[i][j] (rank may be null) = the ids ranked above it (larger logit, or equal logit and lower id), logits[i]
    // (logits may be null) = n_ids[i] rows of n_vocab floats, row j the logits of row j.  keep: afterwards each context holds what
    // eval_rows_batch of these rows leaves; otherwise the call changes nothing of a context but its K / V rows at positions >= n_past[i].
    // The group's first call allocates the scoring scratch (kPrefillMax rows of logits, counted in shared_bytes).  Synchronous.  The
    // caller validates (distinct, one group, ids in range, room in each context).
    static void score_rows(LlamaDevice *const *ctx, int n, const int32_t *const *ids, const int *n_ids, const int *n_past, bool keep,
                           float *const *logprob, int32_t *const *rank, float *const *logits);
    // `steps` sampled decode steps of n (1..kMaxBatch) distinct contexts of one group with no host round trip: each step samples every context's
    // current logits on the device (llama_sample.cuh; p.temp <= 0: the greedy id) into its DeviceState, then runs the decode step (n = 1:
    // the context's own graph or megakernel; n >= 2: the batch graph, every column fed its DeviceState::tokens[0]).  rng[i] holds context
    // i's mt19937 state (624 words and the position) on entry and on return, and with p.mirostat 1 / 2 mu[i] its mirostat μ (mu may be
    // null without mirostat); ids_out[s * n + i] is the id context i was fed at step s.
    // One synchronisation at the end; returns the device ms of the steps.  The caller validates (distinct, one group, room for steps).
    static float sample_steps(LlamaDevice *const *ctx, int n, int steps, const int *n_past, const SamplingArgs &p, uint32_t (*rng)[625],
                              MirostatState *mu, int32_t *ids_out);
    // sample_steps that stops each context after the step whose id's text (not exactly "##") makes its reply end with `stop` (0..32
    // bytes, "" no text stop), or after max_steps.  tail[i]: context i's reply so far (its last 32 bytes decide).  The steps are issued
    // kReplyChunk at a time; the host waits for chunk j - 1's done flags before it issues chunk j + 1 and stops issuing once every
    // context is done, so at most 2 kReplyChunk - 1 steps run past the last stop.  Afterwards context i holds what n_out[i] steps left
    // (logits, DeviceState, arg-max; rng[i], mu[i]), and ids_out[s * n + i] = -1 for s >= n_out[i]; stopped[i] = the text ended it.  Needs
    // the group's token table (set_token_table).  One wait per chunk, none of them stalling the device; returns the device ms.
    static constexpr int kReplyChunk = 4;
    static constexpr int kStopMax = 32;   // longest stop text
    static float sample_until(LlamaDevice *const *ctx, int n, int max_steps, const int *n_past, const SamplingArgs &p, uint32_t (*rng)[625],
                              MirostatState *mu, const std::string &stop, const std::string *tail, int32_t *ids_out, int32_t *n_out, int32_t *stopped);
    // the group's device table of every id's text (off: n_vocab + 1 offsets into bytes), counted in shared_bytes
    bool has_token_table() const;
    void set_token_table(const std::vector<int> &off, const std::string &bytes);
    // sample_until's text check over ids[0, n) from the reply `tail`; returns the index of the id that ends the reply, -1 if none
    int test_reply_stop(const int32_t *ids, int n, const std::string &stop, const std::string &tail);
    const LlamaDims &dims() const { return d_; }
    // Evaluate `n` mixed token / embedding rows (ids < 0: row -1 - id of emb_host) starting at position n_past.  Afterwards logits of the
    // last row are on device and the arg-max id is known.  Returns false if the context would overflow.
    bool eval_rows(const int32_t *ids, int n, const float *emb_host, int n_emb, int n_past);
    void logits_to_host(float *dst);   // n_vocab floats, synchronous
    int32_t argmax();                  // greedy id of the current logits (already in pinned host memory after a sync)
    void sync();
    void sync_decode();              // stream sync that reports the megakernel's spin-guard reason code if the launch failed
    int sm_count() const { return sm_count_; }
    bool uses_megakernel() const { return mega_; }
    bool uses_prefill_gemm() const { return pf_ready_; }
    static constexpr int kPrefillMax = 512;   // rows per prefill pass (the reference's default n_batch)
    int mega_generation() const { return mega_ ? 6 : 0; }
    int mega_trace(long long *out, int max_values);  // debug: per-op clock64 stamps of the last megakernel launch (env MINIGPT4_B200_MEGA_TRACE)
    // one decode step through the captured CUDA graph: feeds `id` (or, if id < 0, the on-device arg-max of the
    // previous step), leaves new logits/arg-max on device.
    bool decode_step(int32_t id, int n_past);
    // bench leg: `steps` chained greedy steps with no host round trip; returns device ms for the loop.
    float decode_chain(int steps, int n_past, int32_t *ids_out);
    // measurement seam: average CUDA-event duration (ms) of one launch of the decode matvec of `kind`
    // (0 qkv, 1 wo, 2 gate/up, 3 down, 4 output) cycling through all layers so every launch streams cold weights.
    float time_matvec(int kind, int reps, double *bytes_per_launch);
    float time_allreduce(int reps);   // us per [1, n_embd] all-reduce on the tensor-parallel path in use (0 without tensor parallelism)
    bool tp_peer_path() const;
    // test taps
    void hidden_to_host(float *dst, int n);  // residual stream after the last evaluated chunk (n rows)
    size_t weight_bytes_per_token() const { return bytes_per_token_; }
    unsigned long long kernel_launches() const { return launches_; }
    cudaStream_t stream() const { return stream_; }

    // kernel-level test hook: y[n][rows] = W x (W given as raw ggml blocks on host), through the same
    // repack + matvec kernels the engine uses.
    static void test_matvec(int gg, int rows, int cols, const void *w_host, const float *x_host, int n, float *y_host);
    // kernel-level test hook: the LLaMA attention of `rows` rows (q F32 [rows][n_head * 128]) over F16 K / V caches [n_ctx][n_head * 128]
    // uploaded from the host, with the exp table load() builds; path 0: attn_kernel, row t at position pos[0] + t; path 1:
    // attn_sessions_kernel through a slot table, row t at pos[t].  false (nothing launched) on arguments outside those ranges.
    static bool test_attention(const float *q_host, const uint16_t *k_host, const uint16_t *v_host, int n_head, int n_ctx, int rows, const int *pos,
                               int path, float *out_host);
    // sampler test hook: n_draws draws from one generator (rng: 624 words and the position) over the same n_vocab logits, as n_draws calls
    // of Sampler::sample make (p.temp > 0); kernel_ms (optional): the average CUDA-event time of one sampling launch.  With p.mirostat
    // 1 / 2, μ starts unset and mu_out (optional) takes μ after each draw (a 4-byte device copy after each launch, inside the timing).
    static void test_sample(const float *logits, int n_vocab, const SamplingArgs &p, const uint32_t *rng, int n_draws, int32_t *out, float *kernel_ms,
                            float *mu_out = nullptr);
    // the device expf (fn 0) / logf (fn 1) / log2f (fn 2) of the float bit patterns lo .. lo + n - 1, or powf(x, y) (fn 3) for the y of them
    static void test_libm(int fn, uint32_t lo, uint32_t n, float *out_host, float x = 0.f);

private:
    struct Layer { QMat qkv, wq, wk, wv, wo, w13, w2; bool fused_qkv; float *attn_norm, *ffn_norm; PQMat pqkv, pwo, pw13, pw2; };
    struct Pass {                    // one pass of all layers over `rows` rows that sit in x (record_layers)
        int rows;
        float *x, *q, *att, *act;    // [rows] activations (act also takes the qkv GEMM's [rows][3 n_embd] output when slots is set)
        unsigned char *qact;         // staged matvec inputs of <= 8 rows
        DeviceState *state;          // what MatvecArgs / PrefillArgs read
        const SessionSlot *slots;    // [rows] each row's position and caches; null: positions state->n_past + t in this context's caches
        bool gemm;                   // tensor-core GEMMs (pf_ready_, rows >= 2); otherwise matvecs over <= 8-row chunks
        cudaStream_t s;
        unsigned long long *counter; // kernel launches
    };
    void record_layers(const Pass &p);
    void add_matvec(k::MatvecArgs a, float *x, const Pass &p);   // wo / down into the residual rows x (+ the tensor-parallel reduce)
    void record_pass(int n, bool want_logits);   // this context's pass over n rows in x_: layers, logits, finalize
    void launch_embed(int n, const DeviceState *st, float *x, cudaStream_t s, unsigned long long *counter) const;
    bool build_prefill();            // tensor-core prefill (llama_prefill.cuh): homogeneous Q4_0 / Q4_1 layers, single GPU
    // one matrix of a prefill pass: stage the input rows into the shared operand scratch, then the GEMM
    void pf_stage(const QMat &w, const float *x, int x_stride, const float *norm_w, int S, const Pass &ps);
    void pf_gemm(const PQMat &p, bool ff_wide, const pf::PrefillArgs &epi, const Pass &ps);
    bool pf_ready_ = false; int pf_S_e_ = 0, pf_S_ff_ = 0;
    signed char *pf_q8_ = nullptr; void *pf_sc_ = nullptr; int32_t *tok_ids_ = nullptr; void *pf_part_ = nullptr; size_t pf_part_bytes_ = 0;
    alignas(64) unsigned char pf_tmB_e_[128], pf_tmS_e_[128], pf_tmB_ff_[128], pf_tmS_ff_[128];
    void build_graph();
    bool build_mega();               // persistent one-launch-per-token decode, generation 6 (llama_mega6.cuh): homogeneous Q4_0 / Q4_1 / Q5_K
    void launch_mega();
    const void *mega_fn() const;
    LlamaDims d_{};
    int n_head_local_ = 0, n_embd_local_ = 0, n_ff_local_ = 0;
    TPLink *tp_ = nullptr;
    std::vector<Layer> layers_;
    QMat output_;
    float *final_norm_ = nullptr;
    void *tok_raw_ = nullptr; int tok_type_ = -1;  // tok_embeddings kept as raw ggml blocks (row gather only)
    __half *kcache_ = nullptr, *vcache_ = nullptr;
    float2 *rope_ = nullptr;                        // [n_ctx][head_dim/2] {cos, sin}, host-computed with libm like ggml
    __half *tab_exp_ = nullptr, *tab_silu_ = nullptr;  // ggml's fp16 LUTs
    float *x_ = nullptr, *q_ = nullptr, *att_ = nullptr, *act_ = nullptr, *logits_ = nullptr, *partial_ = nullptr;
    float *embd_in_ = nullptr;
    unsigned char *qact_ = nullptr;                 // per-op staged (quantised) activations for the per-op kernels
    DeviceState *state_ = nullptr;
    DeviceState *h_state_ = nullptr;  // pinned
    int32_t *h_argmax_ = nullptr;     // pinned
    cudaStream_t stream_ = nullptr;
    cudaGraphExec_t graph_ = nullptr;
    cudaEvent_t ev0_ = nullptr, ev1_ = nullptr;
    size_t bytes_per_token_ = 0;
    unsigned long long launches_ = 0;
    int graph_kernels_ = 0;
    long long *mega_trace_ = nullptr; int mega_n_ops_ = 0;
    void *mega6_params_ = nullptr; int mega6_nbl_ = 0;
    bool h_state_busy_ = false;
    bool mega_ = false; unsigned *mega_barrier_ = nullptr; size_t mega_smem_ = 0; int mega_type_ = -1;
    int sm_count_ = 132;
    // sessions: every context of a group holds the same weight pointers above; group_ counts the contexts
    std::shared_ptr<LlamaGroup> group_;
    size_t owned_bytes_ = 0;
    std::unique_ptr<SamplerScratch> smp_;   // allocated by the context's first sample_steps call (counted in owned_bytes_ from then on)
    void ensure_sampler();
    std::unique_ptr<ReplyScratch> reply_;   // sample_until's stop state and snapshot, from the context's first call (owned_bytes_)
    void ensure_reply();
    // the set-up both sampling calls share: the batch graph and slot table (n >= 2), each context's sampler, generator and mirostat μ;
    // returns the stream the steps run on
    static cudaStream_t begin_sampling(LlamaDevice *const *c, int n, const int *n_past, const SamplingArgs &p, uint32_t (*rng)[625], MirostatState *mu,
                                       smp::SampleArgsN<kMaxBatch> &a);
    static void sampled_decode(LlamaDevice *const *c, int n, int n_past, cudaStream_t s);
    static float end_sampling(LlamaDevice *const *c, int n, int steps, const SamplingArgs &p, uint32_t (*rng)[625], MirostatState *mu, int32_t *ids_out,
                              cudaStream_t s);
    void alloc_context();            // the per-context buffers (KV cache, activations, state, stream)
    void free_weights();             // by the last context of the group
    void build_group_workspace();    // the batched passes' rows, slot tables and stream (group-owned, at the first batched call)
    void build_batch_graph(int B);   // decode_batch's graph for B columns, captured on the group stream
    void build_score_scratch();      // score_rows' logits rows, entry tables and results (group-owned, at the first scoring call)
};

}  // namespace mg4

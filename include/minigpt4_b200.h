/*
 * minigpt4_b200.h — EXTRA entry points of the H100-native libminigpt4.so.
 *
 * The 18 symbols of minigpt4.h are untouched.  These additions exist because the reference ABI cannot express
 * (a) a tensor-parallel degree / device choice (SURVEY §8b "Extension needed by configs"),
 * (b) raw llama_eval / llama_eval_embd access (the reference links llama.cpp and calls it directly at
 *     minigpt4.cpp:2373 and :2412; parity tests need the same seam), and
 * (c) kernel-level seams so each CUDA kernel can be checked against the CPU oracle through the C ABI.
 * Plain pointers and sizes only; all buffers are HOST memory unless stated.
 */
#ifndef MINIGPT4_B200_EXT_H
#define MINIGPT4_B200_EXT_H
#include "minigpt4.h"

#ifdef __cplusplus
extern "C" {
#endif

/* process setup ---------------------------------------------------------------------------------------- */
MINIGPT4_API int minigpt4_b200_device_count(void);
MINIGPT4_API int minigpt4_b200_set_device(int device);                    /* before minigpt4_model_load */
MINIGPT4_API int minigpt4_b200_tp_unique_id(void *out128);                /* rank 0: NCCL unique id (128 bytes) */
MINIGPT4_API int minigpt4_b200_tp_configure(int rank, int world, const void *id128); /* applies to later loads */
/* tensor-parallel contexts: average device time (us) of one all-reduce of a [1, n_embd] partial on the path in use; *peer_path = 1 for the one-shot
   peer-memory kernel, 0 for ncclAllReduce + add.  Collective: every rank calls it with the same (even) reps. */
MINIGPT4_API int minigpt4_b200_tp_time_allreduce(struct MiniGPT4Context *ctx, int reps, float *us_out, int *peer_path);

/* language model only (config "decode-only"): path = ggjt v3 file; replaces llama_load_model_from_file +
 * llama_new_context_with_model (reference minigpt4.cpp:1783-1784) */
MINIGPT4_API struct MiniGPT4Context *minigpt4_b200_llm_load(const char *llm_model, int n_ctx, int seed, int verbosity);

/* llama.cpp seams (reference call sites minigpt4.cpp:2373 llama_eval, :2412 llama_eval_embd, :2389 llama_tokenize,
 * :2432 llama_get_logits, :2428 llama_n_vocab, :2401 llama_n_embd).  eval_* advance n_past like add_tokens/add_embedding. */
MINIGPT4_API int minigpt4_b200_n_vocab(struct MiniGPT4Context *ctx);
MINIGPT4_API int minigpt4_b200_n_embd(struct MiniGPT4Context *ctx);
MINIGPT4_API int minigpt4_b200_n_past(struct MiniGPT4Context *ctx);
MINIGPT4_API int minigpt4_b200_tokenize(struct MiniGPT4Context *ctx, const char *text, int add_bos, int32_t *out, int max_tokens);
MINIGPT4_API int minigpt4_b200_eval_tokens(struct MiniGPT4Context *ctx, const int32_t *ids, int n);
MINIGPT4_API int minigpt4_b200_eval_embd(struct MiniGPT4Context *ctx, const float *rows, int n);
/* Prompt pieces (minigpt4_begin_chat_image, minigpt4_system_prompt, the two calls above) are queued and evaluated together when the model
   state is needed (sampling, logits, decode); this evaluates the queue now.  Returns 0 on success. */
MINIGPT4_API int minigpt4_b200_flush(struct MiniGPT4Context *ctx);
MINIGPT4_API int minigpt4_b200_get_logits(struct MiniGPT4Context *ctx, float *out_n_vocab);
MINIGPT4_API int minigpt4_b200_greedy_id(struct MiniGPT4Context *ctx);
MINIGPT4_API int minigpt4_b200_get_hidden(struct MiniGPT4Context *ctx, float *out, int n_rows);
MINIGPT4_API const char *minigpt4_b200_token_text(struct MiniGPT4Context *ctx, int32_t id);

/* `steps` greedy decode steps chained on the device (no host round trip); ids_out[steps] receives the ids that were
 * fed; *ms_out the CUDA-event time of the loop.  The bench's device-resident `value` leg. */
MINIGPT4_API int minigpt4_b200_decode_chain(struct MiniGPT4Context *ctx, int steps, int32_t *ids_out, float *ms_out);

/* batch encode (config 5): n images -> n embeddings, same semantics per image as minigpt4_encode_image */
MINIGPT4_API int minigpt4_b200_encode_images(struct MiniGPT4Context *ctx, IN struct MiniGPT4Images *images, OUT struct MiniGPT4Embeddings *embeddings);

struct MiniGPT4B200Stats {
    double llm_weight_bytes_per_token;  /* algorithmic bytes streamed per decoded token on THIS rank */
    double vision_flops_per_image;
    double vision_weight_bytes;
    double last_encode_ms;              /* CUDA-event time of the last encode graph */
    unsigned long long kernel_launches; /* kernels of this library launched so far (both graphs) */
    int n_layer, n_embd, n_ff, n_vocab, n_ctx, tp_rank, tp_world, sm_count;
    int decode_megakernel;              /* > 0: decode step = one persistent kernel per token (value = kernel generation); 0: one launch per op (graph) */
    int prefill_gemm;                   /* 1: prompt / prefix rows (N >= 2) run through the wgmma s8 prefill GEMM; 0: per-op matvec path */
};
MINIGPT4_API int minigpt4_b200_stats(struct MiniGPT4Context *ctx, struct MiniGPT4B200Stats *out);

/* measurement seam for bench.py's roofline: average CUDA-event duration of one launch of the decode matvec `kind`
 * (0 qkv, 1 wo, 2 gate/up, 3 down, 4 output), cycling through the layers so every launch streams cold weights */
MINIGPT4_API int minigpt4_b200_time_matvec(struct MiniGPT4Context *ctx, int kind, int reps, float *avg_ms, double *bytes_per_launch);

/* debug: per-op clock64 stamps {op start, grid barrier passed, activations staged, op done} of CTA 0 and CTA G-1 in the last
 * decode megakernel launch; only recorded when the context was loaded with MINIGPT4_B200_MEGA_TRACE set. Returns #values. */
MINIGPT4_API int minigpt4_b200_mega_trace(struct MiniGPT4Context *ctx, long long *out, int max_values);

/* kernel-level seams (each runs the production kernel on cuda:current and returns to host) -------------- */
/* y[n][rows] = W . x  with W given as raw ggml blocks of `ggml_type` (2 Q4_0, 3 Q4_1, 13 Q5_K, 14 Q6_K, 1 F16) */
MINIGPT4_API int minigpt4_b200_op_matvec(int ggml_type, int rows, int cols, const void *w_blocks, const float *x, int n, float *y);
/* out[T][M] = epi(bias + X[T][K] . W[M][K]^T), F16 operands; epi 0 = bias, 2 = bias+GELU(fp16 LUT) rounded to F16 */
MINIGPT4_API int minigpt4_b200_op_gemm_f16(int M, int T, int K, const void *w_f16, const void *x_f16, const float *bias, int epi, float *out);
MINIGPT4_API int minigpt4_b200_op_layernorm(const float *x, int rows, int n, const float *w, const float *b, float *out);
/* q,k,v: [n][heads*dh]; out [nq][heads*dh] rounded to F16 precision */
MINIGPT4_API int minigpt4_b200_op_attention(const float *q, const float *k, const float *v, int nq, int nk, int heads, int dh, float score_div, float *out);

/* out_f16[n] = the F16 operand the vision graph builds at load time from a non-F16 matrix: `raw` holds n elements as ggml blocks of
 * `ggml_type` (0 F32, 2 Q4_0, 3 Q4_1, 6 Q5_0, 7 Q5_1, 8 Q8_0); values follow ggml's dequantize_row_* and are rounded to F16 */
MINIGPT4_API int minigpt4_b200_op_dequant_f16(int ggml_type, const void *raw, long n, void *out_f16);

/* host-only seams (no GPU touched): the tokenizer / sampler / file readers are host logic and are unit-tested on CPU */
/* tokenise with the vocabulary stored in a ggjt file; returns count or -needed (llama_tokenize convention), -1000000 on read failure */
MINIGPT4_API int minigpt4_b200_host_tokenize(const char *llm_model, const char *text, int add_bos, int32_t *out, int max_tokens);
/* run the sampler chain of minigpt4_end_chat on caller-provided logits (reference minigpt4.cpp:2425-2483) */
MINIGPT4_API int minigpt4_b200_host_sample(const float *logits, int n_vocab, int seed, float temp, int32_t top_k, float top_p, float tfs_z,
                                           float typical_p, int mirostat, float mirostat_tau, float mirostat_eta, int n_draws, int32_t *out_ids);
/* block quantiser behind minigpt4_quantize_model (ggml quantize_row_*_reference): n floats (n % 32 == 0) -> ggml blocks of
 * `ggml_type` (2 Q4_0, 3 Q4_1, 6 Q5_0, 7 Q5_1, 8 Q8_0); returns the bytes written, -1 for an unsupported type or ragged n */
MINIGPT4_API long minigpt4_b200_host_quantize_row(int ggml_type, const float *x, long n, void *out_blocks);
/* parse a MiniGPT-4 container (returns MiniGPT4Error) / ggjt file (0 ok) and report tensor counts */
MINIGPT4_API int minigpt4_b200_host_inspect_container(const char *path, int *n_models, int *n_tensors, int *n_embd_llm);
MINIGPT4_API int minigpt4_b200_host_inspect_ggjt(const char *path, int *n_vocab, int *n_embd, int *n_layer, int *n_tensors);

#ifdef __cplusplus
}
#endif
#endif

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

/* multi-session serving: several conversations over one loaded model ------------------------------------------------
 * A session is a MiniGPT4Context that shares the model of `ctx` (language and vision weights, the prefill operand cache and
 * scratch, encode lanes, tokenizer) and owns a conversation: its KV cache of ctx's n_ctx positions, n_past, prompt queue,
 * logits, device state, decode graph / megakernel and a sampler seeded with `seed`.  All 18 entry points of minigpt4.h work
 * on it.  ctx and its sessions form a group; they may be freed in any order and the weights go with the last of them.
 * The contexts of one group must not be called from two threads at once (the reference's contract for one context).
 * Returns NULL on failure (device memory exhausted, a tensor-parallel ctx, ctx NULL). */
MINIGPT4_API struct MiniGPT4Context *minigpt4_b200_session_create(struct MiniGPT4Context *ctx, int seed);
/* live contexts of ctx's group; device bytes ctx owns (KV cache 2 * n_layer * n_ctx * n_embd * 2 B plus its activations of
 * 512 prompt rows and a few small buffers); device bytes it shares with its group (weights, operand cache, tables, prefill
 * scratch, the workspace of the batched calls once built).  Any pointer may be NULL. */
MINIGPT4_API int minigpt4_b200_session_info(struct MiniGPT4Context *ctx, int *n_contexts, double *owned_bytes, double *shared_bytes);
/* One decode step of n (1..64) distinct contexts of one group: the weights stream once for all of them.  Context i is fed ids[i]
 * (ids[i] < 0: its current on-device greedy id, as in minigpt4_b200_decode_chain) at its own n_past; queued prompt pieces of
 * each context are evaluated first.  Afterwards each context has new logits, n_past + 1, and ids_out[i] = its new greedy id;
 * its logits are the bits a step on its own gives.  n >= 2 runs one batched step: its layers take the per-op matvecs up to 15
 * contexts, and from 16 contexts on the tensor-core GEMM of the prompt passes on models with homogeneous Q4_0 / Q4_1 layers (the
 * per-op matvecs on every other model); either gives the same bits.  Synchronous.  NULL or duplicate contexts, contexts of different groups,
 * n outside 1..64, a full context or an id >= n_vocab return the FailedToAddString error code (8) and change no context. */
MINIGPT4_API int minigpt4_b200_decode_batch(struct MiniGPT4Context **ctxs, int n, const int32_t *ids, int32_t *ids_out);
/* Evaluate the queued prompt rows (add_tokens / add_embedding pieces not yet evaluated) of n (1..64) distinct contexts of one group
 * in shared passes over the weights, at most 512 rows per pass; a context's rows may be split across two passes.  Afterwards each
 * context is exactly as minigpt4_b200_flush would have left it: n_past, KV cache, logits (bit for bit), greedy id and the device
 * state the next decode step continues from.  Contexts with an empty queue are left untouched; n = 1 is that context's own flush.
 * minigpt4_b200_get_hidden(ctx, out, k), with k the number of its rows in the pass that evaluated its last row, returns the residual
 * stream of those rows, i.e. of its last k rows (an own flush leaves the rows of its own last pass the same way).
 * minigpt4_b200_decode_batch and end_chat_batch flush their contexts this way.
 * Synchronous.  NULL or duplicate contexts, contexts of different groups or n outside 1..64 return the FailedToAddString error
 * code (8) and change no context. */
MINIGPT4_API int minigpt4_b200_flush_batch(struct MiniGPT4Context **ctxs, int n);
/* How likely is a known continuation: the log-probability of every id of it, for n (1..64) distinct contexts of one group in shared
 * passes over the weights.  ids holds the contexts' token ids back to back, n_ids[i] >= 1 of them for context i; logprob_out and
 * rank_out have the layout of ids, logits_out (may be NULL) one n_vocab row per id in the same order.  Queued prompt pieces are
 * evaluated first, as in minigpt4_b200_decode_batch; then context i's ids are evaluated at positions n_past .. n_past + n_ids[i] - 1
 * in passes of at most 512 rows (a context's rows may be split across two passes).  For entry j of context i:
 *   logprob_out[j] = log p(ids[j] | the conversation so far and ids[0 .. j-1]): for j = 0 from the context's logits before the call,
 *     for j >= 1 from the logits of row j - 1 of this call.  With n_past = 0 there are no logits before the call: entry 0 is NaN, its
 *     rank -1.  With m the row's largest logit, lp = (float)((z_t - m) - log sum exp((double)z - m)), the sum in double.
 *   rank_out[j] (may be NULL) = the ids with a larger logit plus those with an equal logit and a lower id (the device sampler's tie
 *     rule); rank 0: the greedy step would have picked ids[j].
 *   logits_out row j = the logits of the row of ids[j] (those that predict ids[j + 1]), bit for bit the logits the context would
 *     hold after evaluating its ids up to j.
 * keep = 1: afterwards each context is where minigpt4_b200_eval_tokens(ids) + flush leaves it (n_past, logits, greedy id, device
 * state, minigpt4_b200_get_hidden as for flush_batch; the reply tail is cleared).  keep = 0: afterwards each context is exactly as it
 * was (n_past, logits, greedy id, device state, hidden rows, reply tail, generator and mirostat μ); the call only writes K / V rows at
 * positions >= n_past, which the next evaluated token overwrites before anything reads them, so the K continuations of one prompt are
 * K calls on one context with nothing to undo.  The group's first call allocates 512 rows of logits (counted in
 * minigpt4_b200_session_info's shared bytes: 65.5 MB at n_vocab 32000).  Synchronous.
 * NULL ctxs / ids / n_ids / logprob_out, NULL or duplicate contexts, contexts of different groups, n outside 1..64, n_ids[i] < 1, an
 * id outside the vocabulary, n_past + n_ids[i] > n_ctx, keep outside 0..1 or a tensor-parallel context return the FailedToAddString
 * error code (8) and change no context, before any device work. */
MINIGPT4_API int minigpt4_b200_score_tokens(struct MiniGPT4Context **ctxs, int n, const int32_t *ids, const int32_t *n_ids, int keep,
                                            float *logprob_out, int32_t *rank_out, float *logits_out);
/* Copy the conversation of src into n (1..64) distinct other contexts of its group, so that several sessions continue one shared prefix
 * (a system prompt, an image turn, best-of-N replies) without evaluating it again.  src's queued prompt pieces are evaluated first, by
 * its own flush.  Afterwards every destination has src's conversation: n_past, K / V rows 0 .. n_past - 1 bit for bit, logits, greedy
 * id, device state and the reply tail that minigpt4_b200_sample_until's stop rule reads; its queued pieces are discarded.  Its rows at
 * positions >= n_past are left as they were: no kernel reads a key above a row's position, and the next evaluated row overwrites them.
 * Each destination keeps its own sampler (generator and mirostat μ), so copies into sessions of different seeds draw different replies.
 * The rows of minigpt4_b200_get_hidden are not carried.  src is left exactly as its flush left it.  The call first waits for the steps
 * still running on every context involved (minigpt4_end_chat returns with its step running); it is synchronous and allocates nothing,
 * so minigpt4_b200_session_info's bytes do not change.  One kernel launch reads each source row once and writes it to every destination.
 * NULL src / dsts, n outside 1..64, NULL or duplicate destinations, src among them, a destination of another group or a tensor-parallel
 * context return the FailedToAddString error code (8) before any device work, with no context changed (src's queue not evaluated).
 * The _timed form also returns the CUDA-event time of the copy kernel (kernel_ms may be NULL). */
MINIGPT4_API int minigpt4_b200_session_copy(struct MiniGPT4Context *src, struct MiniGPT4Context **dsts, int n);
MINIGPT4_API int minigpt4_b200_session_copy_timed(struct MiniGPT4Context *src, struct MiniGPT4Context **dsts, int n, float *kernel_ms);
/* Save a conversation to host memory and restore it, in this process or another, into any context whose model has the same fingerprint.
 * state_size: the bytes state_save writes now (n_past counts the queued prompt rows; nothing is evaluated); -1 for NULL or a
 * tensor-parallel ctx.  state_save: evaluates ctx's queue, then writes the state to buf and *written (may be NULL) = its size; cap below
 * the size returns 8 and writes nothing (and evaluates nothing).  state_load: replaces ctx's conversation as minigpt4_b200_session_copy
 * does (its sampler is kept, its queue discarded, its rows above n_past untouched); the state may come from any group, provided
 * n_past <= ctx's n_ctx.  The K / V rows move with one copy per layer plane between buf and the cache, bound by the host link.
 * The state is little-endian, 144 header bytes:
 *   0 "MG4STATE"; 8 uint32 version 1; 12 int32 n_vocab, n_embd, n_head, n_layer, n_ff; 32 uint64 fingerprint of the model (FNV-1a 64
 *   over the LLaMA tensor table, name, type and shape in name order, and the first 4096 bytes of each tensor's data); 40 int32 n_past;
 *   44 int32 reply tail length (0..32); 48 the reply tail, 32 bytes; 80 the 64-byte device state (its n_past is the header's);
 *   then 144: n_vocab float32 logits; then K[n_layer][n_past][n_embd] and V[n_layer][n_past][n_embd] as float16.
 * state_load returns 8 and changes nothing, before any device work, for NULL arguments, a size shorter than the header or other than
 * the header implies, a bad magic or version, other dimensions or fingerprint, n_past above ctx's n_ctx, a device state n_past that
 * disagrees with the header or a reply tail over 32 bytes. */
MINIGPT4_API long long minigpt4_b200_state_size(struct MiniGPT4Context *ctx);
MINIGPT4_API int minigpt4_b200_state_save(struct MiniGPT4Context *ctx, void *buf, long long cap, long long *written);
MINIGPT4_API int minigpt4_b200_state_load(struct MiniGPT4Context *ctx, const void *buf, long long size);
/* minigpt4_end_chat on each context in turn (each samples from its own logits with its own sampler; greedy uses the device
 * arg-max; tokens[i] = the sampled token's text), then the n sampled ids are fed in one minigpt4_b200_decode_batch step.
 * The batch is validated before any sampling. */
MINIGPT4_API int minigpt4_b200_end_chat_batch(struct MiniGPT4Context **ctxs, int n, const char **tokens, float temp, int32_t top_k, float top_p,
                                              float tfs_z, float typical_p, int32_t repeat_last_n, float repeat_penalty, float alpha_presence,
                                              float alpha_frequency, int mirostat, float mirostat_tau, float mirostat_eta, int penalize_nl);
/* `steps` sampled decode steps of n (1..64) distinct contexts of one group with no return to the host in between: each step samples
 * every context's logits on the device with the chain of minigpt4_end_chat (top_k, tail_free, typical, top_p, temperature, draw;
 * mirostat: minigpt4_b200_sample_steps_mirostat) and its own generator, then feeds the n ids in one decode step (n = 1: the context's own decode graph or megakernel;
 * n >= 2: the batched step of minigpt4_b200_decode_batch).  Queued prompt pieces are evaluated first, as in end_chat_batch.
 * Afterwards every context is where `steps` calls of minigpt4_end_chat (n = 1) or minigpt4_b200_end_chat_batch (n >= 2) with these
 * parameters leave it: n_past, KV cache, logits, greedy id and the generator, which a later minigpt4_end_chat continues.
 * ids_out[s * n + i] = the id context i was fed at step s (its text: minigpt4_b200_token_text); *ms_out (may be NULL) the
 * CUDA-event time of the steps.  temp <= 0 is greedy: the ids of minigpt4_b200_decode_chain / decode_batch, generator untouched.
 * The ids equal the host sampler's except where candidates tie: equal logits are ordered by lower id here (DESIGN.md §4.9).
 * A call always runs exactly `steps` steps; to stop at the end of a reply use minigpt4_b200_sample_until.
 * NULL ctxs / ids_out, NULL or duplicate contexts, contexts of different groups, n outside 1..64, steps < 1, a tensor-parallel
 * context or n_past + steps > n_ctx for any context return the FailedToAddString error code (8) before any device work. */
MINIGPT4_API int minigpt4_b200_sample_steps(struct MiniGPT4Context **ctxs, int n, int steps, float temp, int32_t top_k, float top_p,
                                            float tfs_z, float typical_p, int32_t *ids_out, float *ms_out);
/* A whole reply (or a chunk of one) for n (1..64) contexts of one group: the steps of minigpt4_b200_sample_steps, each context stopping
 * where the reference's chat loop (MiniGPT4ChatBot.generate) stops its reply.  That loop appends the text of every token to the reply,
 * skips the check for a token that is exactly "##", and otherwise stops once the reply ends with "###"; the stopping token is fed.  Here
 * context i stops after the first step whose id's text is not exactly "##" and leaves the reply ending with `stop`, or after max_steps.
 *   stop: NULL means "###" (the reference's EOS_SUFFIX); "" means no text stop; at most 32 bytes.
 *   Texts are the bytes of the C strings minigpt4_end_chat returns (id 2 is "</s>"), with no UTF-8 decoding.
 *   The reply is the text fed since the context's last system_prompt, begin_chat, begin_chat_image, reset_chat, b200_eval_tokens or
 *   b200_eval_embd, by end_chat, end_chat_image, end_chat_batch, sample_steps and sample_until alike: a reply streamed as several calls
 *   stops at the same step as one call, also when the stop text spans two calls.
 * ids_out[s * n + i] = the id context i was fed at step s, -1 after its last step (room for max_steps * n); n_out[i] = the ids fed
 * (1..max_steps); stopped[i] (may be NULL) = 1 if the stop text ended it, 0 if max_steps did; *ms_out (may be NULL) the CUDA-event time.
 * Afterwards context i is where n_out[i] calls of minigpt4_end_chat (n = 1) or end_chat_batch (n >= 2) with these parameters leave it:
 * n_past, logits, greedy id and generator.  A context that stops early is not changed by the steps the others still run.
 * The host checks the stop flags every 4 steps without stalling the device, so up to 7 steps run past the last stop; with n = 1 their
 * K/V writes lie above the context's final position, where its next token overwrites them, and with n >= 2 a stopped context's column
 * is parked on its last id and position, rewriting the same K/V bits.  The first call of a group builds a device table of
 * every id's text (counted in minigpt4_b200_session_info's shared bytes); each context's first call allocates its stop state and a
 * snapshot of its logits (owned bytes).
 * NULL ctxs / ids_out / n_out, NULL or duplicate contexts, contexts of different groups, n outside 1..64, max_steps < 1, a stop text
 * over 32 bytes, a tensor-parallel context or n_past + max_steps > n_ctx for any context return 8 before any device work. */
MINIGPT4_API int minigpt4_b200_sample_until(struct MiniGPT4Context **ctxs, int n, int max_steps, const char *stop, float temp, int32_t top_k,
                                            float top_p, float tfs_z, float typical_p, int32_t *ids_out, int32_t *n_out, int32_t *stopped,
                                            float *ms_out);
/* minigpt4_b200_sample_steps and minigpt4_b200_sample_until with the mirostat sampling of minigpt4_end_chat (mirostat 1 or 2,
 * mirostat_tau, mirostat_eta; as there, top_k, top_p, tfs_z and typical_p do not apply).  Every step sorts the whole vocabulary.
 * Each context keeps its own μ per mirostat mode, set to 2 mirostat_tau at the mode's first use by end_chat or these calls, whichever
 * comes first: afterwards a context is also where that many end_chat / end_chat_batch calls leave its μ, which a later end_chat
 * continues.  temp <= 0 is greedy, and neither μ nor the generator is touched.  Arguments, results and refusals are those of the
 * non-mirostat call; mirostat outside 1..2 also returns 8 before any device work. */
MINIGPT4_API int minigpt4_b200_sample_steps_mirostat(struct MiniGPT4Context **ctxs, int n, int steps, float temp, int mirostat,
                                                     float mirostat_tau, float mirostat_eta, int32_t *ids_out, float *ms_out);
MINIGPT4_API int minigpt4_b200_sample_until_mirostat(struct MiniGPT4Context **ctxs, int n, int max_steps, const char *stop, float temp,
                                                     int mirostat, float mirostat_tau, float mirostat_eta, int32_t *ids_out, int32_t *n_out,
                                                     int32_t *stopped, float *ms_out);
/* Log-probabilities of a generated reply (DESIGN.md §4.14): minigpt4_b200_sample_until (mirostat 0) or minigpt4_b200_sample_until_mirostat
 * (mirostat 1 or 2, which ignores top_k .. typical_p) that also reports, for every id it feeds, how likely that id was.
 * Generation is unchanged: ids_out, n_out, stopped, *ms_out and the state every context is left in (n_past, K / V, logits, greedy id,
 * device state, reply tail, generator, mirostat μ, constraint state) are exactly those of the call it stands for, and a reply streamed
 * over several calls of either function stops at the same step.
 * Records: entry e = s * n + i for step s of context i, s < n_out[i].  z is the logits context i held before step s: the raw model
 * distribution (temperature 1, no top_k / tail_free / typical / top_p / mirostat cut, no constraint), as minigpt4_b200_get_logits returns it.
 *   logprob_out[e] = (float)(((double)z[t] - M) - log sum_v exp((double)z[v] - M)), M = max z, t = ids_out[e]: the bits
 *     minigpt4_b200_score_tokens reports for the same id after the same rows (the same sweep and reduction order).
 *   rank_out[e] (may be NULL) = the ids ranked above t (a larger logit, or an equal logit and a lower id), as score_tokens ranks it.
 *   top_ids_out[e * top_n + j] and top_logprob_out[e * top_n + j] (may be NULL), j < min(top_n, n_vocab): the j-th id in the order
 *     (logit descending, id ascending) and its log-probability by the same formula.  Where rank_out[e] is 0, top_logprob_out[e * top_n]
 *     equals logprob_out[e] bit for bit.
 *   No entry (s >= n_out[i], also for steps the device ran past a context's stop, and j >= n_vocab): ids and ranks -1, log-probabilities NaN.
 *   The arrays hold max_steps * n entries (top arrays: max_steps * n * top_n).
 * Memory: a context's first call allocates its record buffer, n_ctx steps of 168 bytes (up to 20 alternatives each; 336 KiB at n_ctx
 * 2048), counted in minigpt4_b200_session_info's owned bytes.  The records cost one extra kernel launch per step and one device-to-host
 * copy per context at the end.
 * Everything sample_until / sample_until_mirostat refuse, and NULL logprob_out, top_n outside 0..20, top_n > 0 with NULL top_ids_out,
 * mirostat outside 0..2, or an empty conversation (n_past 0, queued rows counted; it has no logits to report on) return 8 before any
 * device work, with nothing changed (queued rows are not evaluated). */
MINIGPT4_API int minigpt4_b200_sample_until_logprobs(struct MiniGPT4Context **ctxs, int n, int max_steps, const char *stop, float temp,
                                                     int32_t top_k, float top_p, float tfs_z, float typical_p, int mirostat, float mirostat_tau,
                                                     float mirostat_eta, int top_n, int32_t *ids_out, int32_t *n_out, int32_t *stopped,
                                                     float *logprob_out, int32_t *rank_out, int32_t *top_ids_out, float *top_logprob_out,
                                                     float *ms_out);
/* Repetition, presence and frequency penalties (DESIGN.md §4.15), opt in: minigpt4_end_chat, end_chat_image, end_chat_batch, sample_steps,
 * sample_until, beam search and the logprob calls take or ignore these arguments as the reference does, and never apply them.
 * The semantics follow llama.cpp master-31cfbb1: llama_sample_repetition_penalty, then llama_sample_frequency_and_presence_penalties, then
 * main.cpp's penalize_nl, applied to a copy of the logits before the unchanged sampler.
 *   Window: the caller supplies each context's recent ids, as llama.cpp's sampling API takes last_tokens.  The window W of context i at
 *   step s of a call is the last min(repeat_last_n, n_last[i] + s) entries of last_ids_i ++ (the ids fed to i at steps 0 .. s-1 of this
 *   call).  Unlike llama.cpp's main, which pre-fills its ring with id 0, W holds only real ids; the engine keeps no history of its own, so
 *   the caller decides whether prompt ids count (MiniGPT4ChatBot.generate_on_device passes the ids of the reply so far).
 *   Penalised logits, in float32 with every operation rounded on its own (no contraction): for each id v with c = its count in W, c >= 1,
 *   and z its raw logit,
 *     z1 = repeat_penalty == 1 ? z : (z <= 0 ? z * repeat_penalty : z / repeat_penalty)   (IEEE division),
 *     z' = (alpha_frequency == 0 && alpha_presence == 0) ? z1 : z1 - ((float)c * alpha_frequency + alpha_presence);
 *   ids with c = 0 keep z, and with penalize_nl 0 and n_vocab > 13 id 13 (llama_token_nl() of that llama.cpp) keeps its raw z.  At
 *   master-31cfbb1 main.cpp restored logits[nl] after the candidates had been copied, so there its restore had no effect; this project
 *   implements the intended behaviour.
 *   Sampling: a step samples z' exactly as sample_until / sample_until_mirostat sample z: the same chain, mirostat μ, generator and
 *   constraint (allowed(s) over z'), the same tie rule (lower id); greedy (temp <= 0) takes the first arg-max of z' (over allowed(s) on a
 *   constrained context).  No draw is added or removed.  The stop rule, max_steps, the steps run past a stop and n_out / stopped are
 *   those of sample_until.
 *   End state: each context ends where n_out[i] calls of minigpt4_b200_end_chat_penalized with the same arguments (last_ids there: the
 *   history and the ids fed before) leave it: n_past and K / V, logits (the raw model logits: the buffer minigpt4_b200_get_logits reads is
 *   never overwritten), greedy id, device state, reply tail, generator, μ and constraint state.
 *   Neutral parameters (repeat_penalty 1 with both alphas 0, any penalize_nl; or repeat_last_n 0): ids and end state are bit-identical to
 *   sample_until / sample_until_mirostat, and the call issues exactly their work.
 * last_ids holds the contexts' histories one after another (context i's n_last[i] ids after those of contexts 0 .. i-1); n_last NULL means
 * no history.  mirostat 0 samples with top_k .. typical_p, 1 or 2 with mirostat (which ignores them).  Other arguments and outputs are
 * those of sample_until.
 * Memory: a context's first call with penalties that are not neutral allocates its penalised row and window counts (8 n_vocab bytes) and
 * a history buffer of n_ctx ids (4 n_ctx bytes; 264 KB at n_vocab 32000, n_ctx 2048), counted in minigpt4_b200_session_info's owned bytes;
 * a later call whose window needs more than n_ctx history ids grows the buffer to them.  The penalties cost one kernel launch per step.
 * Everything sample_until / sample_until_mirostat refuse, and mirostat outside 0..2, repeat_last_n < 0, a non-finite or <= 0
 * repeat_penalty, a non-finite alpha, penalize_nl outside 0..1, n_last[i] < 0, n_last[i] > 0 with NULL last_ids or a history id outside
 * 0..n_vocab-1 return 8 before any device work, with nothing changed (queued rows are not evaluated). */
MINIGPT4_API int minigpt4_b200_sample_until_penalized(struct MiniGPT4Context **ctxs, int n, int max_steps, const char *stop, float temp,
                                                      int32_t top_k, float top_p, float tfs_z, float typical_p, int mirostat, float mirostat_tau,
                                                      float mirostat_eta, int32_t repeat_last_n, float repeat_penalty, float alpha_presence,
                                                      float alpha_frequency, int penalize_nl, const int32_t *last_ids, const int32_t *n_last,
                                                      int32_t *ids_out, int32_t *n_out, int32_t *stopped, float *ms_out);
/* Per-conversation settings in one batched reply call (DESIGN.md §4.16): context i of minigpt4_b200_generate_batch runs with params[i].
 * Layout (80 bytes on LP64; every field at its natural alignment, no padding):
 *   offset  0 size, 4 max_steps, 8 stop, 16 temp, 20 top_k, 24 top_p, 28 tfs_z, 32 typical_p, 36 mirostat, 40 mirostat_tau,
 *   44 mirostat_eta, 48 repeat_last_n, 52 repeat_penalty, 56 alpha_presence, 60 alpha_frequency, 64 penalize_nl, 68 n_last, 72 last_ids. */
struct MiniGPT4B200GenParams {
    int32_t size;            /* sizeof(struct MiniGPT4B200GenParams); any other value is refused */
    int32_t max_steps;       /* this context's budget, >= 1; n_past + max_steps <= n_ctx is required of this context only */
    const char *stop;        /* NULL "###", "" no text stop, at most 32 bytes */
    float temp;              /* <= 0: greedy */
    int32_t top_k;           /* mirostat 0: the chain of minigpt4_end_chat */
    float top_p, tfs_z, typical_p;
    int32_t mirostat;        /* 0 the chain; 1 / 2 mirostat, which ignores top_k .. typical_p */
    float mirostat_tau, mirostat_eta;
    int32_t repeat_last_n;   /* the penalties of minigpt4_b200_sample_until_penalized; neutral ones (repeat_penalty 1 with both alphas 0, */
    float repeat_penalty;    /* or repeat_last_n 0) cost nothing */
    float alpha_presence, alpha_frequency;
    int32_t penalize_nl;
    int32_t n_last;          /* the penalty history: n_last ids at last_ids (may be 0 / NULL) */
    const int32_t *last_ids;
};
/* One reply call over n (1..64) contexts of one group where every context has its own sampler, penalties, stop text and budget.
 * Context i ends exactly where it would end if it ran alone (n = 1) with params[i] through the call those settings select:
 * minigpt4_b200_sample_until (mirostat 0, neutral penalties), sample_until_mirostat (mirostat 1 / 2, neutral penalties),
 * sample_until_penalized (penalties that are not neutral), or with records sample_until_logprobs: the ids, n_out, stopped, n_past and
 * K / V rows 0..n_past-1, logits, greedy id, device state, reply tail, generator, mirostat μ and constraint state, bit for bit.  The one
 * combination no single call has, penalties with records, reports records of the raw logits, as sample_until_logprobs defines them.
 *   Steps: each step samples in one launch per kind of context present (the chain with greedy and constrained contexts; mirostat), then
 *   runs one batched decode step for all n.  The call runs at most S = max max_steps steps and ends once every context is done.  A
 *   context whose reply ended is parked: later steps feed its last id again at that id's own position, which rewrites the same K / V
 *   bits, so nothing is written beyond its final n_past and a budget that ends at n_ctx is safe while others run on.
 *   ids_out[s * n + i] (S * n entries) = the id context i was fed at step s, -1 after its last step; n_out[i] its ids (1..max_steps);
 *   stopped[i] (may be NULL) = 1 if its stop text (or </s> on a constrained context) ended it, 0 if its budget did; *ms_out (may be
 *   NULL) the CUDA-event time.
 *   Records: logprob_out NULL means none (top_n must then be 0); otherwise every context gets them, laid out as sample_until_logprobs
 *   lays them out with max_steps = S, and every context needs n_past >= 1.
 * Memory: only what the single calls allocate (stop state and snapshot; records; the penalty scratch of a context with penalties that are
 * not neutral), counted in minigpt4_b200_session_info's owned bytes.
 * Refusals, each checked per context, return 8 before any device work with nothing changed (queued rows are not evaluated): NULL ctxs /
 * params / ids_out / n_out, n outside 1..64, NULL, duplicate or tensor-parallel contexts, contexts of different groups, a size other
 * than sizeof(struct MiniGPT4B200GenParams), max_steps < 1, n_past + max_steps > n_ctx for that context, a stop text over 32 bytes,
 * mirostat outside 0..2, mirostat on a constrained context, the penalty and history refusals of sample_until_penalized, and with
 * records top_n outside 0..20, top_n > 0 with NULL top_ids_out or an empty conversation; without records top_n other than 0. */
MINIGPT4_API int minigpt4_b200_generate_batch(struct MiniGPT4Context **ctxs, int n, const struct MiniGPT4B200GenParams *params, int top_n,
                                              int32_t *ids_out, int32_t *n_out, int32_t *stopped, float *logprob_out, int32_t *rank_out,
                                              int32_t *top_ids_out, float *top_logprob_out, float *ms_out);
/* The host twin of minigpt4_b200_sample_until_penalized: minigpt4_end_chat with the context's own host sampler run on the penalised copy of
 * its logits, the window being the last min(repeat_last_n, n_last) of last_ids (a host loop passes the history and every id it fed
 * since).  *token = the fed id's text, as minigpt4_end_chat returns it; *id_out (may be NULL) = the id.  The reply tail and constraint
 * state advance as minigpt4_end_chat advances them; with neutral penalties the call is minigpt4_end_chat.  NULL ctx / token and the
 * argument refusals of sample_until_penalized (n_last < 0, NULL last_ids with n_last > 0, a history id out of range, mirostat 1 / 2 on a
 * constrained context) return 8 with nothing changed. */
MINIGPT4_API int minigpt4_b200_end_chat_penalized(struct MiniGPT4Context *ctx, const char **token, float temp, int32_t top_k, float top_p,
                                                  float tfs_z, float typical_p, int32_t repeat_last_n, float repeat_penalty, float alpha_presence,
                                                  float alpha_frequency, int penalize_nl, int mirostat, float mirostat_tau, float mirostat_eta,
                                                  const int32_t *last_ids, int n_last, int32_t *id_out);

/* Beam search (DESIGN.md §4.13): the n_hyp best replies of the conversation of ctxs[0] by beam search with n_beams (1..16) beams, with no
 * host round trip between steps.  ctxs[1 .. n_beams-1] are other contexts of its group that serve as working beams; the call overwrites
 * their conversations.  ctxs[0]'s queued prompt pieces are evaluated first, by its own flush; n0 is then its n_past and T0 its reply tail.
 *   Start: one live beam with no ids, score S = 0.0f, tail T0, beam index 0; H, the finished replies, holds at most n_beams entries.
 *   Step t = 0 .. max_steps-1, for each live beam b with logits z after its ids: lp[v] = (float)((((double)z[v] - M) - log sum_u
 *   exp((double)z[u] - M)), M = max z (the log-probabilities of minigpt4_b200_score_tokens, bit for bit); candidate (b, v) scores c =
 *   S_b + lp[v] (a float32 add).  Candidates are ordered by c descending, then beam index ascending, then z[v] descending, then v
 *   ascending (with one beam: the greedy order, ties included).  The first 2 n_beams candidates are walked in that order, rank r = 0, 1..:
 *   a candidate ends its reply by minigpt4_b200_sample_until's rule (its text is not exactly "##", stop is not empty and tail_b + its
 *   text ends with stop).  An ending candidate with r < n_beams is offered to H with final score (float)((double)c / pow(t + 1,
 *   length_penalty)); one with r >= n_beams is dropped.  Each other candidate becomes the next live beam (S = c, beam index = the order it
 *   is taken in) until n_beams are taken; there may be fewer.
 *   Offering: added while |H| < n_beams; otherwise it replaces the worst entry (lowest score, the later offered on equal scores) if its
 *   score is strictly greater.
 *   End: after the step in which |H| reaches n_beams, or when no live beam is left; the live beams are then not offered (HF generate's
 *   early_stopping=True).  A search that runs through step max_steps-1 offers every live beam, in beam order, with stopped 0.
 * Outputs: the n_hyp best entries of H by final score descending, the earlier offered first on equal scores: ids_out[h * max_steps + j]
 * (-1 padded), n_out[h] (the stopping id included), score_out[h] the final score, logprob_out[h] (may be NULL) its S, stopped[h] (may be
 * NULL) 1 if the stop text ended it; entries beyond |H| get n_out 0 and score -INFINITY.  *ms_out (may be NULL): the CUDA-event time of
 * the search's steps; it leaves out the copy of the conversation into ctxs[1..] at the start and, with 2 or more beams, the prompt pass
 * that evaluates the best reply into ctxs[0] at the end (with one beam the steps feed it).
 * Afterwards ctxs[0] is where minigpt4_b200_sample_until leaves it after feeding the best entry's ids (n_past n0 + n_out[0], K / V,
 * logits bit for bit, greedy id, device state, reply tail), and every other context is as minigpt4_b200_session_copy of ctxs[0] before
 * the call leaves it.  No generator or mirostat μ is touched.  n_beams = 1 gives exactly sample_until with temp 0, the same stop and
 * max_steps.  The group's first call allocates the search state (16 KiB), 2 x 16 x n_ctx ids (256 KiB at n_ctx 2048) and one row of logits,
 * counted in minigpt4_b200_session_info's shared bytes.
 * NULL ctxs / ids_out / n_out / score_out, n_beams outside 1..16, NULL or duplicate contexts, contexts of different groups, max_steps < 1,
 * n_hyp outside 1..n_beams, a stop text over 32 bytes, a non-finite length_penalty, a tensor-parallel or constrained context, an empty
 * conversation (n_past 0, queued rows counted) or n0 + max_steps > n_ctx return 8 before any device work, with nothing changed. */
MINIGPT4_API int minigpt4_b200_beam_search(struct MiniGPT4Context **ctxs, int n_beams, int max_steps, const char *stop, float length_penalty,
                                           int n_hyp, int32_t *ids_out, int32_t *n_out, float *score_out, float *logprob_out, int32_t *stopped,
                                           float *ms_out);

/* Constrained replies (DESIGN.md §4.12): sample only the ids a deterministic automaton over bytes allows.  The automaton has n_states
 * states (1..65536), start state 0; next[s * 256 + b] is the state byte b leads to from s, or -1 to reject; accept[s] != 0 marks an
 * accepting state.  The text of an id is the C string minigpt4_end_chat returns for it (an id whose text is empty is never allowed).
 *   allowed(s) = every id other than 2 whose text, walked byte by byte from s, never meets -1 and ends in a live state, plus id 2 (</s>)
 *   if s accepts.  A state is live if some sequence of allowed ids leads from it to an accepting state (computed on the ids, to a fixed
 *   point).  An id moves the state to where its walk ends; id 2 moves it to the finished state, which allows only id 2.
 * On a constrained context, minigpt4_end_chat / end_chat_image, minigpt4_b200_end_chat_batch, sample_steps and sample_until run the
 * unchanged sampler chain over allowed(s) only, in id order: top_k is clamped to |allowed(s)| and temp <= 0 takes the arg-max over
 * allowed(s), the lower id on ties.  Each fed id moves the state; sample_until also stops a constrained context after the step that
 * feeds id 2 (stopped = 1).  decode_chain, decode_batch, the two _mirostat calls and end_chat / end_chat_batch with mirostat 1 or 2
 * return 8 on a constrained context and change nothing; get_logits and greedy_id stay unconstrained.
 * The state restarts where the reply tail does (system_prompt, begin_chat, begin_chat_image, reset_chat, eval_tokens, eval_embd,
 * score_tokens with keep 1) and at state_load (the saved state carries no constraint); session_copy gives a destination with the source's
 * constraint attached the source's state and restarts any other destination's. */
struct MiniGPT4B200Constraint;
/* compile against ctx's vocabulary; the device tables belong to ctx's group (counted in session_info's shared bytes).  NULL for
 * n_states outside 1..65536, next[] outside -1..n_states-1, a start state that is not live, a tensor-parallel ctx, more than 2^31-1
 * transitions, or device memory exhausted. */
MINIGPT4_API struct MiniGPT4B200Constraint *minigpt4_b200_constraint_create(struct MiniGPT4Context *ctx, int n_states, const int32_t *next,
                                                                            const uint8_t *accept);
/* drops the handle; the tables live until no context has them attached */
MINIGPT4_API void minigpt4_b200_constraint_free(struct MiniGPT4B200Constraint *c);
/* attach c to ctx with its state at the start (c NULL: detach); 8 for a constraint compiled for another group */
MINIGPT4_API int minigpt4_b200_constraint_attach(struct MiniGPT4Context *ctx, struct MiniGPT4B200Constraint *c);
/* ctx's state (-1 once finished) and whether it is finished; 8 if no constraint is attached */
MINIGPT4_API int minigpt4_b200_constraint_state(struct MiniGPT4Context *ctx, int *state, int *finished);
/* allowed(state) as compiled: ids ascending (ids may be NULL) and the state each leads to (next_states may be NULL; -1: finished).
 * Returns the count, -count if cap is short, -1 for a state that is not live or outside 0..n_states-1 (a one-id row asked with cap 0
 * also returns -1: ask with cap >= 1). */
MINIGPT4_API int minigpt4_b200_constraint_allowed(struct MiniGPT4B200Constraint *c, int state, int32_t *ids, int32_t *next_states, int cap);
/* host-only seam (no GPU): the same, compiled against the vocabulary of a ggjt file; -1000000 for an unreadable file or a refused
 * automaton */
MINIGPT4_API int minigpt4_b200_host_constraint_allowed(const char *llm_model, int n_states, const int32_t *next, const uint8_t *accept, int state,
                                                       int32_t *ids, int32_t *next_states, int cap);

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
/* Vision kernel seams.  Each runs one production kernel with the launch configuration the vision graph gives it, and returns 8
 * (FailedToAddString) for arguments the kernel cannot take, before any device work.
 * out = epi(X[T][K] . W[M][K]^T) through the wgmma GEMM, F16 operands, the plan (token tile, token split, split-K) built as at load time.
 * epi 0: bias + acc; 1: (bias + acc) * qscale on features < qscale_rows, bias + acc above; 2: GELU (fp16 LUT) of bias + acc, F16 out;
 * 3: aux[t] + (bias + acc) (aux = resid [T][M]; in_place: the pre-filled rows of `out` are the residual, as when the vision graph runs
 * without split-K); 4: out row t + 1 = (0 + bias + acc) + aux[t + 1] (aux = pos [T + 1][M]; row 0 is left alone).
 * tsplit: split the tokens of T > 128 over CTAs (the default; 0 as with MINIGPT4_B200_VISION_TSPLIT=0).  ksplit 1..4 (epi 3 only): when the
 * plan splits K (tsplit, T > 128), grid.z slices of raw sums (bias on slice 0) go to the leading slices of `out`.
 * out: [ksplit][T + 1 + (epi == 4)][M] (F16 for epi 2, F32 otherwise), pre-filled by the caller and returned whole, so the row past the last
 * one written is a guard row.  plan_out (may be NULL): {token tile, grid.y, grid.z, k-blocks per slice}.
 * Out of range: M % 128, K % 64, T outside 1..272, epi outside 0..4, ksplit outside 1..4 or > 1 with epi != 3, a missing aux. */
MINIGPT4_API int minigpt4_b200_op_gemm_f16(int M, int T, int K, const void *w_f16, const void *x_f16, const float *bias, int epi, const float *aux,
                                           float qscale, int qscale_rows, int ksplit, int tsplit, int in_place, void *out, int32_t *plan_out);
/* LayerNorm (eps 1e-5) of rows x [rows][n] with weight w and bias b (may be NULL); out32 F32 and / or out16 F16 [rows][n] (either may be
 * NULL, not both).  n outside 1..1536 is out of range. */
MINIGPT4_API int minigpt4_b200_op_layernorm(const float *x, int rows, int n, const float *w, const float *b, float *out32, void *out16);
/* the LayerNorm that follows a split-K residual GEMM: x [rows][n] (in / out) becomes ((x + parts[0]) + parts[1]) + ... (slice p at element
 * p * part_stride, part_stride >= rows * n), and out16 = F16 LayerNorm of it */
MINIGPT4_API int minigpt4_b200_op_layernorm_fold(float *x, int rows, int n, const float *w, const float *b, const float *parts, int n_parts,
                                                 long long part_stride, void *out16);
/* attention over `heads` heads of dh (64 or 88): q, k, v at element offsets q_off / k_off / v_off of buf[n_buf] with row pitches ldq / ldkv
 * (multiples of 4), scores / score_div, fp16-LUT softmax; q_per_cta queries per CTA (0: ceil(nq / 4)).  out: [nq + 1][ld_out] pre-filled by
 * the caller and returned whole: rows < nq, columns < heads * dh get the F16-rounded context, row nq is a guard row.  Out of range: nk
 * outside 1..288 or past what shared memory holds (dh 88: 268 keys), dh not 64 / 88, spans outside buf. */
MINIGPT4_API int minigpt4_b200_op_attention(const float *buf, long long n_buf, long long q_off, int ldq, long long k_off, long long v_off, int ldkv,
                                            int nq, int nk, int heads, int dh, float score_div, int q_per_cta, int ld_out, float *out);
/* minigpt4_encode_image's forward on ctx's first lane, run eagerly (not as the graph) with every stage copied out once it is complete; each
 * pointer may be NULL.  image F32 CHW [3][224][224]; embed [257][D]: patch embedding + CLS + positions; vit_blocks [n_blocks][257][D]: the
 * residual stream after each block; ln_vision [257][D]: the F16 Q-Former operand as F32; qformer [q_layers][32][768]: the hidden states after
 * each layer; out [32][n_embd_llm]: the embedding minigpt4_encode_image returns.  8 for a NULL ctx / image or a context without vision. */
MINIGPT4_API int minigpt4_b200_encode_taps(struct MiniGPT4Context *ctx, const float *image, float *embed, float *vit_blocks, float *ln_vision,
                                           float *qformer, float *out);
/* the LLaMA attention of the decode step and prompt passes: q F32 [rows][n_head*128], k_f16 / v_f16 F16 caches [n_ctx][n_head*128]
 * (row t sees keys 0 .. its position; rows above are never read), out F32 [rows][n_head*128].  path 0: the single-context kernel, row t
 * at pos[0] + t; path 1: the batched kernel, row t at pos[t].  8 (FailedToAddString) on arguments out of range, before any device work */
MINIGPT4_API int minigpt4_b200_op_llama_attention(const float *q, const void *k_f16, const void *v_f16, int n_head, int n_ctx, int rows, const int32_t *pos,
                                                  int path, float *out);

/* out_f16[n] = the F16 operand the vision graph builds at load time from a non-F16 matrix: `raw` holds n elements as ggml blocks of
 * `ggml_type` (0 F32, 2 Q4_0, 3 Q4_1, 6 Q5_0, 7 Q5_1, 8 Q8_0); values follow ggml's dequantize_row_* and are rounded to F16 */
MINIGPT4_API int minigpt4_b200_op_dequant_f16(int ggml_type, const void *raw, long n, void *out_f16);

/* host-only seams (no GPU touched): the tokenizer / sampler / file readers are host logic and are unit-tested on CPU */
/* tokenise with the vocabulary stored in a ggjt file; returns count or -needed (llama_tokenize convention), -1000000 on read failure */
MINIGPT4_API int minigpt4_b200_host_tokenize(const char *llm_model, const char *text, int add_bos, int32_t *out, int max_tokens);
/* run the sampler chain of minigpt4_end_chat on caller-provided logits (reference minigpt4.cpp:2425-2483) */
MINIGPT4_API int minigpt4_b200_host_sample(const float *logits, int n_vocab, int seed, float temp, int32_t top_k, float top_p, float tfs_z,
                                           float typical_p, int mirostat, float mirostat_tau, float mirostat_eta, int n_draws, int32_t *out_ids);
/* the device twin of minigpt4_b200_host_sample (no mirostat, which minigpt4_b200_op_sample_mirostat covers; temp > 0): n_draws draws
 * over the same logits from one generator seeded with `seed`, through the kernel of minigpt4_b200_sample_steps; 8 for bad arguments.  The _timed form also returns the
 * average CUDA-event time of one sampling launch. */
MINIGPT4_API int minigpt4_b200_op_sample(const float *logits, int n_vocab, int seed, float temp, int32_t top_k, float top_p, float tfs_z,
                                         float typical_p, int n_draws, int32_t *out_ids);
MINIGPT4_API int minigpt4_b200_op_sample_timed(const float *logits, int n_vocab, int seed, float temp, int32_t top_k, float top_p, float tfs_z,
                                               float typical_p, int n_draws, int32_t *out_ids, float *kernel_ms);
/* minigpt4_b200_sample_until's stop rule on the device, over the ids ids[0..n) of ctx's vocabulary from a reply that ends with `tail`
 * (NULL: empty; its last 32 bytes count): *stop_at = the index of the id after which the reply ends, -1 if none; stop as in
 * sample_until.  Changes nothing in ctx.  8 for a NULL ctx / stop_at, an id outside the vocabulary or a stop text over 32 bytes. */
/* mirostat (1 or 2) over the same logits from one generator seeded with `seed` and an unset μ: n_draws calls of the host Sampler
 * (on_device 0) or launches of minigpt4_b200_sample_steps_mirostat's kernel (on_device 1, temp > 0); ids_out[d] = draw d's id and
 * mu_out[d] = μ after it; *kernel_ms (may be NULL) = the average CUDA-event time of one launch (0 on the host).  8 for NULL
 * logits / ids_out / mu_out, n_vocab < 1, n_draws < 1, mirostat outside 1..2, on_device outside 0..1, or temp <= 0 on the device. */
MINIGPT4_API int minigpt4_b200_op_sample_mirostat(const float *logits, int n_vocab, int seed, float temp, int mirostat, float mirostat_tau,
                                                  float mirostat_eta, int n_draws, int on_device, int32_t *ids_out, float *mu_out, float *kernel_ms);
/* minigpt4_b200_beam_search's ordering through its kernels, without the stop rule: n_live (1..n_beams) beams with scores S[n_live] and
 * logits [n_live][n_vocab], n_beams 1..16; parent_out / id_out / c_out [2 n_beams] receive the first min(2 n_beams, n_live n_vocab)
 * candidates in order (the rest is not written).  8 for NULL arguments or out-of-range sizes. */
MINIGPT4_API int minigpt4_b200_op_beam_rank(const float *logits, int n_live, const float *S, int n_beams, int n_vocab, int32_t *parent_out,
                                            int32_t *id_out, float *c_out);
/* minigpt4_b200_sample_until_logprobs' records through its kernel, over host rows: logits [rows][n_vocab] (rows 1..64), ids[rows] (one id
 * per row, 0..n_vocab-1, as if each row's step had fed it), top_n 0..20.  logprob_out[rows], rank_out[rows] (may be NULL),
 * top_ids_out / top_logprob_out (may be NULL) [rows][top_n], with the semantics and the -1 / NaN padding of sample_until_logprobs.
 * *kernel_ms (may be NULL): the average CUDA-event time of one launch over all rows.  8 for NULL logits / ids / logprob_out, a NULL
 * top_ids_out with top_n > 0, or out-of-range sizes or ids, before any device work. */
MINIGPT4_API int minigpt4_b200_op_logprobs(const float *logits, int rows, int n_vocab, const int32_t *ids, int top_n, float *logprob_out,
                                           int32_t *rank_out, int32_t *top_ids_out, float *top_logprob_out, float *kernel_ms);
/* minigpt4_b200_sample_until_penalized's penalised logits over host rows: logits [rows][n_vocab] (rows 1..64), row r's window the last
 * min(repeat_last_n, n_last[r]) of its history (last_ids: the rows' histories one after another; n_last NULL: none), as at step 0 of that
 * call; out [rows][n_vocab] = z'.  on_device 1: its kernel, *kernel_ms (may be NULL) the average CUDA-event time of one launch over all
 * rows; on_device 0: the host sampler's penalize (no GPU touched), *kernel_ms 0.  8 for NULL logits / out, out-of-range sizes, on_device
 * outside 0..1 and the penalty refusals of sample_until_penalized, before any device work. */
MINIGPT4_API int minigpt4_b200_op_penalize(const float *logits, int rows, int n_vocab, const int32_t *last_ids, const int32_t *n_last,
                                           int32_t repeat_last_n, float repeat_penalty, float alpha_presence, float alpha_frequency, int penalize_nl,
                                           int on_device, float *out, float *kernel_ms);
MINIGPT4_API int minigpt4_b200_op_reply_stop(struct MiniGPT4Context *ctx, const int32_t *ids, int n, const char *stop, const char *tail,
                                             int32_t *stop_at);
/* the device sampler's expf (fn 0) / logf (fn 1) over the float bit patterns lo_bits .. hi_bits (inclusive), compared bit for bit with
 * the host libm's; *mismatches = the number that differ */
MINIGPT4_API int minigpt4_b200_op_check_libm(int fn, uint32_t lo_bits, uint32_t hi_bits, long long *mismatches);
/* the same for mirostat's log2f over the bit patterns lo_bits .. hi_bits, and its powf(x, y) over the y of those bit patterns; 8 for
 * hi_bits < lo_bits or a NULL mismatches */
MINIGPT4_API int minigpt4_b200_op_check_log2f(uint32_t lo_bits, uint32_t hi_bits, long long *mismatches);
MINIGPT4_API int minigpt4_b200_op_check_powf(float x, uint32_t lo_bits, uint32_t hi_bits, long long *mismatches);
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

// llama_penalty.cuh — sm_90a kernel of minigpt4_b200_sample_until_penalized (host side LlamaDevice::sample_until in llama.cu, DESIGN.md
// §4.15).
//
// A step of sample_until with penalties runs one extra launch before its sampling launch.  penalty_rows_kernel copies each context's raw
// logits into its penalised row, then rewrites the ids of the step's window there (Sampler::penalize, text.cpp).  Each column carries its
// own parameters, and the launch covers the penalised columns only: the others sample their raw logits and cost nothing here.  The sampling launch's
// columns read that row instead of the raw logits, so the sampling kernels run unchanged; the raw logits, which the decode step writes,
// are never touched.  Greedy columns also get the first arg-max of the penalised row in DeviceState::tokens[0], the id the greedy
// sampling path feeds.
#pragma once
#include "llama_sample.cuh"

namespace mg4 {
namespace pen {

constexpr int kThreads = 256;

struct PenaltyCol {
    const float *logits;              // [n_vocab] the raw row (the decode step's logits)
    float *row;                       // [n_vocab] the penalised row the step samples from
    int *count;                       // [n_vocab] window counts; all zero between launches
    const int *tail;                  // the last n_tail ids of the caller's history (n_tail <= repeat_last_n)
    const int *fed;                   // SampleCtx::ids: the ids fed at steps 0 .. step - 1 of this call
    DeviceState *state;               // greedy: tokens[0] takes the first arg-max of the row (null: not written)
    const smp::ReplyState *reply;     // done != 0: the column stopped (null: it runs, the test seam)
    int n_tail;
    PenaltyParams q;                  // the column's penalties
    int greedy;                       // the column samples greedily (temp <= 0)
};
struct PenaltyArgs {
    PenaltyCol c[LlamaDevice::kMaxBatch];
    int n_vocab, step;
};

// z' of an id with c >= 1 copies in the window (every operation rounded on its own: the build passes -fmad=false)
__device__ __forceinline__ float penalized(float z, int c, const PenaltyParams &a) {
    const float z1 = a.repeat_penalty == 1.0f ? z : (z <= 0.f ? z * a.repeat_penalty : z / a.repeat_penalty);
    return (a.alpha_frequency == 0.f && a.alpha_presence == 0.f) ? z1 : z1 - ((float)c * a.alpha_frequency + a.alpha_presence);
}

// grid = columns, block kThreads.  Window of a column at step s: the last min(repeat_last_n, n_tail + s) entries of tail ++ fed[0, s).
// A column that stopped at the previous step (done 1) gets the raw row copied only: the sampling launch saves that row as the
// context's logits snapshot.  A column already saved (done 2) is left alone.
__global__ void __launch_bounds__(kThreads) penalty_rows_kernel(const __grid_constant__ PenaltyArgs a) {
    const PenaltyCol &col = a.c[blockIdx.x];
    const int done = col.reply ? col.reply->done : 0;
    if (done == 2) return;
    const int tid = threadIdx.x, V = a.n_vocab;
    const float *__restrict__ z = col.logits;
    float *__restrict__ out = col.row;
    // ---- the copy: 16-byte vectors where both rows allow them
    int i0 = 0;
    if ((((uintptr_t)z | (uintptr_t)out) & 15) == 0) {
        const float4 *z4 = (const float4 *)z;
        float4 *o4 = (float4 *)out;
        for (int i = tid; i < V / 4; i += kThreads) o4[i] = z4[i];
        i0 = V / 4 * 4;
    }
    for (int i = i0 + tid; i < V; i += kThreads) out[i] = z[i];
    if (done) return;
    // ---- counts of the window's ids, then each entry rewrites its id (copies of one id write the same value)
    const int T = col.n_tail, end = T + a.step, first = end - min(col.q.repeat_last_n, end);
    for (int j = first + tid; j < end; j += kThreads) atomicAdd(&col.count[j < T ? col.tail[j] : col.fed[j - T]], 1);
    __syncthreads();
    const bool keep_nl = !col.q.penalize_nl && V > 13;
    for (int j = first + tid; j < end; j += kThreads) {
        const int v = j < T ? col.tail[j] : col.fed[j - T];
        if (!(keep_nl && v == 13)) out[v] = penalized(z[v], col.count[v], col.q);
    }
    __syncthreads();
    for (int j = first + tid; j < end; j += kThreads) col.count[j < T ? col.tail[j] : col.fed[j - T]] = 0;
    if (!col.greedy || !col.state) return;
    // ---- greedy: the first arg-max of the penalised row (the largest smp::desc_key: logit desc, then the lower id)
    __shared__ unsigned long long best;
    if (tid == 0) best = 0ull;
    __syncthreads();
    unsigned long long k = 0ull;
    for (int i = tid; i < V; i += kThreads) k = max(k, smp::desc_key(out[i], i));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) k = max(k, __shfl_xor_sync(0xffffffffu, k, o));
    if ((tid & 31) == 0) atomicMax(&best, k);
    __syncthreads();
    if (tid == 0) col.state->tokens[0] = smp::key_id(best);
}

}  // namespace pen
}  // namespace mg4

// llama_logprob.cuh — sm_90a kernel of minigpt4_b200_sample_until_logprobs (host side LlamaDevice::sample_until in llama.cu, DESIGN.md
// §4.14).
//
// A step of sample_until with records runs one extra launch between the sampling launch and the decode step.  At that point each
// context's logits still hold the distribution the step sampled from, and DeviceState::tokens[0] holds the id the decode step is about to
// feed.  logprob_rows_kernel writes that id's log-probability and rank under the raw logits (temperature 1, no cut, no constraint) and the
// row's top_n ids with their log-probabilities into the context's record of the step.
#pragma once
#include "llama_sample.cuh"

namespace mg4 {
namespace lp {

constexpr int kMaxTop = LlamaDevice::kLogprobTop;
constexpr int kThreads = 256;   // score_rows_kernel's block: the same strided sums and reduction tree

struct Record {                 // one step of one context
    float logprob;
    int rank;
    int top_id[kMaxTop];        // -1 past min(top_n, n_vocab)
    float top_lp[kMaxTop];      // NaN there
};
static_assert(sizeof(Record) == LlamaDevice::kLogprobRecordBytes, "the record size the header states");

struct LogprobCol {
    const float *logits;
    const DeviceState *state;          // tokens[0]: the id this step feeds
    const smp::ReplyState *reply;      // the column fed at this step iff n_fed == step + 1; null: it always did (the test seam)
    Record *rec;                       // [n_ctx] the context's records; step s goes to rec[s]
};
struct LogprobArgs {
    LogprobCol c[LlamaDevice::kMaxBatch];
    int n_vocab, step, top_n;
};

// grid = columns, block kThreads.  lp(v) = (float)(((double)z[v] - M) - log S), M = max z, S = sum exp((double)z - M), with the sweep and
// reduction of score_rows_kernel (llama_score.cuh, restated here so that neither kernel's code changes), so the fed id's lp and rank are the
// bits minigpt4_b200_score_tokens reports for it.  The top ids are those of the order (logit desc, id asc): the 8-bit radix select of
// beam_rank_kernel over smp::desc_key, whose first pass is taken during the sweep, then a rank count among the <= kMaxTop winners.
__global__ void __launch_bounds__(kThreads) logprob_rows_kernel(const __grid_constant__ LogprobArgs a) {
    const LogprobCol &col = a.c[blockIdx.x];
    if (col.reply && col.reply->n_fed != a.step + 1) return;   // stopped before this step: nothing was fed
    const int tid = threadIdx.x, top_n = a.top_n;   // (blockDim.x == kThreads)
    const float *__restrict__ z = col.logits;
    Record &rec = col.rec[a.step];
    __shared__ float sm[8];
    __shared__ double ss[8];
    __shared__ int sr[8];
    __shared__ double sh_M, sh_logS;
    __shared__ unsigned hist[256];
    __shared__ unsigned long long sh_prefix;
    __shared__ int sh_need, sh_done, sh_n;
    __shared__ unsigned long long win_key[kMaxTop];
    __shared__ float win_z[kMaxTop];
    if (top_n > 0) hist[tid] = 0u;   // (kThreads == 256 bins)
    __syncthreads();
    const int target = col.state->tokens[0];
    const float zt = z[target];
    // ---- M, S and the rank, as score_rows_kernel takes them; the top byte's histogram on the way
    float m = -INFINITY;
    double s = 0.0;
    int rank = 0;
    // (each thread takes its ids in score_rows_kernel's order, kUnroll loads in flight ahead of the dependent sums)
    constexpr int kUnroll = 8;
    for (int i0 = tid; i0 < a.n_vocab; i0 += kUnroll * kThreads) {
        float vs[kUnroll];
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) vs[u] = i0 + u * kThreads < a.n_vocab ? z[i0 + u * kThreads] : 0.f;
#pragma unroll
        for (int u = 0; u < kUnroll; ++u) {
            const int i = i0 + u * kThreads;
            if (i >= a.n_vocab) break;
            const float v = vs[u];
            rank += (v > zt) || (v == zt && i < target);
            if (v > m) { s = s * exp((double)m - (double)v) + 1.0; m = v; }
            else s += exp((double)v - (double)m);
            if (top_n > 0) atomicAdd(&hist[smp::desc_key(v, i) >> 56], 1u);
        }
    }
    const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float mo = __shfl_xor_sync(0xffffffffu, m, o);
        const double so = __shfl_xor_sync(0xffffffffu, s, o);
        rank += __shfl_xor_sync(0xffffffffu, rank, o);
        const float mm = fmaxf(m, mo);
        s = (m == -INFINITY ? 0.0 : s * exp((double)m - (double)mm)) + (mo == -INFINITY ? 0.0 : so * exp((double)mo - (double)mm));
        m = mm;
    }
    if (lane == 0) { sm[warp] = m; ss[warp] = s; sr[warp] = rank; }
    __syncthreads();
    if (tid == 0) {
        const int nw = (int)(blockDim.x >> 5);
        float M = -INFINITY;
        for (int w = 0; w < nw; ++w) M = fmaxf(M, sm[w]);
        double S = 0.0;
        int R = 0;
        for (int w = 0; w < nw; ++w) {
            if (sm[w] != -INFINITY) S += ss[w] * exp((double)sm[w] - (double)M);
            R += sr[w];
        }
        sh_M = (double)M; sh_logS = log(S);
        rec.logprob = (float)(((double)zt - (double)M) - log(S));
        rec.rank = R;
        sh_prefix = 0ull;
        sh_need = min(top_n, a.n_vocab);
        sh_n = 0;
    }
    const int k = min(top_n, a.n_vocab);
    for (int j = k + tid; j < kMaxTop; j += blockDim.x) { rec.top_id[j] = -1; rec.top_lp[j] = __int_as_float(0x7fffffff); }
    if (k == 0) return;
    // ---- the top k keys: radix select from the top byte to the threshold T with exactly k keys >= T (keys are distinct)
    unsigned long long mask = 0ull;
    for (int shift = 56; shift >= 0; shift -= 8) {
        if (shift != 56) {   // (the top byte's histogram came with the sweep)
            hist[tid] = 0u;
            __syncthreads();
            const unsigned long long pre = sh_prefix;
            for (int i = tid; i < a.n_vocab; i += blockDim.x) {
                const unsigned long long key = smp::desc_key(z[i], i);
                if ((key & mask) == pre) atomicAdd(&hist[(key >> shift) & 255], 1u);
            }
        }
        __syncthreads();
        if (tid == 0) {
            int need = sh_need, d = 255; unsigned cum = 0;
            for (; d > 0; --d) { if (cum + hist[d] >= (unsigned)need) break; cum += hist[d]; }
            need -= (int)cum;
            sh_prefix |= (unsigned long long)d << shift;
            sh_need = need;
            sh_done = hist[d] == (unsigned)need;
        }
        __syncthreads();
        mask |= 255ull << shift;
        if (sh_done) break;
    }
    const unsigned long long T = sh_prefix;
    for (int i = tid; i < a.n_vocab; i += blockDim.x) {
        const float v = z[i];
        const unsigned long long key = smp::desc_key(v, i);
        if (key >= T) { const int j = atomicAdd(&sh_n, 1); win_key[j] = key; win_z[j] = v; }
    }
    __syncthreads();
    // ---- the winners in order: each one's place is the count of winners with a larger key
    if (tid < k) {
        const unsigned long long key = win_key[tid];
        int r = 0;
        for (int j = 0; j < k; ++j) r += win_key[j] > key;
        rec.top_id[r] = smp::key_id(key);
        rec.top_lp[r] = (float)(((double)win_z[tid] - sh_M) - sh_logS);
    }
}

}  // namespace lp
}  // namespace mg4

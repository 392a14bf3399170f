// llama_score.cuh — sm_90a kernel of minigpt4_b200_score_tokens (host side LlamaDevice::score_rows in llama.cu, DESIGN.md §4.10).
//
// A scoring call runs the batched prompt pass over the ids to be scored and computes every row's logits with matvec_sessions_kernel
// (EPI_LOGITS) into a group-owned scratch, so each row's logits are the bits the context would hold after evaluating its ids up to that
// row.  This kernel turns one logits row and a target id into the target's log-probability and rank.
#pragma once
#include <cuda_runtime.h>
#include <math.h>

namespace mg4 {
namespace k {

struct ScoreRow { const float *logits; int target; int pad; };   // one scored entry: the logits that predict it, its id
struct ScoreOut { float logprob; int rank; };

// grid = scored entries, block 256: one sweep over the row keeps, per thread, the max m, the sum of exp(z - m) in double (rescaled when m
// grows), and the count of ids ranked above the target (a larger logit, or an equal logit and a lower id: the device sampler's tie
// rule, DESIGN.md §4.9); the block then merges them.  logprob = (float)((z_t - M) - log S), S = sum exp((double)z - M), M the row's max.
__global__ void __launch_bounds__(256) score_rows_kernel(const ScoreRow *__restrict__ rows, int n_vocab, ScoreOut *__restrict__ out) {
    __shared__ float sm[8];
    __shared__ double ss[8];
    __shared__ int sr[8];
    const ScoreRow r = rows[blockIdx.x];
    const float *__restrict__ z = r.logits;
    const float zt = z[r.target];
    float m = -INFINITY;
    double s = 0.0;
    int rank = 0;
    for (int i = threadIdx.x; i < n_vocab; i += blockDim.x) {
        const float v = z[i];
        rank += (v > zt) || (v == zt && i < r.target);
        if (v > m) { s = s * exp((double)m - (double)v) + 1.0; m = v; }
        else s += exp((double)v - (double)m);
    }
    // warp, then block: (m, s) pairs merged onto the larger max; a thread that saw no id has m = -inf and adds nothing
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
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
    if (threadIdx.x == 0) {
        const int nw = (int)(blockDim.x >> 5);
        float M = -INFINITY;
        for (int w = 0; w < nw; ++w) M = fmaxf(M, sm[w]);
        double S = 0.0;
        int R = 0;
        for (int w = 0; w < nw; ++w) {
            if (sm[w] != -INFINITY) S += ss[w] * exp((double)sm[w] - (double)M);
            R += sr[w];
        }
        out[blockIdx.x] = ScoreOut{(float)(((double)zt - (double)M) - log(S)), R};
    }
}

}  // namespace k
}  // namespace mg4

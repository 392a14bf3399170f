// llama_sessions.cuh — sm_90a kernels of the batched decode step and the batched prompt pass over several contexts that share one
// model (minigpt4_b200_decode_batch / flush_batch; host side LlamaDevice::decode_batch / eval_rows_batch in llama.cu, DESIGN.md §4.8).
//
// Column t of a batch belongs to context t: its own position, KV cache, logits buffer and DeviceState come from a small
// device table (SessionSlot[B]) that the host refreshes with one copy per step, so the captured graph of each batch size is
// position independent like the single-context decode graph.  The weights stream once for all B columns.
//
// BIT-EXACT PARITY: the block dots are the dot2_* functions of llama_kernels.cuh, unchanged, and every row of a matvec is
// reduced on its own whatever the column count, so a column's result is the bits a single-context step produces.  Attention
// calls attention_head with the column's own cache and position (canonical order by construction).  Only the epilogues that
// address per-context memory (QKV append, logits + arg-max) differ from matvec_kernel; the residual and SwiGLU matrices of
// the batch run through matvec_kernel itself.
#pragma once
#include "llama_kernels.cuh"

namespace mg4 {
namespace k {

struct SessionMatvecArgs {
    MatvecArgs m;                 // w, x, norm_w, staged, ntok (= B), rows_per_warp, epi (EPI_QKV | EPI_LOGITS), n_valid, q_out, rope, e_local, half_dim, part
    const SessionSlot *slots;     // [B]
    size_t kv_off;                // this layer's offset into every context's K / V cache (layer * n_ctx * e_local)
};

template <int WT, int NT>
__global__ void __launch_bounds__(kThreads, 2) matvec_sessions_kernel(const SessionMatvecArgs sa) {
    extern __shared__ __align__(16) unsigned char smem[];
    const MatvecArgs &a = sa.m;
    constexpr int ACT = act_of(WT);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const size_t astride = act_bytes(ACT, a.w.cols);
    {   // the B input rows were staged once by stage_kernel
        const uint4 *src = (const uint4 *)a.staged; uint4 *dst = (uint4 *)smem;
        const int n16 = (int)((size_t)a.ntok * astride / 16);
        for (int i = threadIdx.x; i < n16; i += kThreads) dst[i] = src[i];
    }
    __syncthreads();

    const int row_begin = (blockIdx.x * kWarps + warp) * a.rows_per_warp;
    const int row_end = min(row_begin + a.rows_per_warp, a.w.rows);
    unsigned long long best = 0ull;   // EPI_LOGITS: lane t < ntok keeps column t's arg-max key
    for (int r0 = row_begin; r0 < row_end; r0 += 2) {
        float res[2][NT];
        if (WT == GG_Q4_1 || WT == GG_Q4_0) {
            const unsigned char *row0 = (const unsigned char *)a.w.p0 + (size_t)r0 * a.w.row_bytes;
            dot2_q4<NT, false>(row0, row0 + a.w.row_bytes, a.w.cols / 32, a.w.cols, WT == GG_Q4_1, smem, astride, lane, res);
        }
        else if (WT == GG_Q5_K) dot2_q5k<NT>(a.w, r0, smem, astride, lane, res);
        else if (WT == GG_Q4_K) dot2_q4k<NT>(a.w, r0, smem, astride, lane, res);
        else if (WT == GG_Q5_0 || WT == GG_Q5_1 || WT == GG_Q8_0) dot2_b32<WT, NT>(a.w, r0, smem, astride, lane, res);
        else if (WT == GG_Q6_K) dot2_q6k<NT>(a.w, r0, smem, astride, lane, res);
        else dot2_f16<NT>(a.w, r0, smem, astride, lane, res);

#pragma unroll
        for (int t = 0; t < NT; ++t) {
            if (lane != t || t >= a.ntok) continue;
            const SessionSlot &s = sa.slots[t];
            const float v0 = res[0][t], v1 = res[1][t];
            if (a.epi == EPI_LOGITS) {
                s.logits[r0] = v0;
                const unsigned long long k0 = argmax_key(v0, r0);
                best = best > k0 ? best : k0;
                if (r0 + 1 < a.n_valid) {
                    s.logits[r0 + 1] = v1;
                    const unsigned long long k1 = argmax_key(v1, r0 + 1);
                    best = best > k1 ? best : k1;
                }
                continue;
            }
            // EPI_QKV: one token per column, at the column's own position, into the column's own cache
            const int E = a.e_local;
            const int part = a.part >= 0 ? a.part : r0 / E, rr = a.part >= 0 ? r0 : r0 % E;
            const int pos = s.n_past;
            if (part == 2) {
                *(__half2 *)(s.vcache + sa.kv_off + (size_t)pos * E + rr) = __floats2half2_rn(v0, v1);
            } else {
                const float2 cs = a.rope[(size_t)pos * a.half_dim + (rr % (2 * a.half_dim)) / 2];
                const float o0 = v0 * cs.x - v1 * cs.y, o1 = v0 * cs.y + v1 * cs.x;
                if (part == 0) *(float2 *)(a.q_out + (size_t)t * E + rr) = make_float2(o0, o1);
                else *(__half2 *)(s.kcache + sa.kv_off + (size_t)pos * E + rr) = __floats2half2_rn(o0, o1);
            }
        }
    }
    if (a.epi == EPI_LOGITS && lane < a.ntok && best) atomicMax(&sa.slots[lane].state->argmax_key, best);
}

// grid (n_head_local, B): head h of column t over column t's cache up to its position
__global__ void __launch_bounds__(256) attn_sessions_kernel(const float *__restrict__ q, const SessionSlot *slots, size_t kv_off, float *__restrict__ out,
                                                            int E, int n_ctx, float kq_scale, const __half *__restrict__ tab_exp) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ double red[34];
    __shared__ float redf[34];
    __shared__ __align__(16) __half qh[128];
    __shared__ float part[16 * 128];
    const SessionSlot &s = slots[blockIdx.y];
    attention_head(q, s.kcache + kv_off, s.vcache + kv_off, out, s.n_past, (int)blockIdx.x, (int)blockIdx.y, E, n_ctx, kq_scale, tab_exp, smem, red, redf, qh, part);
}

// before the step: the batch's DeviceState gets each column's token (its own id, or the context's on-device greedy id when id < 0,
// the decode_chain convention) so the embed_* kernels gather B rows; each context's arg-max key starts from zero
__global__ void prepare_sessions_kernel(const SessionSlot *slots, int B, DeviceState *batch) {
    const int t = threadIdx.x;
    if (t < B) {
        const SessionSlot &s = slots[t];
        batch->tokens[t] = s.id >= 0 ? s.id : s.state->tokens[0];
        s.state->argmax_key = 0ull;
    }
}

// prepare_sessions_kernel for a step of more than 8 columns (DeviceState::tokens holds 8): column t's token goes to ids[t], which
// embed_rows_kernel gathers; block >= B threads
__global__ void prepare_wide_kernel(const SessionSlot *slots, int B, int *ids) {
    const int t = threadIdx.x;
    if (t < B) {
        const SessionSlot &s = slots[t];
        ids[t] = s.id >= 0 ? s.id : s.state->tokens[0];
        s.state->argmax_key = 0ull;
    }
}

// after the step: every context's DeviceState is what its own decode step leaves (finalize_kernel): n_past + 1, the new arg-max
// as argmax_id and as the next token, the key reset; ids_out[t] = column t's arg-max; block >= B threads
__global__ void finalize_sessions_kernel(const SessionSlot *slots, int B, int *ids_out) {
    const int t = threadIdx.x;
    if (t < B) {
        DeviceState *st = slots[t].state;
        const int id = (int)(0xFFFFFFFFu - (unsigned)(st->argmax_key & 0xFFFFFFFFull));
        st->argmax_id = id; st->tokens[0] = id; st->argmax_key = 0ull;
        st->n_past = slots[t].n_past + 1;
        st->n_tok = 1;
        ids_out[t] = id;
    }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// batched prompt pass (minigpt4_b200_flush_batch; host side LlamaDevice::eval_rows_batch): the queued rows of several contexts
// concatenated, row t at its own context's position slots[t].n_past with that context's caches.  The per-op path appends through
// matvec_sessions_kernel's EPI_QKV one 8-row chunk at a time; the tensor-core path runs the fused qkv GEMM with EPI_PLAIN into
// qkv[rows][3 E] and this kernel applies pf::prefill_epilogue's RoPE and F16 append per row (the same expressions, so the same bits).
// grid (ceil(3 E / 2 / 256), rows), block 256: one thread per adjacent row pair (r0, r0 + 1) of row t
// ---------------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) qkv_rows_kernel(const float *__restrict__ qkv, const SessionSlot *slots, size_t kv_off, float *__restrict__ q_out,
                                                       const float2 *__restrict__ rope, int E, int half_dim) {
    const int t = blockIdx.y, p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= 3 * E / 2) return;
    const int r0 = 2 * p, part = r0 / E, rr = r0 % E;
    const float v0 = qkv[(size_t)t * 3 * E + r0], v1 = qkv[(size_t)t * 3 * E + r0 + 1];
    const SessionSlot &s = slots[t];
    const int pos = s.n_past;
    if (part == 2) {
        s.vcache[kv_off + (size_t)pos * E + rr] = __float2half_rn(v0);
        s.vcache[kv_off + (size_t)pos * E + rr + 1] = __float2half_rn(v1);
    } else {
        const float2 cs = rope[(size_t)pos * half_dim + (rr % (2 * half_dim)) / 2];
        const float o0 = v0 * cs.x - v1 * cs.y, o1 = v0 * cs.y + v1 * cs.x;
        if (part == 0) { q_out[(size_t)t * E + rr] = o0; q_out[(size_t)t * E + rr + 1] = o1; }
        else { s.kcache[kv_off + (size_t)pos * E + rr] = __float2half_rn(o0); s.kcache[kv_off + (size_t)pos * E + rr + 1] = __float2half_rn(o1); }
    }
}

struct RowList { int r[8]; };   // rows of a pass, by value

// the last row of each context that ends in this pass -> contiguous rows for the logits matvec; grid = n rows (<= 8: the contexts that
// end in one pass are finished 8 at a time)
__global__ void gather_rows_kernel(const float *__restrict__ x, const RowList rows, int E, float *__restrict__ out) {
    const float *src = x + (size_t)rows.r[blockIdx.x] * E;
    for (int i = threadIdx.x; i < E; i += blockDim.x) out[(size_t)blockIdx.x * E + i] = src[i];
}

}  // namespace k
}  // namespace mg4

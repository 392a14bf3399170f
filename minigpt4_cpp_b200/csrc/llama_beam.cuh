// llama_beam.cuh — sm_90a kernels of minigpt4_b200_beam_search (host side LlamaDevice::beam_search in llama.cu, DESIGN.md §4.13).
//
// A search runs n_beams (1..16) contexts of one group as slots: each slot holds at most one live beam, and its K / V rows n0 .. hold that
// beam's ids.  One step is four launches with no host round trip: beam_rank_kernel (one CTA per live slot: the row's log-sum-exp and its
// top 2 n_beams ids), beam_merge_kernel (one CTA: the order of all candidates, the walk that offers finished replies and takes the next
// live beams, the slot each new beam goes to), beam_reorder_kernel (the K / V rows a beam that changed slot needs) and the decode step of
// every slot.  The state of the search lives in one BeamState on the device.
#pragma once
#include "llama_sample.cuh"

namespace mg4 {
namespace beam {

constexpr int kMaxBeams = LlamaDevice::kMaxBeams;
constexpr int kCand = 2 * kMaxBeams;   // candidates walked per step (2 n_beams), and the most a beam contributes
constexpr int kRankThreads = 256;      // score_rows_kernel's block: the same strided sums and reduction tree
constexpr int kMergeThreads = 512;     // one thread per candidate of 16 beams
constexpr int kCopyThreads = 256;

struct Cand { float c, z; int beam, id, slot, pad; };   // c = S_beam + lp(id); beam: its index in the order the beams were taken
struct Hyp { float score, logprob; int len, stopped, seq, pad; };   // a finished reply: final score, S, ids, stop text ended it, offer order

struct BeamState {
    int t;                         // the step the next launch runs
    int done;                      // the search has ended (2: one beam's state saved); later launches only keep the columns moving
    int n_h, seq;                  // entries of H, offers made so far
    int beam[kMaxBeams];           // the beam index of each slot's live beam, -1: no live beam
    int valid[kMaxBeams];          // rows n0 .. n0 + valid - 1 of a slot hold the K / V of its ids[0 .. valid)
    float S[kMaxBeams];            // each slot's beam score (sum of log-probabilities, float32 left fold)
    int n_cand[kMaxBeams];
    Cand cand[kMaxBeams][kCand];   // each live slot's best candidates, in no order
    int n_sorted;
    Cand sorted[kCand];            // the first 2 n_beams candidates of the step, in order
    int n_moves;                   // K / V rows rows [r0, r1) (from n0) of slot src go to slot dst before the decode step
    int4 move[kMaxBeams];          // {src, dst, r0, r1}
    Hyp h[kMaxBeams];              // H
    smp::ReplyState tail[kMaxBeams];   // each slot's reply tail and the stop text (sample_until's stop rule)
};

struct BeamArgs {
    BeamState *st;
    const float *logits[kMaxBeams];   // each slot's logits
    DeviceState *state[kMaxBeams];    // tokens[0] takes the slot's next id, which the decode step feeds
    SessionSlot *slots;               // the batched step's column table (null: one beam, the context's own step)
    int *ids;                         // [kMaxBeams][stride] each slot's ids
    int *hids;                        // [kMaxBeams][stride] each entry of H's ids
    int stride, n_beams, n_vocab, max_steps, n0;
    float length_penalty;
    smp::TokenTable tab;
    int rank_only;                    // test seam: order the candidates into st->sorted and stop there
    float *snap;                      // one beam: the context's logits and DeviceState after the step that ended the search (null: none)
    DeviceState *snap_state;
};

// a before b in the search's order: c descending, then beam index ascending, then logit descending, then id ascending
__device__ __forceinline__ bool cand_before(const Cand &a, const Cand &b) {
    if (a.c != b.c) return a.c > b.c;
    if (a.beam != b.beam) return a.beam < b.beam;
    if (a.z != b.z) return a.z > b.z;
    return a.id < b.id;
}

// grid = n_beams slots, block kRankThreads.  A live slot's log-probabilities lp[v] = (float)(((double)z[v] - M) - log S), M = max z,
// S = sum exp((double)z - M), taken with score_rows_kernel's sweep and reduction (llama_score.cuh), so lp is the bits
// minigpt4_b200_score_tokens reports.  c = S_beam + lp[v] grows with z[v], so the beam's best candidates are its top 2 n_beams ids by
// (logit desc, id asc): the radix select of sample_kernel's top_k over the same keys.
__global__ void __launch_bounds__(kRankThreads) beam_rank_kernel(const __grid_constant__ BeamArgs a) {
    BeamState &st = *a.st;
    const int slot = blockIdx.x, tid = threadIdx.x;
    if (st.done || st.beam[slot] < 0) return;
    const float *__restrict__ z = a.logits[slot];
    __shared__ float sm[8];
    __shared__ double ss[8];
    __shared__ double sh_M, sh_logS;
    __shared__ unsigned hist[256];
    __shared__ unsigned long long sh_prefix;
    __shared__ int sh_need, sh_done, sh_n;
    // ---- M and S, as score_rows_kernel takes them
    float m = -INFINITY;
    double s = 0.0;
    for (int i = tid; i < a.n_vocab; i += blockDim.x) {
        const float v = z[i];
        if (v > m) { s = s * exp((double)m - (double)v) + 1.0; m = v; }
        else s += exp((double)v - (double)m);
    }
    const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float mo = __shfl_xor_sync(0xffffffffu, m, o);
        const double so = __shfl_xor_sync(0xffffffffu, s, o);
        const float mm = fmaxf(m, mo);
        s = (m == -INFINITY ? 0.0 : s * exp((double)m - (double)mm)) + (mo == -INFINITY ? 0.0 : so * exp((double)mo - (double)mm));
        m = mm;
    }
    if (lane == 0) { sm[warp] = m; ss[warp] = s; }
    __syncthreads();
    if (tid == 0) {
        const int nw = (int)(blockDim.x >> 5);
        float M = -INFINITY;
        for (int w = 0; w < nw; ++w) M = fmaxf(M, sm[w]);
        double S = 0.0;
        for (int w = 0; w < nw; ++w) if (sm[w] != -INFINITY) S += ss[w] * exp((double)sm[w] - (double)M);
        sh_M = (double)M; sh_logS = log(S);
        sh_prefix = 0ull;
    }
    // ---- the top k keys: radix select, 8 bits at a time from the top, to the threshold T with exactly k keys >= T (keys are distinct)
    const int k = min(2 * a.n_beams, a.n_vocab);
    if (tid == 0) sh_need = k;
    unsigned long long mask = 0ull;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int i = tid; i < 256; i += blockDim.x) hist[i] = 0u;
        __syncthreads();
        const unsigned long long pre = sh_prefix;
        for (int i = tid; i < a.n_vocab; i += blockDim.x) {
            const unsigned long long key = smp::desc_key(z[i], i);
            if ((key & mask) == pre) atomicAdd(&hist[(key >> shift) & 255], 1u);
        }
        __syncthreads();
        if (tid == 0) {
            int need = sh_need, d = 255; unsigned cum = 0;
            for (; d > 0; --d) { if (cum + hist[d] >= (unsigned)need) break; cum += hist[d]; }
            need -= (int)cum;
            sh_prefix = pre | ((unsigned long long)d << shift);
            sh_need = need;
            sh_done = hist[d] == (unsigned)need;
        }
        __syncthreads();
        mask |= 255ull << shift;
        if (sh_done) break;
    }
    if (tid == 0) sh_n = 0;
    __syncthreads();
    const unsigned long long T = sh_prefix;
    const float Sb = st.S[slot];
    const int b = st.beam[slot];
    for (int i = tid; i < a.n_vocab; i += blockDim.x) {
        const float v = z[i];
        if (smp::desc_key(v, i) >= T) {
            const float lp = (float)(((double)v - sh_M) - sh_logS);
            st.cand[slot][atomicAdd(&sh_n, 1)] = Cand{Sb + lp, v, b, i, slot, 0};
        }
    }
    __syncthreads();
    if (tid == 0) st.n_cand[slot] = sh_n;
}

// thread 0: offer a finished reply (the candidate (p, id) of step t, score c) to H; changed[e] records the entry's new ids
__device__ __forceinline__ void offer(const BeamArgs &a, BeamState &st, int t, float c, int p, int id, int stopped, int2 *src) {
    const float score = (float)((double)c / pow((double)(t + 1), (double)a.length_penalty));
    int e = st.n_h;
    if (e < a.n_beams) ++st.n_h;
    else {   // the worst entry: the lowest score, the latest offered among equal ones; it goes only for a strictly greater score
        e = 0;
        for (int j = 1; j < a.n_beams; ++j)
            if (st.h[j].score < st.h[e].score || (st.h[j].score == st.h[e].score && st.h[j].seq > st.h[e].seq)) e = j;
        if (!(score > st.h[e].score)) return;
    }
    st.h[e] = Hyp{score, c, t + 1, stopped, st.seq++, 0};
    src[e] = make_int2(p, id);
}

// one CTA of kMergeThreads.  Orders the live slots' candidates, walks the first 2 n_beams of them (an ending candidate of rank < n_beams
// is offered to H, a non-ending one becomes the next live beam until n_beams are taken), and places the new beams: a slot that is a
// parent keeps its best child, the other children go to slots that are no parent, in slot order, so no K / V copy reads a slot that this
// step writes.  Then each slot's ids, tail, S and next id (DeviceState::tokens[0]), the copies for beam_reorder_kernel, and the done flag.
__global__ void __launch_bounds__(kMergeThreads) beam_merge_kernel(const __grid_constant__ BeamArgs a) {
    BeamState &st = *a.st;
    const int tid = threadIdx.x, B = a.n_beams;
    __shared__ Cand all[kMaxBeams * kCand];
    __shared__ int n_all, sh_t, sh_done, nb, n_moves;
    __shared__ int par[kMaxBeams], nid[kMaxBeams], slot_of[kMaxBeams];
    __shared__ float nS[kMaxBeams];
    __shared__ smp::ReplyState ntail[kMaxBeams];
    __shared__ int2 hsrc[kMaxBeams];
    __shared__ int4 mv[kMaxBeams];
    if (tid == 0) { sh_t = st.t; sh_done = st.done; n_all = 0; }
    __syncthreads();
    const int t = sh_t;
    if (a.slots && tid < B) a.slots[tid].n_past = a.n0 + t;   // every column moves on, live or not
    if (sh_done) {
        // one beam: the decode step after the step that ended the search fed the last id of the reply (the greedy id, which is the
        // beam's); save what it left, as sample_until does, since the steps still issued run past it.  done 2: saved
        const bool save = a.snap && st.done == 1;
        if (save) for (int i = tid; i < a.n_vocab; i += blockDim.x) a.snap[i] = a.logits[0][i];
        __syncthreads();
        if (tid == 0) {
            if (save) { *a.snap_state = *a.state[0]; st.done = 2; }
            st.t = t + 1;
        }
        return;
    }
    // ---- the candidates of the live slots, then each one's rank in the order; the first 2 n_beams are the step's
    if (tid < B * kCand) {
        const int s = tid / kCand, j = tid % kCand;
        if (st.beam[s] >= 0 && j < st.n_cand[s]) all[atomicAdd(&n_all, 1)] = st.cand[s][j];
    }
    __syncthreads();
    const int n = n_all, keep = min(2 * B, n);
    if (tid < n) {
        const Cand x = all[tid];
        int r = 0;
        for (int j = 0; j < n; ++j) r += cand_before(all[j], x);
        if (r < keep) st.sorted[r] = x;
    }
    __syncthreads();
    if (a.rank_only) {
        if (tid == 0) st.n_sorted = keep;
        return;
    }
    // ---- the walk
    if (tid == 0) {
        for (int e = 0; e < B; ++e) hsrc[e] = make_int2(-1, -1);
        int taken = 0;
        for (int r = 0; r < keep; ++r) {
            const Cand x = st.sorted[r];
            smp::ReplyState rs = st.tail[x.slot];
            if (smp::reply_take(rs, a.tab, x.id)) {
                if (r < B) offer(a, st, t, x.c, x.slot, x.id, 1, hsrc);
            } else if (taken < B) {
                par[taken] = x.slot; nid[taken] = x.id; nS[taken] = x.c; ntail[taken] = rs;
                ++taken;
            }
        }
        int done = st.n_h == B || taken == 0;
        if (!done && t == a.max_steps - 1) {   // the search ran through: every live beam is offered, in beam order
            for (int j = 0; j < taken; ++j) offer(a, st, t, nS[j], par[j], nid[j], 0, hsrc);
            done = 1;
        }
        nb = done ? 0 : taken;
        sh_done = done;
        // ---- slots: a parent keeps its best (first taken) child; the other children take the slots of no parent, in order
        bool parent[kMaxBeams] = {};
        int m = 0;
        for (int j = 0; j < nb; ++j) {
            if (!parent[par[j]]) { parent[par[j]] = true; slot_of[j] = par[j]; }
            else slot_of[j] = -1;
        }
        int free_s = 0;
        for (int j = 0; j < nb; ++j) {
            if (slot_of[j] >= 0) continue;
            while (parent[free_s]) ++free_s;
            slot_of[j] = free_s++;
            mv[m++] = make_int4(par[j], slot_of[j], min(st.valid[slot_of[j]], t), t);   // r0: lowered below to the first differing id
        }
        n_moves = m;
    }
    __syncthreads();
    // ---- the ids of the entries of H that changed, from their parents (no parent's ids [0, t) change in this step)
    for (int e = 0; e < B; ++e) {
        const int2 h = hsrc[e];
        if (h.x < 0) continue;
        for (int j = tid; j < t; j += blockDim.x) a.hids[(size_t)e * a.stride + j] = a.ids[(size_t)h.x * a.stride + j];
        if (tid == 0) a.hids[(size_t)e * a.stride + t] = h.y;
    }
    // ---- each move copies only from the first id where the destination's ids differ from its new parent's
    for (int q = 0; q < n_moves; ++q) {
        const int4 v = mv[q];
        const int *ps = a.ids + (size_t)v.x * a.stride, *pd = a.ids + (size_t)v.y * a.stride;
        for (int j = tid; j < v.z; j += blockDim.x)
            if (ps[j] != pd[j]) atomicMin(&mv[q].z, j);
    }
    __syncthreads();
    for (int q = 0; q < n_moves; ++q) {
        const int4 v = mv[q];
        for (int j = v.z + tid; j < t; j += blockDim.x) a.ids[(size_t)v.y * a.stride + j] = a.ids[(size_t)v.x * a.stride + j];
    }
    __syncthreads();
    if (tid < B) {
        st.beam[tid] = -1;
        st.valid[tid] = 0;
    }
    __syncthreads();
    if (tid < nb) {
        const int s = slot_of[tid];
        st.beam[s] = tid;
        st.valid[s] = t + 1;
        st.S[s] = nS[tid];
        st.tail[s] = ntail[tid];
        a.ids[(size_t)s * a.stride + t] = nid[tid];
        a.state[s]->tokens[0] = nid[tid];
    }
    if (tid == 0) {
        st.n_moves = n_moves;
        for (int q = 0; q < n_moves; ++q) st.move[q] = make_int4(mv[q].x, mv[q].y, mv[q].z, mv[q].w);
        st.t = t + 1;
        st.done = sh_done;
    }
}

struct ReorderArgs {
    const BeamState *st;
    uint4 *k[kMaxBeams], *v[kMaxBeams];   // each slot's caches (layer 0)
    long long plane, row;                 // 16-byte chunks of one layer's cache and of one row
    int n_layer, n0;
};

// grid (x, 2 n_layer), block kCopyThreads: plane y (K planes, then V) of every move of the step, rows n0 + r0 .. n0 + r1 - 1 of the source
// slot to the same rows of the destination, the chunking of copy_state_kernel (llama_state.cuh)
__global__ void __launch_bounds__(kCopyThreads) beam_reorder_kernel(const __grid_constant__ ReorderArgs a) {
    const BeamState &st = *a.st;
    const int y = (int)blockIdx.y, n_moves = st.n_moves;
    const bool is_v = y >= a.n_layer;
    const long long base = (long long)(is_v ? y - a.n_layer : y) * a.plane + (long long)a.n0 * a.row;
    const long long stride = (long long)gridDim.x * kCopyThreads, t0 = (long long)blockIdx.x * kCopyThreads + threadIdx.x;
    for (int q = 0; q < n_moves; ++q) {
        const int4 m = st.move[q];
        const uint4 *__restrict__ src = (is_v ? a.v[m.x] : a.k[m.x]) + base;
        uint4 *__restrict__ dst = (is_v ? a.v[m.y] : a.k[m.y]) + base;
        for (long long i = m.z * a.row + t0; i < m.w * a.row; i += stride) dst[i] = src[i];
    }
}

}  // namespace beam
}  // namespace mg4

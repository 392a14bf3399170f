// llama_mega6.cuh — the persistent decode megakernel, generation 6: ONE launch per generated token.
//
// A 7B Q4_1 token streams 4.13 GB of weights through ~160 dependent, short matvecs.  Weights do not depend on activations, so the
// weight stream is kept running ACROSS op boundaries:
//   * grid = one CTA per SM (cooperative launch), 16 warps; warps 0..W-1 (W <= 15) are STREAM warps, every warp of 0..14 also takes part in
//     activation staging, warps 0-7 run the attention op
//   * SELF-REFILLED PER-WARP STREAMS.  Every stream warp owns TWO shared-memory slots and a private cursor over the token's op program.  It
//     walks "its" row pairs of every weight matrix (pairs lo + w, lo + w + W, ... of the CTA's contiguous share) and keeps the next two
//     slot-loads in flight with cp.async.bulk (1-D TMA) + mbarrier complete_tx; right after it has read a slot it re-arms the slot ITSELF.
//     No producer warp and no "empty" barriers: a single producer thread is issue-bound on 5 KB copies (try_wait + expect_tx + issue per
//     copy), which was the limit of generations 2-5; 15 independent issuers per SM are not (tools/ubench_stream.cu measures the primitive
//     with the full Q4_1 dot product in the loop).  The cursor runs straight through grid barriers,
//     staging and the attention op: 2 x W slots (207 KB per SM) are always requested ahead of the consumers.
//   * REGISTER-RESIDENT ACTIVATIONS for n_embd-wide inputs (qkv, wo, gate/up, output): lane l keeps the Q8 blocks l, l+32, ... of the staged
//     vector in registers, so a row pair costs shared-memory reads of the WEIGHTS only (TMA write + one read = 2 x the HBM rate of smem traffic)
//   * per op: [grid barrier -> stage activations (RMSNorm + Q8 quantise) -> per owned row pair: wait slot, dp4a dots, re-arm slot,
//     warp-shuffle reductions, fused epilogue].  Ops exchange x / q / att / act through L2 (ld.global.cg); a grid barrier (atomic counter)
//     separates dependent ops.
//   * NO deeper prefetch than the slots.  A look-ahead warp that asked L2 for the stream beyond the slots while the stream warps were stalled
//     (cp.async.bulk.prefetch.L2, or cp.async into a scratch line) was tried and removed (no gain at 192 KB per CTA, a loss at 384 KB) - the barrier / staging / attention phases between two matvecs are chains of L2 round trips, and every
//     byte of weight traffic in flight during them lengthens those round trips.
// Reduction orders are the canonical ones of llama_kernels.cuh / oracle.cpp: logits are bit-identical to the per-op kernels and the CPU oracle.
#pragma once
#include "llama_kernels.cuh"
#include "tp.h"

namespace mg4 {
namespace mk6 {
using namespace k;

enum OpKind : int { OP_EMBED = 0, OP_QKV = 1, OP_ATTN = 2, OP_WO = 3, OP_GATEUP = 4, OP_DOWN = 5, OP_OUTPUT = 6, OP_FINAL = 7, OP_REDUCE = 8 };

struct Op6 {                 // 32 bytes, lives in the kernel's parameter (constant) space
    unsigned char kind, parts;     // a unit = 2 * row_bytes contiguous bytes, brought by `parts` slot-loads (1: the pair in one slot; 2: one row per slot)
    unsigned short layer;          // (OP_REDUCE: exchange buffer index)
    int cols, n_su, row_bytes;     // n_su = row pairs (units) of the matrix over the whole grid
    const unsigned char *w;        // row-packed Q4 weights (null for non-matvec ops)
    const float *norm_w;
};
static_assert(sizeof(Op6) == 32, "Op6");
constexpr int kMaxOps = 7 * 80 + 3;   // up to 80 layers, tensor-parallel program (7 ops per layer): 18 KB of the 32 764-byte parameter space

struct Params6 {
    int n_ops, W, slot_bytes, act_bytes;   // shared memory: [2 W slots][act: staged Q8 activations / attention scratch][2 W mbarriers]
    int n_su_kind[8];                      // row pairs per op kind (all layers have the same shapes): the CTA's share of each is computed once
    int E, FF, n_head, n_ctx, n_vocab, flags;   // flags bit 0: pull the head's K/V history into L2 while the qkv weights are consumed
    // tensor parallel (world > 1): this rank holds n_head heads (El = 128 n_head columns of q / att / the KV cache), FF / world columns of the
    // feed-forward; wo / down write PARTIAL sums into the rank's exchange buffer and an OP_REDUCE op sums the partials of all ranks straight out
    // of peer memory (NVLink) into x.  The compute and the collective are ONE kernel.
    int El;            // local q / att / KV row width (== E on one GPU)
    TPPeers tp;        // peer mappings of the exchange buffers (tp.h); tp.world <= 1: single GPU
    unsigned *tp_seq;  // all-reduces completed so far by this rank (shared with the per-op path's all-reduce kernel)

    float kq_scale;
    int E_pow2;        // n_embd is a power of two: sum / n_embd == sum * (1 / n_embd) exactly
    double inv_E;
    float *x, *q, *att, *act, *logits;
    __half *kcache, *vcache;
    const float2 *rope; const __half *tab_exp, *tab_silu;
    const unsigned char *tok; int tok_type; size_t tok_row_bytes;
    DeviceState *state; unsigned *barrier;
    long long *trace;  // optional [2 CTAs][n_ops][16]: clock64 at op start, barrier passed, activations staged, op done; then (warp 0) cycles
                       // waiting for slot fills, cycles in the dot products, units processed, cycles in reductions + epilogue; [8..11] sub-stamps
                       // (staging: sum of squares known, quantised; attention: scores, soft-max sum, probabilities, P.V done)
    Op6 ops[kMaxOps];
};
static_assert(sizeof(Params6) <= 32764, "kernel parameter space");
constexpr int kReduceCtas = 16;   // CTAs that pull the peers' partial sums in an OP_REDUCE op (n_embd / 16 elements each)

constexpr int kConsumerWarps = 15, kConsumerThreads = 480, kThreads = 512;
// named barriers: 1 = the 256 threads of warps 0-7 (activation staging, attention); 2 = all 480 threads of warps 0-14
__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 2, 480;" ::: "memory"); }

__device__ __forceinline__ uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mb_init(uint64_t *bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count)); }
__device__ __forceinline__ void mb_expect_tx(uint64_t *bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mb_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "MB_WAIT:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra MB_DONE;\n\t"
        "bra MB_WAIT;\n\t"
        "MB_DONE:\n\t}" ::"r"(smem_addr(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_addr(dst)), "l"(src), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ void prefetch_l2_keep(const void *p) { asm volatile("prefetch.global.L2::evict_last [%0];" ::"l"(p)); }
// A real (discarded) load, unlike a prefetch hint, cannot be dropped on a TLB miss: used to pull data that the weight stream has pushed out of
// L2 (and its page out of the TLB) back in BEFORE it is needed on the critical path.
__device__ __forceinline__ void touch(const void *p) { unsigned v; asm volatile("ld.global.cg.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); }
// The attention op of this layer will read K/V rows 0..pos-1 of head h (256 B per key and tensor, written by earlier tokens) and the negative
// half of the exp table (62 KB); the weight stream has pushed all of it out of L2 - and the pages out of the TLB - since the previous token.
// One op early, every thread of the head's CTA pulls its share of those lines back with real loads (a prefetch hint is dropped on a TLB
// miss), so that the attention's critical path sees L2 hits and warm translations.
__device__ __forceinline__ void touch_kv_head(const __half *kc, const __half *vc, const __half *tab_exp, int pos, int h, int E) {
    for (int i = (int)threadIdx.x; i < 2 * pos; i += kConsumerThreads) {  // (key, 128-byte half of the 256-byte head row)
        const size_t off = (size_t)(i >> 1) * E + h * 128 + (i & 1) * 64;
        touch(kc + off); touch(vc + off);
    }
    for (int i = (int)threadIdx.x; i < 496; i += kConsumerThreads) touch(tab_exp + 0x8000 + i * 64);  // fp16 inputs -0 .. -inf: entries 0x8000 .. 0xfc00
}

// first unit (row pair) of CTA `cta`: units are split evenly over the grid (n_su * G < 2^31: host-checked)
__device__ __forceinline__ int unit_begin(int cta, int n_su, int G) { return (int)((unsigned)cta * (unsigned)n_su / (unsigned)G); }

// all threads of warps 0-14 of all CTAs; `target` = number of arrivals that complete this barrier (monotonic counter, zeroed per launch)
__device__ __forceinline__ void grid_barrier(unsigned *counter, unsigned target) {
    consumer_sync();  // all warps of this CTA have issued their global writes (CTA-scope ordering)
    if (threadIdx.x == 0) {
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");   // cumulative release of the CTA's writes
        unsigned v;
        do { asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory"); } while (v < target);
    }
    consumer_sync();
}

__device__ __forceinline__ int dp4a_us(unsigned a, int b, int c) {  // unsigned bytes x signed bytes
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
// sum_j q_j a_j of one 32-weight Q4 block (16 B of nibbles, q in 0..15) with its Q8 block (two 16-byte planes).  The high nibbles stay in
// place (w & 0xF0F0F0F0 = 16 q): their dp4a sum is an exact multiple of 16, so one shift replaces four - and the two 4-deep dp4a chains are
// independent.  Integer arithmetic: same value as the nibble-by-nibble form of k::dot2_q4.
__device__ __forceinline__ int q4_block_idot(const uint4 q, const int4 lo, const int4 hi) {
    int sl = dp4a_us(q.x & 0x0F0F0F0Fu, lo.x, 0), sh = dp4a_us(q.x & 0xF0F0F0F0u, hi.x, 0);
    sl = dp4a_us(q.y & 0x0F0F0F0Fu, lo.y, sl); sh = dp4a_us(q.y & 0xF0F0F0F0u, hi.y, sh);
    sl = dp4a_us(q.z & 0x0F0F0F0Fu, lo.z, sl); sh = dp4a_us(q.z & 0xF0F0F0F0u, hi.z, sh);
    sl = dp4a_us(q.w & 0x0F0F0F0Fu, lo.w, sl); sh = dp4a_us(q.w & 0xF0F0F0F0u, hi.w, sh);
    return sl + (sh >> 4);
}

// ---- staged activation layout in shared memory (Q8_0 / Q8_1): [lo plane cols/2][64 B pad][hi plane cols/2][d: nb floats][s: nb floats].
// The pad puts the two 16-byte planes of a block 16 banks apart, so the staging stores of a warp (lanes 0-3 -> lo, 4-7 -> hi) do not collide.
__host__ __device__ inline int act6_hi(int cols) { return cols / 2 + 64; }
__host__ __device__ inline int act6_d(int cols) { return cols + 64; }
__host__ __device__ inline size_t act6_bytes(int cols) { return (size_t)cols + 64 + (size_t)cols / 32 * 8; }

constexpr int kNormItems = 5;   // RMS-normed inputs (warps 0-7): n_embd <= 256 threads x 4 floats x 5 = 5120
constexpr int kPlainItems = 8;  // un-normed inputs (all 15 warps): cols <= 480 x 4 x 8 = 15360
// Quantise K float4s per thread (float4 k sits at elements i[k] .. i[k]+3; 8 consecutive lanes cover one 32-element block; `valid` is shared by
// the 8 lanes of a block and all lanes run the shuffles).  A warp issues in order and shuffles cannot be reordered by the compiler, so the
// reduction stages are written STAGE-MAJOR: the K independent chains advance together and their shuffle latencies overlap (item-major order
// costs K x 6 dependent round trips).  Quantisation is order-free (max, integer sums): identical bytes to k::stage_act.
template <int ACT, int K>
__device__ __forceinline__ void quant_items(const float4 (&a)[K], const int (&i)[K], const bool (&valid)[K], int cols, unsigned char *sm) {
    float *d = (float *)(sm + act6_d(cols)); float *s = d + cols / 32;
    const int j8 = threadIdx.x & 7;
    float amax[K];
#pragma unroll
    for (int k = 0; k < K; ++k) amax[k] = fmaxf(fmaxf(fabsf(a[k].x), fabsf(a[k].y)), fmaxf(fabsf(a[k].z), fabsf(a[k].w)));
#pragma unroll
    for (int o = 4; o > 0; o >>= 1)
#pragma unroll
        for (int k = 0; k < K; ++k) amax[k] = fmaxf(amax[k], __shfl_xor_sync(0xffffffffu, amax[k], o));
    int q0[K], q1[K], q2[K], q3[K], sum[K]; float dd[K];
#pragma unroll
    for (int k = 0; k < K; ++k) {
        dd[k] = amax[k] / 127.f;
        const float id = amax[k] != 0.0f ? 127.f / amax[k] : 0.0f;
        q0[k] = __float2int_rn(a[k].x * id); q1[k] = __float2int_rn(a[k].y * id); q2[k] = __float2int_rn(a[k].z * id); q3[k] = __float2int_rn(a[k].w * id);
        sum[k] = (q0[k] + q1[k]) + (q2[k] + q3[k]);
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1)
#pragma unroll
        for (int k = 0; k < K; ++k) sum[k] += __shfl_xor_sync(0xffffffffu, sum[k], o);
#pragma unroll
    for (int k = 0; k < K; ++k) {
        if (valid[k]) {
            const int b = i[k] >> 5;
            *(unsigned *)(sm + (j8 < 4 ? 0 : act6_hi(cols)) + b * 16 + (j8 & 3) * 4) =
                (unsigned)(q0[k] & 0xff) | ((unsigned)(q1[k] & 0xff) << 8) | ((unsigned)(q2[k] & 0xff) << 16) | ((unsigned)(q3[k] & 0xff) << 24);
            if (j8 == 0) {
                if (ACT == ACT_Q8_0) { d[b] = __half2float(__float2half_rn(dd[k])); s[b] = (float)sum[k]; }  // integer block sum (exact): Q4_0's "-8" term
                else { d[b] = dd[k]; s[b] = dd[k] * (float)sum[k]; }
            }
        }
    }
}
// un-normed inputs (wo <- att, down <- act), all 480 threads of warps 0-14: thread t owns the float4s 480 k + t.  The F32 vector is read straight
// from L2 into registers (ld.global.cg: other CTAs wrote it earlier in this launch), all loads of a thread in flight at once.
template <int ACT, int K>
__device__ __forceinline__ void stage_plain_k(const float *__restrict__ x, int cols, unsigned char *sm) {
    const int tid = threadIdx.x;  // tid < 480
    float4 xv[K]; int idx[K]; bool valid[K];
#pragma unroll
    for (int k = 0; k < K; ++k) {
        idx[k] = 4 * (tid + kConsumerThreads * k); valid[k] = idx[k] < cols;
        xv[k] = valid[k] ? __ldcg((const float4 *)(x + idx[k])) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    quant_items<ACT, K>(xv, idx, valid, cols, sm);
}
template <int ACT>
__device__ __forceinline__ void stage_plain(const float *__restrict__ x, int cols, unsigned char *sm) {
    if (cols <= 4 * kConsumerThreads * 3) stage_plain_k<ACT, 3>(x, cols, sm);        // n_embd-wide (wo): <= 5760
    else if (cols <= 4 * kConsumerThreads * 6) stage_plain_k<ACT, 6>(x, cols, sm);   // n_ff <= 11520 (7B: 11008)
    else stage_plain_k<ACT, kPlainItems>(x, cols, sm);
}
// RMS-normed inputs (n_embd wide), warps 0-7.  Thread t owns the float4s at elements 1024 it + 4 t: its RMS partials are the canonical
// partials t (even it) and t + 256 (odd it) of oracle.cpp op_rms_norm_mul, same as k::stage_act; every warp then folds the 16 warp sums the
// way warp 0 of k::stage_act does (one CTA sync instead of two).  The two warp-level butterflies are interleaved (see quant_items).
template <int ACT, int K>
__device__ __forceinline__ void stage_norm_k(const float *__restrict__ x, const float *__restrict__ nw, int cols, unsigned char *sm, double *red, bool pow2, double inv_cols, long long *tr) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;  // tid < 256
    float4 xv[K], w[K]; int idx[K]; bool valid[K];
#pragma unroll
    for (int it = 0; it < K; ++it) {
        idx[it] = 1024 * it + 4 * tid; valid[it] = idx[it] < cols;
        xv[it] = valid[it] ? __ldcg((const float4 *)(x + idx[it])) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int it = 0; it < K; ++it) w[it] = valid[it] ? __ldg((const float4 *)(nw + idx[it])) : make_float4(0.f, 0.f, 0.f, 0.f);   // static: pulled into L2 before the grid barrier
    double ssa = 0.0, ssb = 0.0;
#pragma unroll
    for (int it = 0; it < K; ++it) {
        if (valid[it]) {
            const float4 a = xv[it];
            if (it & 1) { ssb += (double)(a.x * a.x); ssb += (double)(a.y * a.y); ssb += (double)(a.z * a.z); ssb += (double)(a.w * a.w); }
            else        { ssa += (double)(a.x * a.x); ssa += (double)(a.y * a.y); ssa += (double)(a.z * a.z); ssa += (double)(a.w * a.w); }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const double ta = __shfl_xor_sync(0xffffffffu, ssa, o), tb = __shfl_xor_sync(0xffffffffu, ssb, o); ssa += ta; ssb += tb; }   // = warp_sum(ssa), warp_sum(ssb)
    if (lane == 0) { red[warp] = ssa; red[warp + 8] = ssb; }
    cta_sync<true>();
    double t = lane < 16 ? red[lane] : 0.0;
    t = warp_sum(t);
    const float mean = pow2 ? (float)(t * inv_cols) : (float)(t / (double)cols);   // (a power-of-two divisor: the product is the same double)
    const float scale = 1.0f / sqrtf(mean + 1e-6f);
    if (tr) tr[8] = clock64();
    float4 v[K];
#pragma unroll
    for (int it = 0; it < K; ++it) v[it] = make_float4((xv[it].x * scale) * w[it].x, (xv[it].y * scale) * w[it].y, (xv[it].z * scale) * w[it].z, (xv[it].w * scale) * w[it].w);
    quant_items<ACT, K>(v, idx, valid, cols, sm);
}
template <int ACT>
__device__ __forceinline__ void stage_norm(const float *__restrict__ x, const float *__restrict__ nw, int cols, unsigned char *sm, double *red, bool pow2, double inv_cols, long long *tr) {
    if (cols <= 4096) stage_norm_k<ACT, 4>(x, nw, cols, sm, red, pow2, inv_cols, tr);
    else stage_norm_k<ACT, kNormItems>(x, nw, cols, sm, red, pow2, inv_cols, tr);
}

// ---- dot products: per-lane partial sums of two rows (lane l: blocks l, l+32, ... increasing = the order of k::dot2_q4); the caller reduces ----
struct Acc4 { float d0, m0, d1, m1; };
// shared-memory activations (n_ff-wide inputs, and every input of models whose n_embd is not 1024 * NBL).  Q4_0's "-8" is applied as
// sum (q-8) a = sum q a - 8 sum a  with the integer activation sum the staging pass leaves in the `s` plane.
template <bool Q41>
__device__ __forceinline__ Acc4 dot2_q4_smem(const unsigned char *row0, const unsigned char *row1, int nb, int cols, const unsigned char *act, int lane) {
    const uint4 *qs0 = (const uint4 *)row0, *qs1 = (const uint4 *)row1;
    const unsigned char *sc0 = row0 + (size_t)nb * 16, *sc1 = row1 + (size_t)nb * 16;
    const int4 *alo = (const int4 *)act, *ahi = (const int4 *)(act + act6_hi(cols));
    const float *ad = (const float *)(act + act6_d(cols)), *as = ad + nb;
    Acc4 r{0.f, 0.f, 0.f, 0.f};
#pragma unroll 2
    for (int b = lane; b < nb; b += 32) {
        const uint4 q0 = qs0[b], q1 = qs1[b];
        const int4 la = alo[b], ha = ahi[b];
        const float adv = ad[b], asv = as[b];
        int s0 = q4_block_idot(q0, la, ha), s1 = q4_block_idot(q1, la, ha);
        if (Q41) {
            const float2 f0 = __half22float2(((const __half2 *)sc0)[b]), f1 = __half22float2(((const __half2 *)sc1)[b]);
            r.d0 = fmaf(f0.x * adv, (float)s0, r.d0); r.m0 = fmaf(f0.y, asv, r.m0);
            r.d1 = fmaf(f1.x * adv, (float)s1, r.d1); r.m1 = fmaf(f1.y, asv, r.m1);
        } else {
            const float d0 = __half2float(((const __half *)sc0)[b]), d1 = __half2float(((const __half *)sc1)[b]);
            const int i8 = 8 * (int)asv;
            s0 -= i8; s1 -= i8;
            r.d0 += ((float)s0 * d0) * adv; r.d1 += ((float)s1 * d1) * adv;
        }
    }
    return r;
}
// register-resident activations: lane l holds blocks l + 32 i (i < NBL) of the staged vector; same per-lane order and arithmetic
template <int NBL> struct ActRegs { int4 lo[NBL], hi[NBL]; float d[NBL], s[NBL]; };
template <int NBL>
__device__ __forceinline__ void load_act_regs(const unsigned char *act, int cols, int lane, ActRegs<NBL> &r) {
    const int4 *alo = (const int4 *)act, *ahi = (const int4 *)(act + act6_hi(cols));
    const float *ad = (const float *)(act + act6_d(cols)), *as = ad + (cols >> 5);
#pragma unroll
    for (int i = 0; i < NBL; ++i) { const int b = lane + 32 * i; r.lo[i] = alo[b]; r.hi[i] = ahi[b]; r.d[i] = ad[b]; r.s[i] = as[b]; }
}
template <bool Q41, int NBL>
__device__ __forceinline__ Acc4 dot2_q4_reg(const unsigned char *row0, const unsigned char *row1, const ActRegs<NBL> &a, int lane) {
    constexpr int nb = 32 * NBL;
    const uint4 *qs0 = (const uint4 *)row0, *qs1 = (const uint4 *)row1;
    const unsigned char *sc0 = row0 + (size_t)nb * 16, *sc1 = row1 + (size_t)nb * 16;
    Acc4 r{0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < NBL; ++i) {
        const int b = lane + 32 * i;
        const uint4 q0 = qs0[b], q1 = qs1[b];
        int s0 = q4_block_idot(q0, a.lo[i], a.hi[i]), s1 = q4_block_idot(q1, a.lo[i], a.hi[i]);
        if (Q41) {
            const float2 f0 = __half22float2(((const __half2 *)sc0)[b]), f1 = __half22float2(((const __half2 *)sc1)[b]);
            r.d0 = fmaf(f0.x * a.d[i], (float)s0, r.d0); r.m0 = fmaf(f0.y, a.s[i], r.m0);
            r.d1 = fmaf(f1.x * a.d[i], (float)s1, r.d1); r.m1 = fmaf(f1.y, a.s[i], r.m1);
        } else {
            const float d0 = __half2float(((const __half *)sc0)[b]), d1 = __half2float(((const __half *)sc1)[b]);
            const int i8 = 8 * (int)a.s[i];
            s0 -= i8; s1 -= i8;
            r.d0 += ((float)s0 * d0) * a.d[i]; r.d1 += ((float)s1 * d1) * a.d[i];
        }
    }
    return r;
}

// ---- K-quant weights (Q5_K): Q8_K activations -------------------------------------------------------------------------------------------
// Staged layout = k::stage_act: [int8 q: cols][float d: cols / 256][int16 bsums: cols / 16].  Per 256-element super-block (ggml
// quantize_row_q8_K): max = the element of largest |x| (first index on ties), iscale = -128 / max, q = min(127, rint(iscale x)), d = 1 / iscale,
// bsums = sums of 16 q.  One warp per super-block (lane l: elements 8 l .. 8 l + 7), all 15 warps; RMS-normed inputs: warps 0-7 first form the
// canonical sum of squares (stage_norm_k), every warp folds the 16 warp sums.  Identical bytes to k::stage_act.
constexpr int kQ8kRounds = 4;   // super-blocks per warp: cols <= 15 x 4 x 256 = 15360
__device__ __forceinline__ void stage_q8k(const float *__restrict__ x, const float *__restrict__ nw, int cols, unsigned char *sm, double *red, bool pow2, double inv_cols, long long *tr) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nsb = cols >> 8;  // tid < 480
    constexpr int kNormRounds = 2;   // RMS-normed inputs are n_embd wide: <= 15 x 2 x 256 = 7680
    float4 xa[kQ8kRounds], xb[kQ8kRounds], wa[kNormRounds], wb[kNormRounds];
#pragma unroll
    for (int k = 0; k < kQ8kRounds; ++k) {   // this warp's super-blocks warp, warp + 15, ...: all loads in flight at once
        const int sb = warp + kConsumerWarps * k;
        const bool on = sb < nsb;
        const int i = sb * 256 + lane * 8;
        xa[k] = on ? __ldcg((const float4 *)(x + i)) : make_float4(0.f, 0.f, 0.f, 0.f);
        xb[k] = on ? __ldcg((const float4 *)(x + i + 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
        if (k < kNormRounds) { if (nw) { wa[k] = on ? __ldg((const float4 *)(nw + i)) : make_float4(0.f, 0.f, 0.f, 0.f); wb[k] = on ? __ldg((const float4 *)(nw + i + 4)) : make_float4(0.f, 0.f, 0.f, 0.f); } }
    }
    float scale = 1.0f;
    if (nw) {
        if (warp < 8) {
            double ssa = 0.0, ssb = 0.0;
#pragma unroll
            for (int it = 0; it < kNormItems; ++it) {
                const int i = 1024 * it + 4 * tid;
                if (i < cols) {
                    const float4 a = __ldcg((const float4 *)(x + i));
                    if (it & 1) { ssb += (double)(a.x * a.x); ssb += (double)(a.y * a.y); ssb += (double)(a.z * a.z); ssb += (double)(a.w * a.w); }
                    else        { ssa += (double)(a.x * a.x); ssa += (double)(a.y * a.y); ssa += (double)(a.z * a.z); ssa += (double)(a.w * a.w); }
                }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) { const double ta = __shfl_xor_sync(0xffffffffu, ssa, o), tb = __shfl_xor_sync(0xffffffffu, ssb, o); ssa += ta; ssb += tb; }
            if (lane == 0) { red[warp] = ssa; red[warp + 8] = ssb; }
        }
        consumer_sync();
        double t = lane < 16 ? red[lane] : 0.0;
        t = warp_sum(t);
        const float mean = pow2 ? (float)(t * inv_cols) : (float)(t / (double)cols);
        scale = 1.0f / sqrtf(mean + 1e-6f);
    }
    if (tr) tr[8] = clock64();
    int8_t *qs = (int8_t *)sm; float *d = (float *)(sm + cols); int16_t *bs = (int16_t *)(sm + cols + nsb * 4);
#pragma unroll
    for (int k = 0; k < kQ8kRounds; ++k) {
        const int sb = warp + kConsumerWarps * k;
        if (sb < nsb) {   // (warp-uniform)
            float v[8] = {xa[k].x, xa[k].y, xa[k].z, xa[k].w, xb[k].x, xb[k].y, xb[k].z, xb[k].w};
            if (k < kNormRounds) {
                if (nw) {
                    const float w8[8] = {wa[k < kNormRounds ? k : 0].x, wa[k < kNormRounds ? k : 0].y, wa[k < kNormRounds ? k : 0].z, wa[k < kNormRounds ? k : 0].w,
                                         wb[k < kNormRounds ? k : 0].x, wb[k < kNormRounds ? k : 0].y, wb[k < kNormRounds ? k : 0].z, wb[k < kNormRounds ? k : 0].w};
#pragma unroll
                    for (int j = 0; j < 8; ++j) v[j] = (v[j] * scale) * w8[j];
                }
            }
            float amax = 0.f, mx = 0.f; int mi = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) { const float a = fabsf(v[j]); if (a > amax) { amax = a; mx = v[j]; mi = lane * 8 + j; } }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {  // first-index arg-max of |x| (strict > in the sequential reference)
                const float oa = __shfl_xor_sync(0xffffffffu, amax, o), om = __shfl_xor_sync(0xffffffffu, mx, o);
                const int oi = __shfl_xor_sync(0xffffffffu, mi, o);
                if (oa > amax || (oa == amax && oi < mi)) { amax = oa; mx = om; mi = oi; }
            }
            int q[8]; int sum = 0;
            const float iscale = amax != 0.f ? -128.f / mx : 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) { int t = __float2int_rn(iscale * v[j]); t = t < 127 ? t : 127; q[j] = t; sum += t; }
            if (amax == 0.f) sum = 0;
            const unsigned w0 = (q[0] & 0xff) | ((q[1] & 0xff) << 8) | ((q[2] & 0xff) << 16) | ((unsigned)(q[3] & 0xff) << 24);
            const unsigned w1 = (q[4] & 0xff) | ((q[5] & 0xff) << 8) | ((q[6] & 0xff) << 16) | ((unsigned)(q[7] & 0xff) << 24);
            *(uint2 *)(qs + sb * 256 + lane * 8) = make_uint2(w0, w1);
            const int s2 = sum + __shfl_xor_sync(0xffffffffu, sum, 1);
            if ((lane & 1) == 0) bs[sb * 16 + (lane >> 1)] = (int16_t)s2;
            if (lane == 0) d[sb] = amax != 0.f ? 1.0f / iscale : 0.f;
        }
    }
}
// Two Q5_K rows in shared memory (row = [nsb x 128 B qs][nsb x 32 B qh][nsb x 16 B {scales[12], d, dmin}]) against the staged Q8_K vector: the
// lane mapping (8 lanes per super-block, 4 super-blocks per pass), integer arithmetic and float order of k::dot2_q5k.  Result = sum d - sum m.
__device__ __forceinline__ Acc4 dot2_q5k_smem(const unsigned char *row0, const unsigned char *row1, int nsb, int cols, const unsigned char *act, int lane) {
    const int sub = lane >> 3, j = (lane & 7) >> 1, hf = lane & 1;
    const float *ad = (const float *)(act + cols);
    const int16_t *abs_ = (const int16_t *)(act + cols + nsb * 4);
    Acc4 r{0.f, 0.f, 0.f, 0.f};
    for (int sb0 = 0; sb0 < nsb; sb0 += 4) {
        const int sb = sb0 + sub;
        if (sb < nsb) {
            const int4 a0 = *(const int4 *)(act + sb * 256 + 64 * j + 16 * hf);
            const int4 a1 = *(const int4 *)(act + sb * 256 + 64 * j + 32 + 16 * hf);
            const float d8 = ad[sb];
            const int b0 = abs_[sb * 16 + 4 * j + hf], b1 = abs_[sb * 16 + 4 * j + 2 + hf];
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const unsigned char *row = rr ? row1 : row0;
                const uint4 qs = *((const uint4 *)row + sb * 8 + j * 2 + hf);
                const uint4 qh = *((const uint4 *)(row + (size_t)nsb * 128) + sb * 2 + hf);
                const uint4 sc = *((const uint4 *)(row + (size_t)nsb * 160) + sb);
                const unsigned qv[4] = {qs.x, qs.y, qs.z, qs.w}, hv[4] = {qh.x, qh.y, qh.z, qh.w};
                int lo[4], hi[4];
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    lo[i] = (int)((qv[i] & 0x0F0F0F0Fu) | (((hv[i] >> (2 * j)) & 0x01010101u) << 4));
                    hi[i] = (int)(((qv[i] >> 4) & 0x0F0F0F0Fu) | (((hv[i] >> (2 * j + 1)) & 0x01010101u) << 4));
                }
                int sca, scb, mna, mnb;
                const unsigned char *sp = (const unsigned char *)&sc;
                scale_min_k4(sp, 2 * j, sca, mna); scale_min_k4(sp, 2 * j + 1, scb, mnb);
                const float2 f = __half22float2(*(const __half2 *)&sc.w);
                int s0 = __dp4a(lo[0], a0.x, 0); s0 = __dp4a(lo[1], a0.y, s0); s0 = __dp4a(lo[2], a0.z, s0); s0 = __dp4a(lo[3], a0.w, s0);
                int s1 = __dp4a(hi[0], a1.x, 0); s1 = __dp4a(hi[1], a1.y, s1); s1 = __dp4a(hi[2], a1.z, s1); s1 = __dp4a(hi[3], a1.w, s1);
                const float dv = (f.x * d8) * (float)(sca * s0 + scb * s1), mv = (f.y * d8) * (float)(mna * b0 + mnb * b1);
                if (rr) { r.d1 += dv; r.m1 += mv; } else { r.d0 += dv; r.m0 += mv; }
            }
        }
    }
    return r;
}

// shared memory carve-up (dynamic): [2 W slots][act][2 W "full" mbarriers]
struct Smem6 { unsigned char *slots, *actb; uint64_t *full; };
__device__ __forceinline__ Smem6 carve6(const Params6 &P) {
    extern __shared__ __align__(128) unsigned char smem[];
    Smem6 m;
    m.slots = smem; m.actb = smem + (size_t)2 * P.W * P.slot_bytes;
    m.full = (uint64_t *)(m.actb + P.act_bytes);
    return m;
}

// ---- the warp's private stream cursor: which slot-load to request next.  Everything is warp-uniform and lives in registers; lane 0 issues.
//   src / bytes: the next slot-load; stride: added to src after it (parts == 2: alternates between "next row" and "first row of my next pair"
//   via stride ^= stride_xor); left: slot-loads of the current op still to request; cnt: loads requested so far (slot = cnt & 1).
struct Fill { const unsigned char *src; unsigned bytes, stride, stride_xor; int left, oi; unsigned cnt; };
__device__ __forceinline__ void fill_seek(const Params6 &P, const int2 *share, Fill &f, int warp) {   // first op at or after f.oi that has a unit for this warp
    f.left = 0;
    for (; f.oi < P.n_ops; ++f.oi) {
        const Op6 &op = P.ops[f.oi];
        if (!op.w) continue;
        const int2 lh = share[op.kind];
        const int mine = lh.y - lh.x - warp;   // units lo + warp, lo + warp + W, ...
        if (mine <= 0) continue;
        const unsigned ub = 2u * (unsigned)op.row_bytes, w_ub = (unsigned)P.W * ub;
        f.src = op.w + (size_t)(lh.x + warp) * ub;
        if (op.parts == 2) { f.bytes = (unsigned)op.row_bytes; f.stride = f.bytes; f.stride_xor = f.bytes ^ (w_ub - f.bytes); }
        else { f.bytes = ub; f.stride = w_ub; f.stride_xor = 0u; }
        f.left = ((mine + P.W - 1) / P.W) * op.parts;
        return;
    }
}
__device__ __forceinline__ void fill_one(const Params6 &P, const Smem6 &m, const int2 *share, Fill &f, int warp, int lane) {
    if (f.left == 0) return;
    if (lane == 0) {
        const unsigned j = 2u * (unsigned)warp + (f.cnt & 1u);
        mb_expect_tx(&m.full[j], f.bytes);
        bulk_g2s(m.slots + (size_t)j * P.slot_bytes, f.src, f.bytes, &m.full[j]);
    }
    f.src += f.stride; f.stride ^= f.stride_xor; ++f.cnt;
    if (--f.left == 0) { ++f.oi; fill_seek(P, share, f, warp); }
}

// The matvec phase of one op for one stream warp: for each of its row pairs wait for the slot(s), dot, re-arm the slot(s), reduce, epilogue.
//   cc = slot-loads this warp has consumed so far: load n sits in slot n & 1 and completes phase (n >> 1) & 1 of that slot's barrier.
template <int WT, int KIND, int NBL, bool TRACE>
__device__ __forceinline__ void consume6(const Params6 &P, const Smem6 &m, const int2 *share, int oi, Fill &f, unsigned &cc, int pos, long long *tr) {
    constexpr bool Q41 = WT == GG_Q4_1, Q5K = WT == GG_Q5_K;
    const Op6 &op = P.ops[oi];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int W = P.W;
    if (warp >= W) return;
    const int2 lh = share[KIND];
    const int lo = lh.x, hi = lh.y;
    const int cols = op.cols, nb = cols >> 5, parts = op.parts;
    const unsigned rb = (unsigned)op.row_bytes;
    // n_embd-wide RMS-normed inputs (qkv, gate/up, output) are held in registers; wo (8 % of the bytes; El wide under tensor parallelism) and
    // down read the staged vector from shared memory
    constexpr bool REG = !Q5K && NBL > 0 && KIND != OP_DOWN && KIND != OP_WO;
    ActRegs<REG ? NBL : 1> ar;
    if (REG) load_act_regs<REG ? NBL : 1>(m.actb, cols, lane, ar);
    unsigned char *const slot0 = m.slots + (size_t)(2 * warp) * P.slot_bytes;
    uint64_t *const full0 = &m.full[2 * warp];
    const bool hi16 = (lane & 16) != 0, hi8 = (lane & 8) != 0;
    unsigned long long best = 0ull;
    // gate/up epilogue (lane 0): the SiLU table lookup of a unit is issued after its dot product and consumed after the NEXT unit's, so its L2
    // latency is off the warp's critical path
    __half pend_h = __ushort_as_half((unsigned short)0); float pend_up = 0.f; int pend_i = -1;
    long long t_wait = 0, t_dot = 0, t_epi = 0; int n_units = 0;
    for (int u = lo + warp; u < hi; u += W) {
        const int r0 = u * 2;
        // QKV: rows [0, El) = q, [El, 2 El) = k, [2 El, 3 El) = v (El = this rank's heads); rr = row inside the part (head_dim 128: RoPE pair index (rr & 127) / 2)
        const int partn = KIND == OP_QKV ? (r0 >= P.El) + (r0 >= 2 * P.El) : 0, rr = r0 - partn * P.El;
        float2 rs = make_float2(0.f, 0.f);  // residual rows of this pair / RoPE (cos, sin) of this pair: fetched before the wait
        if ((KIND == OP_WO || KIND == OP_DOWN) && P.tp.world <= 1) rs = __ldcg((const float2 *)(P.x + r0));
        if (KIND == OP_QKV) { if (partn < 2) rs = __ldg(&P.rope[(size_t)pos * 64 + ((rr & 127) >> 1)]); }
        long long tw0 = 0, tw1 = 0, tw2 = 0;
        if (TRACE && tr) tw0 = clock64();
        const unsigned j0 = cc & 1u;
        mb_wait(full0 + j0, (cc >> 1) & 1u);
        const unsigned char *row0 = slot0 + (size_t)j0 * P.slot_bytes, *row1 = row0 + rb;
        if (parts == 2) { mb_wait(full0 + (j0 ^ 1u), ((cc + 1u) >> 1) & 1u); row1 = slot0 + (size_t)(j0 ^ 1u) * P.slot_bytes; }
        cc += (unsigned)parts;
        if (TRACE && tr) tw1 = clock64();
        Acc4 a;
        if (Q5K) a = dot2_q5k_smem(row0, row1, cols >> 8, cols, m.actb, lane);
        else if (REG) a = dot2_q4_reg<Q41, REG ? NBL : 1>(row0, row1, ar, lane);
        else a = dot2_q4_smem<Q41>(row0, row1, nb, cols, m.actb, lane);
        // Butterfly reductions of the four partial sums, PACKED: stage 16 leaves (d, m) of row 0 in lanes 0-15 and of row 1 in lanes 16-31,
        // stage 8 leaves one quantity per lane (d in lanes with bit 3 clear, m in the others), stages 4-2-1 are plain.  Every surviving lane
        // performs exactly the additions the plain butterfly performs at that lane (float addition commutes), so the sums are bit-identical to
        // warp_sum().  A lane's stage-16 operands are final only after all of its reads of the slot have returned -> the slot can be re-armed.
        float x = hi16 ? a.d1 : a.d0, y = hi16 ? a.m1 : a.m0;
        x += __shfl_xor_sync(0xffffffffu, hi16 ? a.d0 : a.d1, 16);
        y += __shfl_xor_sync(0xffffffffu, hi16 ? a.m0 : a.m1, 16);
        fill_one(P, m, share, f, warp, lane);
        if (parts == 2) fill_one(P, m, share, f, warp, lane);
        if (TRACE && tr) { tw2 = clock64(); t_wait += tw1 - tw0; t_dot += tw2 - tw1; ++n_units; }
        float z = hi8 ? y : x;
        z += __shfl_xor_sync(0xffffffffu, hi8 ? x : y, 8);
        z += __shfl_xor_sync(0xffffffffu, z, 4); z += __shfl_xor_sync(0xffffffffu, z, 2); z += __shfl_xor_sync(0xffffffffu, z, 1);
        // lanes 0-7: sum d of row 0, 8-15: sum m of row 0, 16-23: sum d of row 1, 24-31: sum m of row 1
        const float zz = __shfl_xor_sync(0xffffffffu, z, 8);
        const float v = Q5K ? z - zz : z + zz;              // lane 0: row 0 = warp_sum(d0) + warp_sum(m0) (Q5_K: minus, the mins term); lane 16: row 1
        const float v1 = __shfl_xor_sync(0xffffffffu, v, 16), v0 = v;
        if (lane == 0) {
            if (KIND == OP_QKV) {
                const size_t kvo = ((size_t)op.layer * P.n_ctx + pos) * P.El + rr;
                if (partn == 2) { *(__half2 *)(P.vcache + kvo) = __floats2half2_rn(v0, v1); }
                else {
                    const float2 cs = rs;
                    const float o0 = v0 * cs.x - v1 * cs.y, o1 = v0 * cs.y + v1 * cs.x;
                    if (partn == 0) *(float2 *)(P.q + rr) = make_float2(o0, o1);
                    else *(__half2 *)(P.kcache + kvo) = __floats2half2_rn(o0, o1);
                }
            } else if (KIND == OP_WO || KIND == OP_DOWN) {
                if (P.tp.world <= 1) *(float2 *)(P.x + r0) = make_float2(v0 + rs.x, v1 + rs.y);
                else *(float2 *)(P.tp.partial[P.tp.rank][KIND == OP_WO ? 0 : 1] + r0) = make_float2(v0, v1);   // partial sum over this rank's columns
            } else if (KIND == OP_GATEUP) {
                if (pend_i >= 0) P.act[pend_i] = __half2float(pend_h) * pend_up;
                pend_h = P.tab_silu[__half_as_ushort(__float2half_rn(v0))]; pend_up = v1; pend_i = r0 >> 1;
            } else {  // OP_OUTPUT
                P.logits[r0] = v0;
                const unsigned long long k0 = argmax_key(v0, r0);
                best = best > k0 ? best : k0;
                if (r0 + 1 < P.n_vocab) { P.logits[r0 + 1] = v1; const unsigned long long k1 = argmax_key(v1, r0 + 1); best = best > k1 ? best : k1; }
            }
        }
        if (TRACE && tr) t_epi += clock64() - tw2;
    }
    if (KIND == OP_GATEUP) { if (lane == 0 && pend_i >= 0) P.act[pend_i] = __half2float(pend_h) * pend_up; }
    if (KIND == OP_OUTPUT) { if (lane == 0 && best) atomicMax(&P.state->argmax_key, best); }
    if (TRACE && tr) { tr[4] = t_wait; tr[5] = t_dot; tr[6] = n_units; tr[7] = t_epi; }
}

// ---- attention of one head (256 threads = warps 0-7 of CTA h): k::attention_head with the CTA-wide reductions restructured for latency
// (4 named-barrier syncs instead of 10: the max comes out of the score loop, the second level of the soft-max sum is done redundantly by every
// warp).  Every float / double operation and its order are those of k::attention_head (max is order-free), so the output is bit-identical.
// out-of-line so that the attention code gets its own register allocation (it runs on n_head CTAs only)
__device__ __noinline__ void attention6(const float *__restrict__ q, const __half *__restrict__ kc, const __half *__restrict__ vc, float *__restrict__ out,
                                         int pos, int h, int E, int n_ctx, float kq_scale, const __half *__restrict__ tab_exp,
                                         unsigned char *dyn, double *red, float *redf, float *part /*[16*128]*/, long long *tr) {
    float *sc = (float *)dyn; __half *ph = (__half *)(dyn + (size_t)n_ctx * 4);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nkv = pos + 1;
    constexpr int B = 12;  // keys in flight per half-warp (192 keys per pass): all loads of a batch are issued before the first use
    float wmax = -INFINITY;
    {
        const int sub = lane >> 4, l16 = lane & 15;
        __half2 q2[4];
        bool have_q = false;
        for (int kb0 = warp * 2; kb0 < nkv || !have_q; kb0 += 16 * B) {  // warp-uniform trip counts (both half-warps shuffle together)
            uint4 kv[B];
#pragma unroll
            for (int u = 0; u < B; ++u) {
                const int key = min(kb0 + u * 16 + sub, nkv - 1);  // clamped, unconditional: a predicated load would demote kv[] to local memory
                kv[u] = __ldcg((const uint4 *)(kc + (size_t)key * E + h * 128 + l16 * 8));
            }
            if (!have_q) {
                const float4 qa = __ldcg((const float4 *)(q + h * 128 + l16 * 8)), qb = __ldcg((const float4 *)(q + h * 128 + l16 * 8 + 4));
                q2[0] = __floats2half2_rn(qa.x, qa.y); q2[1] = __floats2half2_rn(qa.z, qa.w); q2[2] = __floats2half2_rn(qb.x, qb.y); q2[3] = __floats2half2_rn(qb.z, qb.w);
                have_q = true;
            }
            float sv[B];
#pragma unroll
            for (int u = 0; u < B; ++u) {
                const int key = kb0 + u * 16 + sub;
                float s = 0.f;
                if (key < nkv) {
                    const __half2 *k2 = (const __half2 *)&kv[u];
#pragma unroll
                    for (int j = 0; j < 4; ++j) { const float2 a = __half22float2(k2[j]), b = __half22float2(q2[j]); s = fmaf(a.x, b.x, s); s = fmaf(a.y, b.y, s); }
                }
                sv[u] = s;
            }
#pragma unroll
            for (int o = 8; o > 0; o >>= 1)   // stage-major: the B butterflies advance together (see quant_items)
#pragma unroll
                for (int u = 0; u < B; ++u) sv[u] += __shfl_xor_sync(0xffffffffu, sv[u], o);
#pragma unroll
            for (int u = 0; u < B; ++u) {
                const int key = kb0 + u * 16 + sub;
                if (key < nkv && l16 == 0) { const float v = sv[u] * kq_scale; sc[key] = v; wmax = fmaxf(wmax, v); }
            }
        }
    }
    // the first batch of V rows does not depend on the scores - request it now, so its round trip runs under the soft-max
    constexpr int BV = 12;
    uint4 vv0[BV];
#pragma unroll
    for (int u = 0; u < BV; ++u) { const int key = min((tid >> 4) + 16 * u, nkv - 1); vv0[u] = __ldcg((const uint4 *)(vc + (size_t)key * E + h * 128 + (tid & 15) * 8)); }
    wmax = warp_max(wmax);
    if (lane == 0) redf[warp] = wmax;
    cta_sync<true>();   // (1) scores and the eight warp maxima are visible
    if (tr) tr[8] = clock64();
    float mx = redf[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) mx = fmaxf(mx, redf[w]);
    double sum = 0.0;
    for (int i = tid; i < nkv; i += 256) { const float v = lut_f16(tab_exp, sc[i] - mx); sc[i] = v; sum += (double)v; }
    sum = warp_sum(sum);
    if (lane == 0) red[warp] = sum;
    cta_sync<true>();   // (2) the eight warp sums are visible; every warp folds them the way k::block_sum's warp 0 does
    double t = lane < 8 ? red[lane] : 0.0;
    t = warp_sum(t);
    if (tr) tr[9] = clock64();
    const float inv = (float)(1.0 / t);
    for (int i = tid; i < nkv; i += 256) ph[i] = __float2half_rn(sc[i] * inv);
    cta_sync<true>();   // (3) probabilities are visible
    if (tr) tr[10] = clock64();
    // P.V : thread = (key group g of 16, dim octet o of 16); groups are combined by a pairwise tree (canonical order)
    {
        const int g = tid >> 4, o = tid & 15;
        float acc[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = 0.f;
#pragma unroll
        for (int u = 0; u < BV; ++u) {  // the batch requested before the soft-max (keys g, g+16, ...: same sequential FMA order)
            const int key = g + 16 * u;
            if (key < nkv) {
                const float p = __half2float(ph[key]);
                const __half2 *v2 = (const __half2 *)&vv0[u];
#pragma unroll
                for (int j = 0; j < 4; ++j) { const float2 v = __half22float2(v2[j]); acc[2 * j] = fmaf(v.x, p, acc[2 * j]); acc[2 * j + 1] = fmaf(v.y, p, acc[2 * j + 1]); }
            }
        }
        for (int key0 = g + 16 * BV; key0 < nkv; key0 += 16 * B) {  // batch the V loads (192 keys per pass); the FMA order over keys stays sequential
            uint4 vv[B];
#pragma unroll
            for (int u = 0; u < B; ++u) { const int key = min(key0 + 16 * u, nkv - 1); vv[u] = __ldcg((const uint4 *)(vc + (size_t)key * E + h * 128 + o * 8)); }
#pragma unroll
            for (int u = 0; u < B; ++u) {
                const int key = key0 + 16 * u;
                if (key < nkv) {
                    const float p = __half2float(ph[key]);
                    const __half2 *v2 = (const __half2 *)&vv[u];
#pragma unroll
                    for (int j = 0; j < 4; ++j) { const float2 v = __half22float2(v2[j]); acc[2 * j] = fmaf(v.x, p, acc[2 * j]); acc[2 * j + 1] = fmaf(v.y, p, acc[2 * j + 1]); }
                }
            }
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) part[g * 128 + o * 8 + e] = acc[e];
    }
    cta_sync<true>();   // (4) the 16 partial outputs per dimension are visible
    if (tid < 128) {
        float v[16];
#pragma unroll
        for (int g = 0; g < 16; ++g) v[g] = part[g * 128 + tid];
#pragma unroll
        for (int st = 1; st < 16; st <<= 1)
#pragma unroll
            for (int g = 0; g < 16; g += 2 * st) v[g] = v[g] + v[g + st];
        out[h * 128 + tid] = v[0];
    }
    if (tr) tr[11] = clock64();
}

template <int WT, int NBL, bool TRACE>
__global__ void __launch_bounds__(kThreads, 1) decode_megakernel6(const __grid_constant__ Params6 P) {
    __shared__ double red[34];
    __shared__ float redf[34];
    __shared__ float part[16 * 128];
    __shared__ int2 share[8];   // this CTA's contiguous share [lo, hi) of the row pairs of each op kind
    constexpr int ACT = act_of(WT);
    const Smem6 m = carve6(P);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int G = (int)gridDim.x, cta = (int)blockIdx.x;

    if (tid == 0) {
        for (int s = 0; s < 2 * P.W; ++s) mb_init(&m.full[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (tid < 8) share[tid] = make_int2(unit_begin(cta, P.n_su_kind[tid], G), unit_begin(cta + 1, P.n_su_kind[tid], G));
    __syncthreads();  // the only CTA-wide barrier; afterwards warps 0-14 use named barriers 2 (480 threads) and 1 (256 threads)
    if (warp >= kConsumerWarps) return;   // (warp 15 only pads the CTA to four warps per scheduler)

    // start the stream: the first two slot-loads of this warp
    Fill f{nullptr, 0u, 0u, 0u, 0, 0, 0u};
    unsigned cc = 0;
    if (warp < P.W) {
        fill_seek(P, share, f, warp);
        fill_one(P, m, share, f, warp, lane);
        fill_one(P, m, share, f, warp, lane);
    }

    unsigned bar_target = 0, n_reduce = 0;
    const unsigned tp_seq0 = P.tp.world > 1 ? __ldcg(P.tp_seq) : 0u;
    const int pos = __ldcg(&P.state->n_past);  // position of the token being decoded (state only changes in OP_FINAL)
    for (int oi = 0; oi < P.n_ops; ++oi) {
        const int kind = P.ops[oi].kind;
        long long *tr = nullptr;
        if (TRACE) { if (P.trace && tid == 0 && (cta == 0 || cta == G - 1)) tr = P.trace + ((size_t)(cta == 0 ? 0 : 1) * P.n_ops + oi) * 16; }
        if (TRACE && tr) { tr[0] = clock64(); for (int i = 2; i < 16; ++i) tr[i] = 0; }
        if (oi > 0) bar_target += (unsigned)G;
        if (kind == OP_EMBED || kind == OP_ATTN || kind == OP_FINAL) {
            if (oi > 0) grid_barrier(P.barrier, bar_target);
            if (TRACE && tr) tr[1] = clock64();
            if (kind == OP_EMBED) {   // token embedding row -> x (dequantised on the fly), spread over the grid
                const int token = __ldcg(&P.state->tokens[0]);
                const unsigned char *row = P.tok + (size_t)token * P.tok_row_bytes;
                for (int i = cta * kConsumerThreads + tid; i < P.E; i += G * kConsumerThreads) P.x[i] = dequant_elem(P.tok_type, row, i);
            } else if (kind == OP_ATTN) {
                if (cta < P.n_head && tid < 256) {  // one head per CTA, 256 threads (named barrier 1)
                    const size_t lo = (size_t)P.ops[oi].layer * P.n_ctx * P.El;
                    attention6(P.q, P.kcache + lo, P.vcache + lo, P.att, pos, cta, P.El, P.n_ctx, P.kq_scale, P.tab_exp, m.actb, red, redf, part, TRACE ? tr : nullptr);
                }
            } else if (cta == 0 && tid == 0) {
                DeviceState *st = P.state;
                const unsigned long long key = __ldcg((const unsigned long long *)&st->argmax_key);
                const int id = (int)(0xFFFFFFFFu - (unsigned)(key & 0xFFFFFFFFull));
                st->argmax_id = id; st->tokens[0] = id; st->argmax_key = 0ull;
                st->n_past += 1; st->n_tok = 1;
                if (P.tp.world > 1) *P.tp_seq = tp_seq0 + n_reduce;   // (every reduce of this launch has completed on this rank)
            }
            if (TRACE && tr) tr[3] = clock64();
            continue;
        }
        if (kind == OP_REDUCE) {
            // Tensor-parallel sum of the partial vectors of the row-split matmul that just ran (wo: exchange buffer 0, down: buffer 1):
            //   x += sum over ranks, in rank order, of partial_r          (the same additions in the same order on every rank)
            // [grid barrier: this rank's partial is complete] -> CTA 0 publishes a sequence number into every rank's flag words (one store per peer
            // over NVLink) -> kReduceCtas CTAs wait for all ranks' flags, then read their slice of every partial straight out of peer memory.
            // A buffer is rewritten two reduces later; by then every peer has passed the reduce in between, i.e. finished reading this one.
            const unsigned seq = tp_seq0 + (++n_reduce);
            const int buf = P.ops[oi].layer;   // (the op's `layer` field carries the buffer index: 0 after wo, 1 after down)
            grid_barrier(P.barrier, bar_target);
            if (TRACE && tr) tr[1] = clock64();
            if (cta == 0 && tid < P.tp.world) {
                asm volatile("fence.acq_rel.sys;" ::: "memory");
                asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(P.tp.flags[tid] + P.tp.rank), "r"(seq) : "memory");
            }
            if (cta < kReduceCtas) {
                if (tid < P.tp.world) {
                    unsigned v, spins = 0; const unsigned *fl = P.tp.flags[P.tp.rank] + tid;
                    for (;;) {
                        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(fl) : "memory");
                        if ((int)(v - seq) >= 0) break;
                        if (++spins > (1u << 24)) asm volatile("trap;");   // a lost peer must end in a failed launch, never in a hung GPU
                        __nanosleep(64);
                    }
                }
                consumer_sync();
                if (TRACE && tr) tr[2] = clock64();
                const int per = P.E / kReduceCtas;   // (n_embd % 256 == 0: a multiple of 16)
                for (int i = cta * per + tid * 4; i < (cta + 1) * per; i += kConsumerThreads * 4) {
                    float4 acc = __ldcg((const float4 *)(P.x + i));
                    for (int r = 0; r < P.tp.world; ++r) {
                        float4 v;
                        asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(P.tp.partial[r][buf] + i) : "memory");
                        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                    }
                    *(float4 *)(P.x + i) = acc;
                }
            }
            if (TRACE && tr) tr[3] = clock64();
            continue;
        }
        // ---- matvec ops: [norm weights asked into L2 -> grid barrier -> stage activations] then [own row pairs: slot -> dot -> re-arm -> epilogue] ----
        {
            const int cols = P.ops[oi].cols;
            const float *nw = P.ops[oi].norm_w;
            if (nw && tid * 32 < cols) touch(nw + tid * 32);   // (before the barrier: the round trip runs under the wait)
            grid_barrier(P.barrier, bar_target);
            if (TRACE && tr) tr[1] = clock64();
            const float *src = kind == OP_WO ? P.att : kind == OP_DOWN ? P.act : P.x;
            if (ACT == ACT_Q8_K) stage_q8k(src, nw, cols, m.actb, red, P.E_pow2 != 0, P.inv_E, TRACE ? tr : nullptr);
            else if (nw) { if (tid < 256) stage_norm<ACT == ACT_Q8_K ? ACT_Q8_1 : ACT>(src, nw, cols, m.actb, red, P.E_pow2 != 0, P.inv_E, TRACE ? tr : nullptr); }
            else stage_plain<ACT == ACT_Q8_K ? ACT_Q8_1 : ACT>(src, cols, m.actb);
            if (TRACE && tr) tr[9] = clock64();
            consumer_sync();
            if (TRACE && tr) tr[2] = clock64();
        }
        if (kind == OP_QKV && (P.flags & 1) && cta < P.n_head) {   // (the loads are in flight while this CTA consumes its qkv rows)
            const size_t lo = (size_t)P.ops[oi].layer * P.n_ctx * P.El;
            touch_kv_head(P.kcache + lo, P.vcache + lo, P.tab_exp, pos, cta, P.El);
        }
        switch (kind) {
            case OP_QKV:    consume6<WT, OP_QKV, NBL, TRACE>(P, m, share, oi, f, cc, pos, tr); break;
            case OP_WO:     consume6<WT, OP_WO, NBL, TRACE>(P, m, share, oi, f, cc, pos, tr); break;
            case OP_GATEUP: consume6<WT, OP_GATEUP, NBL, TRACE>(P, m, share, oi, f, cc, pos, tr); break;
            case OP_DOWN:   consume6<WT, OP_DOWN, NBL, TRACE>(P, m, share, oi, f, cc, pos, tr); break;
            default:        consume6<WT, OP_OUTPUT, NBL, TRACE>(P, m, share, oi, f, cc, pos, tr); break;
        }
        if (TRACE && tr) tr[3] = clock64();  // (thread 0 = warp 0 only; other warps may still be consuming)
    }
}

}  // namespace mk6
}  // namespace mg4

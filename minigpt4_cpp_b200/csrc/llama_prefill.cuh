// llama_prefill.cuh — tensor-core prefill for Q4_0 / Q4_1 LLaMA matrices: N >= 2 rows of llama_eval / llama_eval_embd in ONE pass over
// the weights (reference call sites minigpt4.cpp:2365-2382 add_tokens in n_batch chunks, :2399-2415 add_embedding = 32 rows at once).
//
// Semantics are ggml's quantised mul_mat, exactly as the decode matvec (llama_kernels.cuh): activations quantised to Q8_0 / Q8_1 per 32,
// INTEGER block dot products, F32 scaling.  Here the integer dots run on the Hopper tensor cores:
//   * a CTA owns 128 weight rows x 32 tokens; each of its four consumer warpgroups owns a 64-row x 16-token quarter and issues one
//     wgmma.mma_async m64n16k32 s8 x s8 -> s32 (K = 32 = ONE quant block, no accumulation) per quant block, which leaves the exact int32
//     block dots in its registers (a thread holds 2 rows x 4 tokens); the per-block scales cannot be folded into the MMA, so
//   * the same sixteen warps apply  d_w * d_a * isum  and  m_w * s_a  on the CUDA cores and
//     accumulate in the CANONICAL FLOAT ORDER of oracle.cpp / k::dot2_q4: "lane" class l = b mod 32 accumulates its blocks l, l+32, ...
//     in increasing order; the 32 class sums are then combined by the xor-butterfly tree (16, 8, 4, 2, 1).  The K loop therefore walks
//     the classes in bit-reversed order (0, 16, 8, 24, ...), which turns the butterfly into a post-order tree walk with a 5-deep stack
//     per output (level 0 in registers, levels 1-4 in shared memory).  Result: bit-identical to the matvec path, for any N.
//   * operands come from a load-time "prefill operand cache": the nibbles expanded to int8 (Q4_0: q - 8, so the "-8 * sum(a)" term is
//     inside the integer dot) in CLASS-MAJOR order — row r = [class l][slot i][32 bytes] — so that one 128-byte TMA box row holds four
//     consecutive blocks of one class (SWIZZLE_128B, the layout the tensor core reads); the staged activations use the same order.
//     (Trade: +1 byte per weight of HBM for the cache, 6.5 GB for a 7B model; the decode path keeps streaming the 4-bit original.)
// The kernel is epilogue-bound by construction (5 CUDA-core instructions per (row, token, block) against 32 int8 MACs on the tensor core):
// exact Q8 semantics cost that; what the tensor core removes is the 8 dp4a + nibble unpacking per (row, token, block) of the matvec path.
// Inside a warp nothing overlaps its MMAs (issue, commit, wait, scale); whether the other warps of a scheduler hide that wait is not measured.
#pragma once
#include "llama_kernels.cuh"
#include <cuda.h>

namespace mg4 {
namespace pf {
using namespace k;

constexpr int kTok = 32;          // tokens per CTA
constexpr int kRows = 128;        // weight rows per CTA
constexpr int kStages = 4;        // shared-memory pipeline depth (tiles of 4 blocks)
constexpr int kStageBytes = 16384 + 4096 + 1024;  // A 128 x 128 B | B 32 x 128 B | activation scales 32 x 4 x {d, s}
constexpr int kConsWarps = 16;    // four warpgroups: (row half, token half) of the tile, wgmma M = 64, N = 16
constexpr int kOut = 8;           // outputs per consumer thread: 2 rows x 4 tokens, in wgmma accumulator order
constexpr int kThreads = 32 * kConsWarps + 32;    // warps 0-15 = MMA + epilogue, warp 16 = TMA producer
constexpr int kStackBytes = 4 * kTok * kRows * 8; // stack levels 1-4: [level][output of the thread][thread] {d-tree, m-tree}
static_assert(kOut * 32 * kConsWarps == kTok * kRows, "one stack slot per output of the tile");

struct PrefillArgs {
    int rows;            // valid weight rows (the operand cache is padded to a multiple of 128 rows)
    int n_tok;           // valid tokens (grid.y = ceil(n_tok / 32))
    int nb, S;           // quant blocks per row; slots per class in the class-major layout (multiple of 4)
    const __half2 *wsc;  // [rows_pad][32 * S] {d, m} of the block in (class, slot) order
    int epi;             // k::Epi (EPI_PLAIN, EPI_QKV, EPI_RESID, EPI_SWIGLU)
    float *out; int out_stride; const float *resid;
    float *q_out; __half *kcache; __half *vcache; const float2 *rope; int e_local; int half_dim;
    const DeviceState *state;
    const __half *tab_silu;
    // K split (grid.z > 1): slice z covers the classes of the leaves jr in [z * jr_per_z, (z + 1) * jr_per_z) of the butterfly tree - a complete
    // subtree - and writes its root {d-tree, m-tree} to partial[(z * part_tok + t) * part_rows + r]; prefill_combine folds the roots and runs the epilogue
    int jr_per_z; float2 *partial; int part_tok, part_rows;
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "PF_WAIT:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra PF_DONE;\n\t"
        "bra PF_WAIT;\n\t"
        "PF_DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, int c0, int c1, uint64_t *bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// D[64 x 16] = A[64 x 32] . B[16 x 32]^T from shared memory, int8 x int8 -> int32, no accumulation (every quant block gets its own registers):
// thread (warp w, lane) of the warpgroup holds d[4 j + 2 h + e] = D[16 w + lane / 4 + 8 h][8 j + 2 (lane % 4) + e]
__device__ __forceinline__ void wgmma_i8_n16(int (&d)[kOut], uint64_t adesc, uint64_t bdesc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 0, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k32.s32.s8.s8 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p;\n\t}"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]) : "l"(adesc), "l"(bdesc));
}
// K-major, SWIZZLE_128B shared-memory matrix descriptor (as vision_kernels.cuh: layout type 1 in bits 62-63, SBO = 8 rows * 128 B)
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
__device__ __forceinline__ uint4 ldg_nc16(const void *p) {
    uint4 r;
    asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__host__ __device__ __forceinline__ int bitrev5(int v) { return ((v & 1) << 4) | ((v & 2) << 2) | (v & 4) | ((v & 8) >> 2) | ((v & 16) >> 4); }
// valid blocks of tile j of class l: blocks b = l + 32 i, i = 4 j .. 4 j + 3, b < nb
__host__ __device__ __forceinline__ int tile_blocks(int nb, int l, int j) {
    const int n_l = nb > l ? (nb - l + 31) / 32 : 0;
    const int v = n_l - 4 * j;
    return v < 0 ? 0 : (v > 4 ? 4 : v);
}

// fused output of one result (row r, token t): res = this row, other = the adjacent row of the pair (RoPE / SwiGLU pair adjacent rows);
// the epilogues of k::matvec_kernel
__device__ __forceinline__ void prefill_epilogue(const PrefillArgs &g, int r, int t, int n_past, float res, float other) {
    if (g.epi == EPI_QKV) {
        const int E = g.e_local, part = r / E, rr = r % E, pos = n_past + t;
        if (part == 2) g.vcache[(size_t)pos * E + rr] = __float2half_rn(res);
        else {
            const float2 cs = g.rope[(size_t)pos * g.half_dim + (rr % (2 * g.half_dim)) / 2];
            const float v0 = (rr & 1) ? other : res, v1 = (rr & 1) ? res : other;
            const float o = (rr & 1) ? (v0 * cs.y + v1 * cs.x) : (v0 * cs.x - v1 * cs.y);
            if (part == 0) g.q_out[(size_t)t * E + rr] = o;
            else g.kcache[(size_t)pos * E + rr] = __float2half_rn(o);
        }
    } else if (g.epi == EPI_RESID) {
        const size_t o = (size_t)t * g.out_stride + r;
        g.out[o] = res + g.resid[o];
    } else if (g.epi == EPI_SWIGLU) {  // rows are interleaved: even = gate(ff), odd = up(ff)
        if ((r & 1) == 0) g.out[(size_t)t * g.out_stride + (r >> 1)] = lut_f16(g.tab_silu, res) * other;
    } else {
        g.out[(size_t)t * g.out_stride + r] = res;
    }
}

// grid (rows_pad / 128, ceil(n_tok / 32)); block 544; dynamic smem = 1024 (alignment) + 4 stages + stack + barriers
template <bool Q41>
__global__ void __launch_bounds__(kThreads, 1) prefill_gemm_q4(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                                                                  const __grid_constant__ CUtensorMap tmS, const PrefillArgs g) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char *smem = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    float2 *stack = (float2 *)(smem + (size_t)kStages * kStageBytes);
    uint64_t *full = (uint64_t *)((unsigned char *)stack + kStackBytes);
    uint64_t *empty = full + kStages;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m_tile = blockIdx.x, t_tile = blockIdx.y;
    const int tpc = g.S >> 2;  // tiles per class
    const int jr0 = (int)blockIdx.z * g.jr_per_z, jr1 = jr0 + g.jr_per_z;   // leaves (classes in bit-reversed order) of this CTA's subtree

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmS) : "memory");
        for (int i = 0; i < kStages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], kConsWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == kConsWarps) {
        // ---------------- TMA producer ----------------
        if (lane == 0) {
            unsigned cnt = 0;
            for (int jr = jr0; jr < jr1; ++jr) {
                const int l = bitrev5(jr);
                for (int j = 0; j < tpc; ++j) {
                    if (tile_blocks(g.nb, l, j) == 0) continue;
                    const int s = (int)(cnt % kStages); const uint32_t ph = (cnt / kStages) & 1u; ++cnt;
                    mbar_wait(&empty[s], ph ^ 1u);
                    unsigned char *sa = smem + (size_t)s * kStageBytes;
                    mbar_expect_tx(&full[s], (uint32_t)kStageBytes);
                    const int slot0 = l * g.S + 4 * j;
                    tma_load_2d(sa, &tmA, slot0 * 32, m_tile * kRows, &full[s]);
                    tma_load_2d(sa + 16384, &tmB, slot0 * 32, t_tile * kTok, &full[s]);
                    tma_load_2d(sa + 16384 + 4096, &tmS, slot0 * 8, t_tile * kTok, &full[s]);
                }
            }
        }
        return;
    }
    // ---------------- consumers: block dots, scale, accumulate in canonical order, butterfly tree, fused output ----------------
    // output o = 4 j + 2 h + e of this thread: row row_in + 8 h, token tok0 + 8 j + e (the wgmma accumulator layout)
    const int wg = warp >> 2, rh = wg & 1, th = wg >> 1;
    const int row_in = rh * 64 + (warp & 3) * 16 + (lane >> 2), r = m_tile * kRows + row_in, tok0 = th * 16 + 2 * (lane & 3);
    const __half2 *wrow = g.wsc + (size_t)r * (32 * g.S);
    const size_t wrow8 = (size_t)8 * (32 * g.S);
    float2 *mystack = stack + threadIdx.x;   // level lev, output o: mystack[((lev - 1) * kOut + o) * 32 * kConsWarps]
    float accd[kOut], accm[kOut], l0d[kOut], l0m[kOut];
#pragma unroll
    for (int o = 0; o < kOut; ++o) { accd[o] = 0.f; accm[o] = 0.f; l0d[o] = 0.f; l0m[o] = 0.f; }
    unsigned cnt = 0;
    for (int jr = jr0; jr < jr1; ++jr) {
        const int l = bitrev5(jr);
        for (int j = 0; j < tpc; ++j) {
            const int v = tile_blocks(g.nb, l, j);
            if (v == 0) continue;
            const int s = (int)(cnt % kStages); const uint32_t ph = (cnt / kStages) & 1u; ++cnt;
            const uint4 w4[2] = {ldg_nc16(wrow + l * g.S + 4 * j), ldg_nc16(wrow + wrow8 + l * g.S + 4 * j)};   // {d, m} of the four blocks of both rows (issued before the wait)
            mbar_wait(&full[s], ph);       // operands and activation scales of the tile are in shared memory
            const uint32_t sa = smem_u32(smem + (size_t)s * kStageBytes) + (uint32_t)rh * 8192u, sb = sa - (uint32_t)rh * 8192u + 16384u + (uint32_t)th * 2048u;
            int isum[4][kOut];
            wgmma_fence();
#pragma unroll
            for (int i = 0; i < 4; ++i)   // all four: the slots past the last block of a class are zero padding, and an unconditional issue keeps the MMAs asynchronous
                wgmma_i8_n16(isum[i], wgmma_desc_sw128(sa + i * 32), wgmma_desc_sw128(sb + i * 32));
            wgmma_commit();
            wgmma_wait_all();
            const float2 *asc = (const float2 *)(smem + (size_t)s * kStageBytes + 16384 + 4096);  // [token][4] {d, s}
            const unsigned wv[2][4] = {{w4[0].x, w4[0].y, w4[0].z, w4[0].w}, {w4[1].x, w4[1].y, w4[1].z, w4[1].w}};
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                if (i < v) {
                    const float2 f[2] = {__half22float2(*(const __half2 *)&wv[0][i]), __half22float2(*(const __half2 *)&wv[1][i])};
#pragma unroll
                    for (int o = 0; o < kOut; ++o) {
                        const int h = (o >> 1) & 1;
                        const float2 ds = asc[(tok0 + 8 * (o >> 2) + (o & 1)) * 4 + i];
                        if (Q41) { accd[o] = fmaf(f[h].x * ds.x, (float)isum[i][o], accd[o]); accm[o] = fmaf(f[h].y, ds.y, accm[o]); }
                        else accd[o] += ((float)isum[i][o] * f[h].x) * ds.x;
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[s]);
        }
        // class l is complete: fold it into the butterfly tree (post-order walk, jr = leaf number in bit-reversed class order)
        const int jl = jr - jr0;   // leaf number inside this CTA's subtree (jr0 is a multiple of the subtree size)
        if ((jl & 1) == 0) {
#pragma unroll
            for (int o = 0; o < kOut; ++o) { l0d[o] = accd[o]; l0m[o] = accm[o]; accd[o] = 0.f; accm[o] = 0.f; }
        } else {
            int ones = 1; while (ones < 5 && ((jl >> ones) & 1)) ++ones;  // trailing ones of jl (>= 1)
#pragma unroll
            for (int o = 0; o < kOut; ++o) {
                float vd = l0d[o] + accd[o], vm = l0m[o] + accm[o];
                accd[o] = 0.f; accm[o] = 0.f;
                for (int lev = 1; lev < ones; ++lev) {
                    const float2 p = mystack[(size_t)((lev - 1) * kOut + o) * (32 * kConsWarps)];
                    vd = p.x + vd; vm = p.y + vm;
                }
                if (jr != jr1 - 1) mystack[(size_t)((ones - 1) * kOut + o) * (32 * kConsWarps)] = make_float2(vd, vm);
                else { l0d[o] = vd; l0m[o] = vm; }
            }
        }
    }
    // results: res[o] = d-tree + m-tree (k::dot2_q4: warp_sum(accd) + warp_sum(accm)); fused epilogues of k::matvec_kernel
    const int n_past = g.state->n_past;
#pragma unroll
    for (int o = 0; o < kOut; ++o) {
        const int t = t_tile * kTok + tok0 + 8 * (o >> 2) + (o & 1), ro = r + 8 * ((o >> 1) & 1);
        if (gridDim.z > 1) {   // K split: the root of this CTA's subtree; prefill_combine finishes the tree
            if (t < g.n_tok && ro < g.rows) g.partial[((size_t)blockIdx.z * g.part_tok + t) * g.part_rows + ro] = make_float2(l0d[o], l0m[o]);
            continue;
        }
        const float res = l0d[o] + l0m[o];
        const float other = __shfl_xor_sync(0xffffffffu, res, 4);   // the pair row (RoPE / SwiGLU pair adjacent rows) sits four lanes away
        if (t >= g.n_tok || ro >= g.rows) continue;
        prefill_epilogue(g, ro, t, n_past, res, other);
    }
}

// K-split GEMMs: fold the subtree roots of the grid.z slices (pairwise, in leaf order = the upper levels of the butterfly tree), then the epilogue.
// One thread per (token, row pair); nz = 2, 4 or 8.
__global__ void __launch_bounds__(256) prefill_combine(const PrefillArgs g, int nz) {
    const int pairs = g.rows >> 1;
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)g.n_tok * pairs) return;
    const int t = (int)(idx / pairs), r0 = 2 * (int)(idx % pairs);
    float res[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        float d[8], m[8];
        for (int z = 0; z < nz; ++z) { const float2 p = g.partial[((size_t)z * g.part_tok + t) * g.part_rows + r0 + k]; d[z] = p.x; m[z] = p.y; }
        for (int st = 1; st < nz; st <<= 1)
            for (int z = 0; z < nz; z += 2 * st) { d[z] = d[z] + d[z + st]; m[z] = m[z] + m[z + st]; }
        res[k] = d[0] + m[0];
    }
    const int n_past = g.state->n_past;
    prefill_epilogue(g, r0, t, n_past, res[0], res[1]);
    prefill_epilogue(g, r0 + 1, t, n_past, res[1], res[0]);
}

// ---------------------------------------------------------------------------------------------------------------------------------
// load time: row-packed Q4 rows ([nb x 16 B nibbles][nb x scales], llama.h) -> int8 class-major operand cache + {d, m} in the same order
// ---------------------------------------------------------------------------------------------------------------------------------
__global__ void expand_q4_classmajor(const unsigned char *src, int row_bytes, int rows, int nb, int q41, int S, signed char *q, __half2 *sc) {
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)rows * nb) return;
    const int r = (int)(idx / nb), b = (int)(idx % nb);
    const unsigned char *row = src + (size_t)r * row_bytes;
    const uint4 nib = ((const uint4 *)row)[b];
    const unsigned w[4] = {nib.x, nib.y, nib.z, nib.w};
    unsigned lo[4], hi[4];
    for (int k4 = 0; k4 < 4; ++k4) {
        lo[k4] = w[k4] & 0x0F0F0F0Fu; hi[k4] = (w[k4] >> 4) & 0x0F0F0F0Fu;
        if (!q41) { lo[k4] = __vsub4(lo[k4], 0x08080808u); hi[k4] = __vsub4(hi[k4], 0x08080808u); }
    }
    const int slot = (b & 31) * S + (b >> 5);
    uint4 *dst = (uint4 *)(q + ((size_t)r * 32 * S + slot) * 32);
    dst[0] = make_uint4(lo[0], lo[1], lo[2], lo[3]);   // elements 0..15 (low nibbles)
    dst[1] = make_uint4(hi[0], hi[1], hi[2], hi[3]);   // elements 16..31 (high nibbles)
    const unsigned char *scp = row + (size_t)nb * 16;
    __half2 v;
    if (q41) v = ((const __half2 *)scp)[b];
    else v = __halves2half2(((const __half *)scp)[b], __ushort_as_half((unsigned short)0));
    sc[(size_t)r * 32 * S + slot] = v;
}

// activations of N rows: (optional RMSNorm) + quantise exactly as k::stage_act, written in the class-major order of the operand cache:
// q8 [n_pad][32 * S * 32] int8, scales [n_pad][32 * S] {d, s}.  grid = n rows, 256 threads, dynamic smem = act_bytes(ACT, cols)
template <int ACT>
__global__ void __launch_bounds__(256) stage_rows_classmajor(const float *x, int x_stride, const float *norm_w, int cols, int S, signed char *q8, float2 *sc) {
    extern __shared__ __align__(16) unsigned char sm[];
    __shared__ double red[34];
    const int t = blockIdx.x, nb = cols >> 5;
    stage_act<ACT>(x + (size_t)t * x_stride, norm_w, cols, sm, red);
    __syncthreads();
    const float *d = (const float *)(sm + cols), *s = d + nb;
    for (int i = threadIdx.x; i < nb * 2; i += 256) {  // 16-byte halves of the blocks: lo plane [b], hi plane [b]
        const int b = i >> 1, hf = i & 1;
        const uint4 v = *(const uint4 *)(sm + (hf ? cols / 2 : 0) + b * 16);
        const int slot = (b & 31) * S + (b >> 5);
        *(uint4 *)(q8 + ((size_t)t * 32 * S + slot) * 32 + hf * 16) = v;
    }
    for (int b = threadIdx.x; b < nb; b += 256) sc[(size_t)t * 32 * S + (b & 31) * S + (b >> 5)] = make_float2(d[b], s[b]);
}

}  // namespace pf
}  // namespace mg4
